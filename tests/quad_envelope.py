"""Quadrotor states from the whole flight envelope, and plain float64 / literal restatements to judge a step by.

envelope_batch() draws [n, 22] float32 states (p3 v3 w3 prop4 R9, the state_dict() layout) in named families that
reach what reset states and recorded reference episodes never do: every attitude including the branch cuts of the
observed angles and gimbal lock, non-orthogonal rotation matrices, angular rates up to 900 rad/s, speeds up to 95 m/s,
positions up to 990 m, rotor speeds the applied voltage does not sustain and actions outside the voltage range.

observe_f64() is the observation of a state (metagym/quadrotor/quadrotorsim.py:111-120,260-293, env.py:193-209) in
float64 numpy with np.linalg.inv and np.arctan2, and collides_literal() is env.py:248-260 restated literally, with a
real numpy slice of the map.  CPU only: numpy, no torch.
"""
import math
from collections import namedtuple

import numpy as np

# the reference's config.json values this module needs (metagym/quadrotor/config.json)
PHI, RA, MM = 0.017242179827506, 0.2010, 0.010
MIN_V, MAX_V = 0.10, 15.0
FAIL_W, FAIL_V, FAIL_R = 1000.0, 100.0, 1000.0
GRAVITY = np.float32(-9.8)

# roll, pitch and yaw of the attitude grid: the quarter turns and both sides of the +-pi branch cut
GRID_ANGLES = (0.0, math.pi / 4, -math.pi / 4, math.pi / 2, -math.pi / 2, 3 * math.pi / 4, -3 * math.pi / 4,
               math.pi, -math.pi, math.pi - 1e-6, -(math.pi - 1e-6))

FAMILIES = ("grid", "inverted", "gimbal", "haar", "drifted", "rates_body", "rates_random", "velocity", "position",
            "altitude", "rotors", "actions", "counters", "control")

Envelope = namedtuple("Envelope", ["state", "ct", "act", "family"])


def zero_thrust_voltage():
    """The float32 voltage V at which a rotor at rest stays at rest: (phi/ra) V rounds to Mm exactly in float32
    (quadrotorsim.py:136-145, w' = w + h/Jm (me - Mm) with me = (phi/ra)(V - phi w)).  Four such rotors give no thrust
    and no torque, so a state with w = 0 keeps its attitude to the bit through a step."""
    k1, mm = np.float32(PHI / RA), np.float32(MM)
    v = np.float32(float(mm) / float(k1))
    for _ in range(64):
        prod = np.float32(np.float64(k1) * np.float64(v))
        if prod == mm:
            return v
        v = np.nextafter(v, np.float32(np.inf) if prod < mm else np.float32(-np.inf))
    raise AssertionError("no float32 voltage holds a resting rotor at rest")


def hover_speed(volt=MAX_V):
    """Rotor speed the voltage sustains: me = Mm, i.e. w = (V - Mm ra / phi) / phi (about 863 rad/s at 15 V)."""
    return (volt - MM * RA / PHI) / PHI


def euler_to_R(roll, pitch, yaw):
    """[.., 3, 3] float64 R = Rz(yaw) Ry(pitch) Rx(roll), the convention _get_pitch_roll_yaw inverts."""
    cr, sr, cp, sp, cy, sy = (np.cos(roll), np.sin(roll), np.cos(pitch), np.sin(pitch), np.cos(yaw), np.sin(yaw))
    return np.stack([np.stack([cy * cp, cy * sp * sr - sy * cr, cy * sp * cr + sy * sr], -1),
                     np.stack([sy * cp, sy * sp * sr + cy * cr, sy * sp * cr - cy * sr], -1),
                     np.stack([-sp, cp * sr, cp * cr], -1)], -2)


def haar_rotations(rng, n):
    """[n, 3, 3] float64 rotations, uniform (Haar) over SO(3): unit quaternions from four normal draws."""
    q = rng.normal(size=(n, 4))
    w, x, y, z = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                     np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                     np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)


def _unit(rng, n):
    u = rng.normal(size=(n, 3))
    return u / np.linalg.norm(u, axis=1, keepdims=True)


def _rows(n, R=None):
    """n float64 state rows at rest at the origin (R = I unless given)."""
    s = np.zeros((n, 22))
    s[:, 13:22] = np.eye(3).reshape(9) if R is None else np.asarray(R).reshape(n, 9)
    return s


def envelope_batch(seed=0, nt=50):
    """Envelope(state [n, 22] float32, ct [n] int32, act [n, 4] float32, family [n] str) over FAMILIES.

    The attitude families (grid, inverted, gimbal) start at rest with equal rotor speeds and equal voltages, cycling
    through three rotor settings: at rest with the zero-thrust voltage (the attitude is kept to the bit), spinning up at
    8 V, and at the 15 V equilibrium.  The gimbal family holds exact gimbal-lock matrices (pitch +-pi/2) with R[0], R[3],
    R[7] and R[8] set to +0.0 or -0.0 in all sixteen patterns.  Counters: ct is drawn from [0, nt - 3] except in the
    counters family, which takes 0, nt - 2 and nt - 1 (the step that reads the last target row and the one that ends
    the episode by time)."""
    rng = np.random.RandomState(seed)
    v0 = float(zero_thrust_voltage())
    rotor_settings = ((0.0, v0), (300.0, 8.0), (hover_speed(), MAX_V))
    states, acts, fams = [], [], []

    def add(name, s, a):
        states.append(s)
        acts.append(np.asarray(a, np.float64).reshape(-1, 4))
        fams.extend([name] * s.shape[0])

    def at_rest(name, R):
        s = _rows(R.shape[0], R)
        k = np.arange(R.shape[0]) % len(rotor_settings)
        w = np.array([rotor_settings[i][0] for i in k])
        s[:, 9:13] = w[:, None]
        add(name, s, np.repeat(np.array([rotor_settings[i][1] for i in k])[:, None], 4, axis=1))

    # ---- attitudes: the grid, the three half turns, gimbal lock
    g = np.array(GRID_ANGLES)
    roll, pitch, yaw = [a.reshape(-1) for a in np.meshgrid(g, g, g, indexing="ij")]
    at_rest("grid", euler_to_R(roll, pitch, yaw))
    inv = np.stack([np.diag(d) for d in ((1.0, -1.0, -1.0), (-1.0, 1.0, -1.0), (-1.0, -1.0, 1.0))])
    at_rest("inverted", np.repeat(inv, len(rotor_settings), axis=0))
    gl = []
    for sp in (1.0, -1.0):
        for psi in (0.0, math.pi / 3, -2 * math.pi / 3, math.pi):
            R = euler_to_R(0.0, sp * math.pi / 2, psi)
            R[2, 0] = -sp
            for bits in range(16):
                Rz = R.copy()
                for j, (r, c) in enumerate(((0, 0), (1, 0), (2, 1), (2, 2))):
                    Rz[r, c] = -0.0 if (bits >> j) & 1 else 0.0
                gl.append(Rz)
    at_rest("gimbal", np.repeat(np.stack(gl), len(rotor_settings), axis=0))

    def flying(name, R, v=None, w=None, p=None, rotors=None, act=None):
        n = R.shape[0]
        s = _rows(n, R)
        s[:, 0:3] = 0.0 if p is None else p
        s[:, 3:6] = rng.uniform(-2.0, 2.0, (n, 3)) if v is None else v
        s[:, 6:9] = rng.uniform(-5.0, 5.0, (n, 3)) if w is None else w
        s[:, 9:13] = rng.uniform(0.0, 1000.0, (n, 4)) if rotors is None else rotors
        add(name, s, rng.uniform(MIN_V, MAX_V, (n, 4)) if act is None else act)

    # ---- random attitudes, and drifted copies R (I + E): not orthogonal, det != 1
    H = haar_rotations(rng, 256)
    flying("haar", H)
    E = rng.normal(size=(256, 3, 3))
    E *= (10.0 ** rng.uniform(-5.0, -2.0, 256) / np.linalg.norm(E, axis=(1, 2)))[:, None, None]
    flying("drifted", H @ (np.eye(3) + E))

    # ---- rates up to 900 rad/s (fail.w = 1000), along the body axes and along random axes
    axes = np.repeat(np.concatenate([np.eye(3), -np.eye(3)]), 16, axis=0)
    flying("rates_body", haar_rotations(rng, axes.shape[0]),
           w=axes * (10.0 ** rng.uniform(-2.0, math.log10(900.0), axes.shape[0]))[:, None])
    flying("rates_random", haar_rotations(rng, 160), w=_unit(rng, 160) * (10.0 ** rng.uniform(-2.0, math.log10(900.0),
                                                                                               160))[:, None])
    # ---- speeds up to 95 m/s (fail.velocity = 100) and positions up to 990 m (fail.range = 1000)
    flying("velocity", haar_rotations(rng, 128), v=_unit(rng, 128) * rng.uniform(0.0, 95.0, 128)[:, None])
    flying("position", haar_rotations(rng, 128), p=_unit(rng, 128) * rng.uniform(0.0, 990.0, 128)[:, None])
    # altitude: far above and below the hover target, past the -20 clamp of the hover reward (|p_z| > 20.5) and, for
    # the floor tasks, under the floor (p_z < -5)
    pz = np.concatenate([rng.uniform(20.5, 900.0, 24), -rng.uniform(20.5, 900.0, 24), rng.uniform(-20.5, 20.5, 16)])
    p = np.zeros((pz.size, 3))
    p[:, 2] = pz
    flying("altitude", haar_rotations(rng, pz.size), p=p)
    # ---- rotors from rest to well above the 15 V equilibrium, also at voltages that do not sustain them (me < 0)
    flying("rotors", haar_rotations(rng, 128), rotors=rng.uniform(0.0, 2.5 * hover_speed(), (128, 4)))
    # actions below min_voltage, negative, above max_voltage and exactly at both bounds (as float32)
    choices = np.array([np.float32(MIN_V), np.float32(MAX_V), 0.0, -3.0, 0.05, 15.5, 100.0, -0.0])
    flying("actions", haar_rotations(rng, 128), act=np.where(rng.random_sample((128, 4)) < 0.75,
                                                             choices[rng.randint(0, choices.size, (128, 4))],
                                                             rng.uniform(MIN_V, MAX_V, (128, 4))))
    # ---- ct at 0, nt - 2 and nt - 1, and the control: reset states (R = I, |v| <= 2, |w| <= 5)
    flying("counters", np.repeat(np.eye(3)[None], 66, axis=0))
    flying("control", np.repeat(np.eye(3)[None], 256, axis=0), rotors=np.zeros((256, 4)))

    state = np.concatenate(states).astype(np.float32)
    family = np.array(fams)
    ct = rng.randint(0, max(nt - 2, 1), family.size).astype(np.int32)
    cnt = family == "counters"
    ct[cnt] = np.resize(np.array([0, nt - 2, nt - 1], np.int32), int(cnt.sum()))
    return Envelope(state=state, ct=ct, act=np.concatenate(acts).astype(np.float32), family=family)


def observe_f64(state, task):
    """[n, 16] float64 observation of float32 states [n, 22] (the target columns of velocity_control are left out):
    body velocity and position R^-1 v, R^-1 p and the IMU R^-1 (0, 0, -9.8) with R^-1 = np.linalg.inv(R) in float64;
    gyro = w; pitch, roll, yaw by np.arctan2 of the float32 entries in the reference's argument order; z + z_offset."""
    s = np.asarray(state, dtype=np.float32).astype(np.float64)
    R = s[:, 13:22].reshape(-1, 3, 3)
    Ri = np.linalg.inv(R)
    o = np.empty((s.shape[0], 16))
    o[:, 0:3] = np.einsum("nij,nj->ni", Ri, s[:, 3:6])
    o[:, 3:6] = np.einsum("nij,nj->ni", Ri, s[:, 0:3])
    o[:, 6:9] = Ri[:, :, 2] * np.float64(GRAVITY)
    o[:, 9:12] = s[:, 6:9]
    for k, (y, x) in enumerate(atan2_args(s)):
        o[:, 12 + k] = np.arctan2(y, x)
    o[:, 15] = s[:, 2] + (0.0 if task == "velocity_control" else 5.0)
    return o


def atan2_args(state):
    """((y, x) of pitch, (y, x) of roll, (y, x) of yaw), float64 [n] each: the arguments of the three np.arctan2 calls
    of _get_pitch_roll_yaw (quadrotorsim.py:111-120) for float32 states [n, 22]."""
    s = np.asarray(state, dtype=np.float32).astype(np.float64)
    R = s[:, 13:22].reshape(-1, 3, 3)
    return ((-R[:, 2, 0], np.sqrt(R[:, 2, 1] ** 2 + R[:, 2, 2] ** 2)), (R[:, 2, 1], R[:, 2, 2]), (R[:, 1, 0], R[:, 0, 0]))


def collides_literal(map_matrix, x_off, y_off, old, new, z_off=5.0):
    """Quadrotor._check_collision (env.py:248-260) as the reference evaluates it.  old / new: the simulator's float32
    global positions (x, y, z) before and after the step; map_matrix: the map with its start cell cleared; x_off,
    y_off: the start cell (numpy int64 from np.where, so x and y are float64 sums); z_off: the python float 5.0, so z is
    a float32 sum."""
    xo, yo = np.float64(np.float32(old[0])) + np.int64(x_off), np.float64(np.float32(old[1])) + np.int64(y_off)
    xn, yn = np.float64(np.float32(new[0])) + np.int64(x_off), np.float64(np.float32(new[1])) + np.int64(y_off)
    zo, zn = np.float32(old[2]) + np.float32(z_off), np.float32(new[2]) + np.float32(z_off)
    x_min, x_max = int(math.floor(min(xo, xn))), int(math.ceil(max(xo, xn)))
    y_min, y_max = int(math.floor(min(yo, yn))), int(math.ceil(max(yo, yn)))
    z_min, z_max = int(math.floor(min(zo, zn))), int(math.ceil(max(zo, zn)))
    taken_pos = np.asarray(map_matrix)[y_min:y_max + 1, x_min:x_max + 1]
    return bool(z_min < np.any(taken_pos) or z_max < np.any(taken_pos))
