"""TEST INFRASTRUCTURE -- ctypes front end of oracle/quad_oracle.c (CPU restatement of the quadrotor path).

Follows metagym/quadrotor/quadrotorsim.py:50-109 (_parse_cfg) for turning a simulator config into numbers, and
exposes ``sim_step`` (quadrotorsim.py:295-304) and ``env_step`` (env.py:127-165) in three precisions:
``f32`` (never-reset simulator), ``mix`` (after reset(): float64 velocity vectors) and ``f64`` (arbiter).
"""
import copy
import ctypes
import json

import numpy as np

from . import build as _build
from . import philox

TASKS = {"no_collision": 0, "hovering_control": 1, "velocity_control": 2}

# Default physical parameters: the values of the reference's metagym/quadrotor/config.json:1-59.
DEFAULT_PARAMS = dict(
    precision=0.001, quality=0.5,
    inertia=dict(xx=0.0135, xy=0.0, xz=0.0, yy=0.0135, yz=0.0, zz=0.024),
    drag=dict(m_xx=0.074, m_yy=0.074, m_zz=0.0506, f_xx=0.12, f_yy=0.12, f_zz=0.10),
    gravity_center=dict(x=0.0, y=0.0, z=0.0),
    thrust=dict(CT=["1.538e-5", "-2.5e-4", "0.0"], Mm="0.010", Jm="2.573e-4", RA="0.2010",
                phi="0.017242179827506"),
    propeller=[dict(x=0.18, y=0.18, z=0.0), dict(x=-0.18, y=0.18, z=0.0),
               dict(x=-0.18, y=-0.18, z=0.0), dict(x=0.18, y=-0.18, z=0.0)],
    fail=dict(velocity=100.0, w=1000.0, range=1000.0),
    electric=dict(min_voltage=0.10, max_voltage=15.0),
    init_velocity=dict(x=0, y=0, z=0, noisy=2.0),
    init_angular_velocity=dict(x=0, y=0, z=0, noisy=5.0),
)


class _Cfg(ctypes.Structure):
    _fields_ = [("h", ctypes.c_double), ("m", ctypes.c_double), ("Iinv", ctypes.c_double * 9),
                ("Dm", ctypes.c_double * 3), ("Df", ctypes.c_double * 3), ("cg", ctypes.c_double * 3),
                ("ct0", ctypes.c_double), ("ct1", ctypes.c_double), ("ct2", ctypes.c_double),
                ("mm", ctypes.c_double), ("jm", ctypes.c_double), ("phi", ctypes.c_double), ("ra", ctypes.c_double),
                ("fail_v", ctypes.c_double), ("fail_r", ctypes.c_double), ("fail_w", ctypes.c_double),
                ("prop", ctypes.c_double * 12), ("lm", ctypes.c_double * 4),
                ("vmin", ctypes.c_double), ("vmax", ctypes.c_double)]


def make_cfg(params=None):
    p = DEFAULT_PARAMS if params is None else params
    if isinstance(p, str):
        with open(p) as f:
            p = json.load(f)
    c = _Cfg()
    c.h = float(p["precision"])
    c.m = float(p["quality"])
    ine = p["inertia"]
    I = np.array([[ine["xx"], ine["xy"], ine["xz"]], [ine["xy"], ine["yy"], ine["yz"]],
                  [ine["xz"], ine["yz"], ine["zz"]]], dtype=np.float64).astype(np.float32)
    c.Iinv[:] = [float(x) for x in np.linalg.inv(I).reshape(-1)]
    d = p["drag"]
    c.Dm[:] = [float(np.float32(d[k])) for k in ("m_xx", "m_yy", "m_zz")]
    c.Df[:] = [float(np.float32(d[k])) for k in ("f_xx", "f_yy", "f_zz")]
    c.cg[:] = [float(np.float32(p["gravity_center"][k])) for k in "xyz"]
    th = p["thrust"]
    c.ct0, c.ct1, c.ct2 = (float(x) for x in th["CT"])
    c.mm, c.jm, c.phi, c.ra = float(th["Mm"]), float(th["Jm"]), float(th["phi"]), float(th["RA"])
    c.fail_v, c.fail_r, c.fail_w = (float(p["fail"][k]) for k in ("velocity", "range", "w"))
    prop = np.array([[q["x"], q["y"], q["z"]] for q in p["propeller"]], dtype=np.float64).astype(np.float32)
    c.prop[:] = [float(x) for x in prop.reshape(-1)]
    c.lm[:] = [float(np.linalg.norm(prop[i])) for i in range(4)]
    c.vmin = float(p["electric"]["min_voltage"])
    c.vmax = float(p["electric"]["max_voltage"])
    return c


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(_build.build())
    return _lib


def _ptr(a, ct):
    return a.ctypes.data_as(ctypes.POINTER(ct)) if a is not None else None


def zero_state(n):
    """[n,22] float64 carrier of p3 v3 om3 w4 R9 in the reference's _zero_state (quadrotorsim.py:20-28)."""
    s = np.zeros((n, 22), dtype=np.float64)
    s[:, 13] = s[:, 17] = s[:, 21] = 1.0
    return s


def sim_step(cfg, state, act, substeps, mode="mix"):
    n = state.shape[0]
    assert state.dtype == np.float64 and state.flags.c_contiguous and state.shape == (n, 22)
    act = np.ascontiguousarray(act, dtype=np.float32).reshape(n, 4)
    power = np.zeros(n, dtype=np.float64)
    fail = np.zeros(n, dtype=np.int32)
    fn = getattr(lib(), "qo_%s_sim_step" % mode)
    fn(ctypes.byref(cfg), ctypes.c_int(n), _ptr(state, ctypes.c_double), _ptr(act, ctypes.c_float),
       ctypes.c_int(substeps), _ptr(power, ctypes.c_double), _ptr(fail, ctypes.c_int))
    return power, fail


def env_step(cfg, state, ct, act, task, dt, nt, healthy=1.0, targets=None, env2task=None, mode="mix"):
    """One Quadrotor.step for n envs.  state [n,22] f64 and ct [n] i32 are updated in place."""
    n = state.shape[0]
    task_id = TASKS[task] if isinstance(task, str) else int(task)
    assert state.dtype == np.float64 and state.flags.c_contiguous and state.shape == (n, 22)
    assert ct.dtype == np.int32 and ct.shape == (n,)
    act = np.ascontiguousarray(act, dtype=np.float32).reshape(n, 4)
    obs = np.zeros((n, 19 if task_id == 2 else 16), dtype=np.float32)
    rew = np.zeros(n, dtype=np.float64)
    done = np.zeros(n, dtype=np.uint8)
    fail = np.zeros(n, dtype=np.int32)
    power = np.zeros(n, dtype=np.float64)
    if task_id == 2:
        targets = np.ascontiguousarray(targets, dtype=np.float32)
        assert targets.ndim == 3 and targets.shape[1] == nt and targets.shape[2] == 3
        env2task = np.ascontiguousarray(env2task, dtype=np.int32)
    fn = getattr(lib(), "qo_%s_env_step" % mode)
    fn(ctypes.byref(cfg), ctypes.c_int(n), _ptr(state, ctypes.c_double), _ptr(ct, ctypes.c_int),
       _ptr(act, ctypes.c_float), ctypes.c_int(task_id), ctypes.c_double(dt), ctypes.c_int(nt),
       ctypes.c_double(healthy), _ptr(targets, ctypes.c_float) if task_id == 2 else None,
       _ptr(env2task, ctypes.c_int) if task_id == 2 else None, _ptr(obs, ctypes.c_float),
       _ptr(rew, ctypes.c_double), _ptr(done, ctypes.c_ubyte), _ptr(fail, ctypes.c_int), _ptr(power, ctypes.c_double))
    return obs, rew, done, fail, power


def reset_state(cfg_params, noise):
    """State after QuadrotorSim.reset() (quadrotorsim.py:239-258) given the 12 uniform draws it consumes.

    noise [n,12] float64 = the np.random.random draws in reference order: sign_v(3), mag_v(3), sign_w(3), mag_w(3).
    """
    p = DEFAULT_PARAMS if cfg_params is None else cfg_params
    noise = np.asarray(noise, dtype=np.float64).reshape(-1, 12)
    s = zero_state(noise.shape[0])
    iv, iw = p["init_velocity"], p["init_angular_velocity"]
    sv = (noise[:, 0:3] > 0.5).astype(int) * 2 - 1.0
    sw = (noise[:, 6:9] > 0.5).astype(int) * 2 - 1.0
    base_v = np.array([iv["x"], iv["y"], iv["z"]], dtype=np.float32)
    base_w = np.array([iw["x"], iw["y"], iw["z"]], dtype=np.float32)
    s[:, 3:6] = base_v + (float(iv["noisy"]) * noise[:, 3:6]) * sv
    s[:, 6:9] = base_w + (float(iw["noisy"]) * noise[:, 9:12]) * sw
    return s


def general_params():
    """A config that leaves the engine's specialised kernels (SIMPLE = false): off-diagonal inertia, a
    centre-of-gravity offset, CT[2] != 0 and rotors out of the body plane."""
    p = copy.deepcopy(DEFAULT_PARAMS)
    p["inertia"].update(xy=0.001, xz=-0.0005, yz=0.0007)
    p["gravity_center"] = {"x": 0.01, "y": -0.02, "z": 0.015}
    p["thrust"]["CT"][2] = "1.0e-3"
    for i, z in enumerate([0.02, -0.01, 0.03, 0.0]):
        p["propeller"][i]["z"] = z
    return p


class StepResult(object):
    """What OracleBatch.step returns: obs / rew / done / fail as env_step computes them, except that rows of envs an
    auto-reset replaced hold the reset observation and `final_obs` holds their terminal one (NaN elsewhere);
    `pre_state` / `end_state` are the states before the step and after the integrator (before any reset)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class OracleBatch(object):
    """The engine's batch semantics around env_step(mode="mix"): per-env step counters `ct`, episode counters `ep`,
    and resets whose twelve draws come from the engine's counter-based generator (oracle/philox.py), keyed by
    `rng_seed`, the global env index env_index_base + e and `ep`.

    `subset` (local env indices) makes the batch follow only those envs of an n-env batch; step() still takes the
    actions of all n envs.  Rules for `ep`: it starts at 0; reset() without noise and every auto-reset increment it and
    then draw; reset(noise=...) leaves it alone.  A reset state follows the engine's typing: float32 init values and
    noise scales, one float64 expression, one rounding to float32.
    """

    def __init__(self, n, task, dt, nt, params=None, healthy=1.0, targets=None, env2task=None, map_matrix=None,
                 rng_seed=0, env_index_base=0, auto_reset=False, subset=None):
        self.params = DEFAULT_PARAMS if params is None else params
        self.cfg = make_cfg(self.params)
        self.n, self.task, self.dt, self.nt, self.healthy = int(n), task, float(dt), int(nt), float(healthy)
        self.idx = np.arange(self.n, dtype=np.int64) if subset is None else np.asarray(subset, dtype=np.int64)
        self.genv = int(env_index_base) + self.idx
        self.rng_seed, self.auto_reset = int(rng_seed), bool(auto_reset)
        self.targets = None if targets is None else np.ascontiguousarray(targets, dtype=np.float32)
        self.env2task = None if env2task is None else np.ascontiguousarray(np.asarray(env2task, np.int32)[self.idx])
        self.map_matrix = map_matrix
        self.z_off = 0.0 if task == "velocity_control" else 5.0
        self.obs_dim = 19 if task == "velocity_control" else 16
        m = self.idx.size
        self.state, self.ct, self.ep = zero_state(m), np.zeros(m, np.int32), np.zeros(m, np.int64)
        iv, iw = self.params["init_velocity"], self.params["init_angular_velocity"]
        self._base = [np.array([iv[k] for k in "xyz"], np.float32), np.array([iw[k] for k in "xyz"], np.float32)]
        self._scale = [np.float32(iv["noisy"]), np.float32(iw["noisy"])]

    def reset_rows(self, u):
        """[k,22] reset states for the draws u [k,12] (reset_env in quad.cu)."""
        u = np.asarray(u, dtype=np.float64).reshape(-1, 12)
        s = zero_state(u.shape[0])
        for blk, (sign, mag) in enumerate([(0, 3), (6, 9)]):
            sg = np.where(u[:, sign:sign + 3] > 0.5, 1.0, -1.0)
            x = np.float64(self._base[blk]) + (np.float64(self._scale[blk]) * u[:, mag:mag + 3]) * sg
            s[:, 3 + 3 * blk:6 + 3 * blk] = x.astype(np.float32)
        return s

    def reset_obs(self, rows):
        """Observation of the freshly reset envs `rows` (bool mask or indices): R = I, p = 0."""
        s = self.state[rows]
        o = np.zeros((s.shape[0], self.obs_dim), np.float32)
        o[:, 0:3] = s[:, 3:6]
        o[:, 6:8] = np.float32(0.0) * np.float32(-9.8)
        o[:, 8] = np.float32(-9.8)
        o[:, 9:12] = s[:, 6:9]
        o[:, 12] = -0.0
        o[:, 15] = np.float32(self.z_off)
        if self.task == "velocity_control":
            t = np.minimum(self.ct[rows], self.nt - 1)
            o[:, 16:19] = self.targets[self.env2task[rows], t]
        return o

    def _redraw(self, rows):
        self.ep[rows] += 1
        self.state[rows] = self.reset_rows(philox.quad_reset_draws(self.rng_seed, self.genv[rows], self.ep[rows]))

    def reset(self, mask=None, noise=None):
        """Quadrotor.reset of the envs in `mask` ([n] over the whole batch; None = all); `noise` [n,12] replays draws.
        ct is left alone, as in the reference.  Returns the reset observation rows (NaN for envs left alone)."""
        rows = np.ones(self.idx.size, bool) if mask is None else np.asarray(mask, bool)[self.idx]
        if noise is None:
            self._redraw(rows)
        else:
            self.state[rows] = self.reset_rows(np.asarray(noise, np.float64).reshape(self.n, 12)[self.idx][rows])
        o = np.full((self.idx.size, self.obs_dim), np.nan, np.float32)
        o[rows] = self.reset_obs(rows)
        return o

    def step(self, act):
        """One engine step of the followed envs; act [n,4] for the whole batch."""
        act = np.ascontiguousarray(np.asarray(act, np.float32).reshape(self.n, 4)[self.idx])
        pre = self.state.copy()
        set_map(self.map_matrix)
        obs, rew, done, fail, _ = env_step(self.cfg, self.state, self.ct, act, self.task, self.dt, self.nt,
                                           self.healthy, self.targets, self.env2task, mode="mix")
        done = done.astype(bool)
        end = self.state.copy()
        final = np.full_like(obs, np.nan)
        if self.auto_reset and done.any():
            final[done] = obs[done]
            self._redraw(done)
            obs[done] = self.reset_obs(done)
        return StepResult(obs=obs, rew=rew, done=done, fail=fail, final_obs=final, pre_state=pre, end_state=end)


def rk4_step(cfg, state, act, dt, rk4_steps=1, mode="f64"):
    """Classical RK4 on the continuous-time model (NOT a reference mode; parity unpinned).  state [n,22] f64 in place."""
    n = state.shape[0]
    assert state.dtype == np.float64 and state.flags.c_contiguous and state.shape == (n, 22)
    act = np.ascontiguousarray(act, dtype=np.float32).reshape(n, 4)
    fn = getattr(lib(), "qo_%s_rk4_step" % mode)
    fn(ctypes.byref(cfg), ctypes.c_int(n), _ptr(state, ctypes.c_double), _ptr(act, ctypes.c_float),
       ctypes.c_double(dt), ctypes.c_int(rk4_steps))


_map_keepalive = None


def set_map(map_matrix):
    """Obstacle map for the following env_step calls (None = flat).  map_matrix as Quadrotor.load_map returns it (one
    cell == -1 marks the start); returns (x_offset, y_offset)."""
    global _map_keepalive
    if map_matrix is None:
        lib().qo_set_map(None, 0, 0, 0, 0)
        _map_keepalive = None
        return 0, 0
    m = np.array(map_matrix, dtype=np.int64)
    ys, xs = np.where(m == -1)
    assert len(ys) == 1
    m[ys[0], xs[0]] = 0
    sat = np.zeros((m.shape[0] + 1, m.shape[1] + 1), dtype=np.int32)
    sat[1:, 1:] = np.cumsum(np.cumsum((m != 0).astype(np.int32), axis=0), axis=1)
    sat = np.ascontiguousarray(sat)
    _map_keepalive = sat
    lib().qo_set_map(_ptr(sat, ctypes.c_int), ctypes.c_int(m.shape[0]), ctypes.c_int(m.shape[1]),
                     ctypes.c_int(int(xs[0])), ctypes.c_int(int(ys[0])))
    return int(xs[0]), int(ys[0])
