"""CPU: pin the references of the flight-envelope tests (tests/quad_envelope.py) before the GPU is judged by them.

observe_f64 against the oracle's observation, on every envelope state; collides_literal against the oracle's map
collision, on every small window of a 7 x 9 map; and the invariants of the state generator.
"""
import math

import numpy as np
import pytest

import quad_envelope as qe
from oracle import quad_oracle as qo
from util import OBS_GROUPS, group_rel_err_rows

EPS32 = 2.0 ** -24


def _oracle_obs(states, task, dt, mode, nt=50):
    """(obs, post-step state) of one oracle env.step; velocity_control gets an all-zero target table."""
    cfg = qo.make_cfg()
    st = np.ascontiguousarray(states, dtype=np.float64)
    n = st.shape[0]
    kw = {}
    if task == "velocity_control":
        kw = dict(targets=np.zeros((1, nt, 3), np.float32), env2task=np.zeros(n, np.int32))
    qo.set_map(None)
    obs = qo.env_step(cfg, st, np.zeros(n, np.int32), np.full((n, 4), 5.0, np.float32), task, dt, nt, mode=mode,
                      **kw)[0]
    return obs[:, :16].astype(np.float64), st


def _angle_err(a, ref):
    """|a - ref| wrapped into [0, pi]: angles on either side of the +-pi cut are close."""
    d = np.abs(np.asarray(a, np.float64) - ref) % (2 * math.pi)
    return np.minimum(d, 2 * math.pi - d)


def _check_obs(obs, ref, state):
    """The oracle's float32 observation against the float64 one: 8 float32 roundings of each group's scale for the
    vectors (their products with R^-1), 2 roundings of the angle for pitch / roll / yaw, and at the branch cuts of
    np.arctan2 (y = +-0) the very value np.arctan2 returns, sign of zero included."""
    vec = [g for g in OBS_GROUPS if g[0] != 12]
    assert (group_rel_err_rows(obs, ref, vec) <= 8 * EPS32).all()
    err = _angle_err(obs[:, 12:15], ref[:, 12:15])
    assert (err <= 2 * EPS32 * np.maximum(np.abs(ref[:, 12:15]), 1.0) + 1e-12).all(), float(err.max())
    for k, (y, x) in enumerate(qe.atan2_args(state)):
        cut = y == 0.0
        want = np.arctan2(y[cut], x[cut]).astype(np.float32)
        got = obs[cut, 12 + k].astype(np.float32)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), k


@pytest.mark.parametrize("task", ["no_collision", "hovering_control", "velocity_control"])
def test_observe_f64_vs_oracle_without_substeps(task):
    """dt below the 1 ms substep: the oracle's step integrates nothing, and its observation is that of the given state."""
    env = qe.envelope_batch(0)
    obs, st = _oracle_obs(env.state, task, 0.0005, "mix")
    assert np.array_equal(st.astype(np.float32), env.state)
    _check_obs(obs, qe.observe_f64(env.state, task), env.state)


def test_observe_f64_vs_oracle_after_a_step():
    """The all-float32 oracle's observation of the state its own step returns (failed envs stop where they failed)."""
    env = qe.envelope_batch(1)
    obs, st = _oracle_obs(env.state, "hovering_control", 0.01, "f32")
    s32 = st.astype(np.float32)
    ok = np.isfinite(s32).all(axis=1) & (np.abs(s32) < 1e30).all(axis=1)
    assert ok.mean() > 0.95
    _check_obs(obs[ok], qe.observe_f64(s32[ok], "hovering_control"), s32[ok])


def test_observe_f64_at_the_cuts():
    """The values the angle tests rely on: np.arctan2 at (+-0, -0) is +-pi and at (+-0, +0) it is +-0."""
    s = np.zeros((6, 22), np.float32)
    s[:4, 13:22] = [0, 0, 1, 0, 1, 0, -1, 0, 0]                      # gimbal lock: yaw = atan2(R[3], R[0]) of zeros
    s[1, 13] = s[2, 13] = s[2, 16] = s[3, 16] = -0.0
    s[4:, 13:22] = np.diag([-1.0, -1.0, 1.0]).reshape(9)            # yaw = atan2(+-0, -1), pitch = atan2(-0, 1)
    s[5, 16] = -0.0
    o = qe.observe_f64(s, "hovering_control")
    yaw = o[:, 14]
    assert yaw[0] == 0 and not np.signbit(yaw[0]) and yaw[1] == math.pi and yaw[2] == -math.pi
    assert yaw[3] == 0 and np.signbit(yaw[3]) and yaw[4] == math.pi and yaw[5] == -math.pi
    assert (o[:4, 12] == math.pi / 2).all() and np.signbit(o[4:, 12]).all() and (o[4:, 12] == 0).all()


# --------------------------------------------------------------------------------------------------------------------
# collides_literal against the oracle's collision rule
# --------------------------------------------------------------------------------------------------------------------
def _small_map(start):
    rng = np.random.RandomState(7)
    m = (rng.random_sample((7, 9)) < 0.35).astype(np.int64) * rng.randint(1, 9, (7, 9))
    m[0, 8] = m[6, 0] = 0          # free and taken cells on every edge
    m[6, 8] = m[0, 3] = 2
    m[start] = -1
    return m


@pytest.mark.parametrize("start", [(0, 0), (3, 4)], ids=["corner", "interior"])
def test_collides_literal_vs_oracle_windows(start):
    """Every window swept from map cell (sx, sy) to (sx + Lx, sy + Ly), sx, sy in [-12, 12), Lx, Ly in [0, 4], and the
    same with both ends half a cell further (floor / ceil): windows that start negative (the slice wraps once), end past
    the far edge (clamped), or lie wholly outside.  At z = 0.5 the collision rule is `np.any(window)` itself."""
    m = _small_map(start)
    ys, xs = start
    free = m.copy()
    free[ys, xs] = 0
    qo.set_map(m)
    try:
        n_any = n = 0
        for sx in range(-12, 12):
            for lx in range(5):
                for sy in range(-12, 12):
                    for ly in range(5):
                        for d in (0.0, 0.5):
                            old = (sx + d - xs, sy + d - ys, 0.5 - 5.0)
                            new = (sx + lx + d - xs, sy + ly + d - ys, 0.5 - 5.0)
                            lit = qe.collides_literal(free, xs, ys, old, new)
                            ora = qo.map_any_obstacle(sx + d, sy + d, sx + lx + d, sy + ly + d)
                            assert lit == ora, (sx, lx, sy, ly, d)
                            n_any += lit
                            n += 1
        assert 0.2 < n_any / n < 0.8
    finally:
        qo.set_map(None)


def _z_values():
    """Barometer heights z = p_z + 5 (float32) at the integers 0 and 1 and one float32 step of p_z around them."""
    out = []
    for pz in (-5.0, -4.0):
        p = np.float32(pz)
        out += [np.nextafter(p, np.float32(-np.inf)), p, np.nextafter(p, np.float32(np.inf))]
    return out


@pytest.mark.parametrize("start", [(0, 0), (3, 4)], ids=["corner", "interior"])
def test_collides_literal_vs_oracle_env_step(start):
    """Through the oracle's env_step with no substep (the position does not move, so only the collision decides done)
    at every cell and half cell of a band around the map, and at z on and one float32 step around 0 and 1."""
    m = _small_map(start)
    ys, xs = start
    free = m.copy()
    free[ys, xs] = 0
    coords = np.arange(-3.0, 12.0, 0.5)
    X, Y, Z = [a.reshape(-1) for a in np.meshgrid(coords, coords, np.array(_z_values(), np.float64), indexing="ij")]
    n = X.size
    st = qo.zero_state(n)
    st[:, 0] = (X - xs).astype(np.float32)
    st[:, 1] = (Y - ys).astype(np.float32)
    st[:, 2] = Z
    s32 = st.astype(np.float32)
    qo.set_map(m)
    try:
        ct = np.zeros(n, np.int32)
        _, _, done, fail, _ = qo.env_step(qo.make_cfg(), st, ct, np.full((n, 4), 5.0, np.float32), "no_collision",
                                          0.0005, 1000, mode="mix")
    finally:
        qo.set_map(None)
    assert not fail.any() and np.array_equal(st.astype(np.float32), s32)
    lit = np.array([qe.collides_literal(free, xs, ys, s32[i, :3], s32[i, :3]) for i in range(n)])
    assert np.array_equal(done.astype(bool), lit)
    assert 0.2 < lit.mean() < 0.8


# --------------------------------------------------------------------------------------------------------------------
# the generator
# --------------------------------------------------------------------------------------------------------------------
def test_generator_invariants():
    a, b, c = qe.envelope_batch(0, nt=40), qe.envelope_batch(0, nt=40), qe.envelope_batch(1, nt=40)
    n = a.state.shape[0]
    assert a.state.shape == (n, 22) and a.state.dtype == np.float32 and a.act.shape == (n, 4)
    assert a.ct.shape == (n,) and a.ct.dtype == np.int32 and a.family.shape == (n,)
    assert np.isfinite(a.state).all() and np.isfinite(a.act).all()
    assert set(a.family) == set(qe.FAMILIES)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert not np.array_equal(a.state, c.state)
    st, fam = a.state.astype(np.float64), a.family
    # inside the failure limits, and reaching towards them
    for lo, lim, reach in ((0, qe.FAIL_R, 900.0), (3, qe.FAIL_V, 80.0), (6, qe.FAIL_W, 700.0)):
        norm = np.linalg.norm(st[:, lo:lo + 3], axis=1)
        assert norm.max() < lim and norm.max() > reach
    assert (st[fam == "altitude", 2] > 20.5).any() and (st[fam == "altitude", 2] < -20.5).any()
    R = st[:, 13:22].reshape(-1, 3, 3)
    # the grid's yaw reaches both sides of the cut; gimbal lock comes in all sixteen signed-zero patterns
    yaw = np.arctan2(R[fam == "grid", 1, 0], R[fam == "grid", 0, 0])
    assert (yaw > 3.14159).any() and (yaw < -3.14159).any()
    g = a.state[fam == "gimbal"][:, [13, 16, 20, 21]]
    assert (g == 0).all() and len({tuple(r) for r in np.signbit(g)}) == 16
    assert set(np.abs(a.state[fam == "gimbal", 19])) == {1.0}
    det = np.linalg.det(R)
    orth = np.abs(np.einsum("nij,nkj->nik", R, R) - np.eye(3)).max(axis=(1, 2))
    assert (np.abs(det[fam == "haar"] - 1) < 1e-6).all() and (orth[fam == "haar"] < 1e-6).all()
    drift = orth[fam == "drifted"]
    assert drift.min() > 1e-6 and drift.max() > 5e-3 and (np.abs(det[fam == "drifted"] - 1) > 1e-7).mean() > 0.9
    # rotors past the 15 V equilibrium, actions outside the voltage range and exactly at its bounds
    assert a.state[fam == "rotors", 9:13].max() > 2 * qe.hover_speed()
    act = a.act[fam == "actions"]
    for v in (np.float32(qe.MIN_V), np.float32(qe.MAX_V)):
        assert (act == v).any()
    assert (act < 0).any() and (act > qe.MAX_V).any() and ((act > 0) & (act < qe.MIN_V)).any()
    assert set(a.ct[fam == "counters"]) == {0, 38, 39} and a.ct.max() == 39
    ctl = st[fam == "control"]
    assert (ctl[:, 13:22] == np.eye(3).reshape(9)).all() and np.abs(ctl[:, 3:6]).max() <= 2
    # the zero-thrust voltage holds a resting rotor at rest in float32
    v0 = qe.zero_thrust_voltage()
    assert np.float32(np.float32(qe.PHI / qe.RA) * v0) == np.float32(qe.MM) and qe.MIN_V < v0 < qe.MAX_V
