"""GPU: one quadrotor step from anywhere in the flight envelope (tests/quad_envelope.py), on every step path.

The parity suite elsewhere starts from reset states or recorded reference episodes, so it only sees a vehicle flying
close to level.  Here the batch holds every attitude (the branch cuts of the observed angles, gimbal lock, upside
down), non-orthogonal rotation matrices, rates up to 900 rad/s, speeds up to 95 m/s, positions up to 990 m, rotors the
voltage does not sustain and actions outside the voltage range, and each step is judged

 * against the CPU oracle, within 4x the oracle's own float32 error against its float64 arbiter for that env;
 * for the observation, against observe_f64 of the GPU's own post-step state: a few float32 roundings, and at the
   branch cuts of atan2 exactly np.arctan2's value, sign of zero included;
 * across the tile, wide, packed, streaming, rollout and host zero-copy paths: the same bits;
 * and, over an obstacle map, the collision against the reference's literal slice of the map, exactly.
"""
import math

import numpy as np
import pytest

import quad_envelope as qe
from test_quadrotor_gpu import _done_flip_is_marginal, _kernel_suffix, _stream_size, get_state, make_env, set_state
from util import OBS_GROUPS, STATE_GROUPS, group_rel_err_rows

pytestmark = pytest.mark.gpu

NT = 50
FLOOR = 1e-5          # the per-step parity bound of the rest of the suite
OWN = 4.0             # x the oracle's own float32-vs-float64 error of the env
# The angular-velocity groups are judged against at least 1 rad/s, the rate one rotor's torque arm adds in a step.
# A balanced vehicle at rest stays at w = 0 exactly in the reference's arithmetic, whose rotor torques th * py cancel
# pairwise (a + a - a - a); the kernel sums them in one chain of fused multiply-adds, whose rounding (< 1 ulp of one
# rotor's torque) leaves |w| ~ 1e-8..1e-7 rad/s after one step -- far below the 1e-5 relative bound at any rate the
# vehicle actually flies, but 1e-5 of the 1e-3 floor the suite's groups use elsewhere.
W_FLOOR = 1.0
STATE_GROUPS_W = [g if g[0] != 6 else (6, 9, W_FLOOR) for g in STATE_GROUPS]
VEC_GROUPS = [(g if g[0] != 9 else (9, 12, W_FLOOR)) for g in OBS_GROUPS if g[0] != 12]
ANGLE_SCALE = [g for g in OBS_GROUPS if g[0] == 12][0][2]
# observe() against observe_f64 of the same state, in float32 roundings of each group's scale, plus the documented
# 7.5e-8 rad of fast_atan2's polynomial for the angles.  Measured on an H100 80GB HBM3 (700 W power limit): at most
# 3.15 roundings for the vector groups and 0.75 for the angles.
OBS_ULPS = 8
ATAN_POLY = 7.5e-8


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def _params(config):
    from oracle import quad_oracle as qo
    return qo.general_params() if config == "general" else None


def _wrap(d):
    """Angle differences wrapped into [0, pi]."""
    d = np.abs(np.asarray(d, np.float64)) % (2 * math.pi)
    return np.minimum(d, 2 * math.pi - d)


def _obs_err_rows(obs, ref_obs, ref_state):
    """Per env: group_rel_err_rows of the vector groups, and for pitch / roll / yaw the wrapped angle difference times
    min(1, |(y, x)|) of the reference's atan2 arguments -- the distance the two angles put between points at that
    radius.  Where the arguments are tiny (gimbal lock: atan2 of two entries that are exactly 0 in the reference's
    arithmetic and 1e-10 in a fused one) the angle carries no information; the rotation matrix is compared as state."""
    err = group_rel_err_rows(obs[:, :16], ref_obs[:, :16], VEC_GROUPS)
    scale = np.maximum(np.abs(ref_obs[:, 12:15]).max(axis=1), ANGLE_SCALE)
    for k, (y, x) in enumerate(qe.atan2_args(ref_state.astype(np.float32))):
        err = np.maximum(err, _wrap(obs[:, 12 + k] - ref_obs[:, 12 + k]) * np.minimum(np.hypot(y, x), 1.0) / scale)
    return err


def _rew_err(a, ref):
    return np.abs(np.asarray(a, np.float64) - ref) / np.maximum(np.abs(ref), 1.0)


def _envelope_env(n, task, dt, config, **kw):
    if task == "velocity_control":
        kw["seed"] = [0, 1, 2]
    return make_env(n, task, dt=dt, nt=NT, simulator_conf=_params(config), **kw)


# --------------------------------------------------------------------------------------------------------------------
# teacher-forced single steps against the oracle
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [0.01, 0.005])
@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task", ["no_collision", "hovering_control", "velocity_control"])
def test_teacher_forced_step_vs_oracle(torch_mod, task, config, dt):
    """Every envelope state, one step with auto_reset=False, against OracleBatch (mode="mix") on the same state and
    action.  Per env, the post-step state, the observation and the reward lie within max(1e-5, 4 x |mix - f64|) of
    the oracle; ct, done, fail codes and the target rows are exact (a done flag may differ only where
    _done_flip_is_marginal allows it)."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    env_b = qe.envelope_batch(seed=11, nt=NT)
    n = env_b.state.shape[0]
    env = _envelope_env(n, task, dt, config)
    vel = task == "velocity_control"
    targets = env.velocity_targets.cpu().numpy() if vel else None
    e2t = env.env2task.cpu().numpy() if vel else None
    set_state(env, env_b.state, env_b.ct)
    obs, rew, done, _ = env.step(torch.as_tensor(env_b.act).cuda())
    obs, rew, done = obs.cpu().numpy().astype(np.float64), rew.cpu().numpy(), done.cpu().numpy().astype(bool)
    fail = env.fail_code.cpu().numpy()
    gs, gct = get_state(env)
    env.close()

    ob = qo.OracleBatch(n, task, dt, NT, params=_params(config), targets=targets, env2task=e2t)
    ob.state[:] = env_b.state
    ob.ct[:] = env_b.ct
    r = ob.step(env_b.act)
    f64 = env_b.state.astype(np.float64)
    o64, r64, _, _, _ = qo.env_step(ob.cfg, f64, env_b.ct.copy(), env_b.act, task, dt, NT, targets=targets,
                                    env2task=e2t, mode="f64")

    flip = (done != r.done) | (fail != r.fail)
    for i in np.nonzero(flip)[0]:
        assert _done_flip_is_marginal(ob, r, i, fail[i]), (i, env_b.family[i], bool(done[i]), int(fail[i]))
    assert flip.sum() <= 3, np.nonzero(flip)[0]
    ok = ~flip
    assert np.array_equal(gct[ok], ob.ct[ok])
    if vel:
        assert np.array_equal(obs[:, 16:], r.obs[:, 16:].astype(np.float64))
    report = {}
    for name, err, own in (
            ("state", group_rel_err_rows(gs, r.end_state, STATE_GROUPS_W),
             group_rel_err_rows(r.end_state, f64, STATE_GROUPS_W)),
            ("obs", _obs_err_rows(obs, r.obs.astype(np.float64), r.end_state),
             _obs_err_rows(r.obs.astype(np.float64), o64.astype(np.float64), f64)),
            ("rew", _rew_err(rew, r.rew), _rew_err(r.rew, r64))):
        tol = np.maximum(FLOOR, OWN * own)
        bad = ok & ~(err <= tol)
        worst = int(np.argmax(np.where(ok, err / tol, 0)))
        report[name] = (float(err[ok].max()), float((err / tol)[ok].max()), str(env_b.family[worst]))
        assert not bad.any(), (name, [(int(i), env_b.family[i], float(err[i]), float(tol[i]))
                                      for i in np.nonzero(bad)[0][:8]])
    print("worst (error, error / bound, family):", report, "done:", int(done.sum()), "fail:", np.bincount(fail))


# --------------------------------------------------------------------------------------------------------------------
# observe() on the GPU's own post-step state
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task", ["hovering_control", "velocity_control"])
def test_observation_of_the_gpu_state(torch_mod, task, config):
    """The observation a step returns against observe_f64 of the state the same step leaves (state_dict()): no
    integration between the two, so the bound is tight -- OBS_ULPS float32 roundings of each group's scale, plus
    ATAN_POLY for the angles.  At the branch cuts (y = +-0) the angle equals np.arctan2's to the bit: +-pi by the sign
    of the zero, and atan2(+-0, +-0) = +-0 or +-pi."""
    torch = torch_mod
    env_b = qe.envelope_batch(seed=12, nt=NT)
    n = env_b.state.shape[0]
    env = _envelope_env(n, task, 0.01, config)
    set_state(env, env_b.state, env_b.ct)
    obs, _, _, _ = env.step(torch.as_tensor(env_b.act).cuda())
    obs = obs.cpu().numpy()
    gs = env.state_dict()["state"].cpu().numpy()
    env.close()
    ref = qe.observe_f64(gs, task)
    worst = {}
    for lo, hi, *_ in [g for g in OBS_GROUPS if g[0] != 12]:
        ulp = np.spacing(np.abs(ref[:, lo:hi]).max(axis=1).astype(np.float32)).astype(np.float64)
        ulp = np.maximum(ulp, np.spacing(np.float32(1e-30)))
        e = (np.abs(obs[:, lo:hi] - ref[:, lo:hi]).max(axis=1) / ulp)
        worst[(lo, hi)] = float(e.max())
        assert (e <= OBS_ULPS).all(), ((lo, hi), float(e.max()), env_b.family[int(np.argmax(e))])
    ang = obs[:, 12:15].astype(np.float64)
    aulp = np.spacing(np.maximum(np.abs(ref[:, 12:15]), 1.0).astype(np.float32)).astype(np.float64)
    e = (_wrap(ang - ref[:, 12:15]) - ATAN_POLY) / aulp
    worst["angles"] = float(e.max())
    assert (e <= OBS_ULPS).all(), (float(e.max()), env_b.family[int(np.argmax(e.max(axis=1)))])
    n_cut = 0
    for k, (y, x) in enumerate(qe.atan2_args(gs)):
        cut = y == 0.0
        n_cut += int(cut.sum())
        want = np.arctan2(y[cut], x[cut]).astype(np.float32)
        got = obs[cut, 12 + k]
        bad = got.view(np.int32) != want.view(np.int32)
        assert not bad.any(), (k, list(zip(got[bad][:4], want[bad][:4], y[cut][bad][:4], x[cut][bad][:4])))
    assert n_cut >= 100 or config == "general"      # its gravity torque turns every attitude off the cut
    print("worst error in float32 roundings of the group scale:", worst, "angles on a cut:", n_cut)


# --------------------------------------------------------------------------------------------------------------------
# every path gives the same bits
# --------------------------------------------------------------------------------------------------------------------
def _pinned(torch, shape, dtype):
    return torch.zeros(shape, dtype=dtype).pin_memory()


def _run_path(torch, monkeypatch, path, state, ct, act, task, config, **kw):
    """(kernel name, obs, rew, done, fail or None, post-step state, ct) of one step along `path`."""
    from metagym_b200 import _lib
    env_vars = {"tile": {"MGB_STREAM_KERNEL": "0", "MGB_WIDE_KERNEL": "0"}, "wide": {"MGB_WIDE_KERNEL": "1"},
                "packed": {"MGB_PACKED": "1"}}.get(path, {})
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    n = state.shape[0]
    env = _envelope_env(n, task, 0.01, config, **kw)
    for k in env_vars:
        monkeypatch.delenv(k)
    name = env.step_kernel_name()
    set_state(env, state, ct)
    fail = None
    if path == "rollout":
        out = env.rollout(1, actions=torch.as_tensor(act[None]).cuda())
        obs, rew, done = out["obs"][0], out["rew"][0], out["done"][0]
    elif path == "host_zerocopy":
        h = [_pinned(torch, s, d) for s, d in (((n, 4), torch.float32), ((n, env.obs_dim), torch.float32),
                                               ((n,), torch.float32), ((n,), torch.uint8), ((n,), torch.int32))]
        h[0].numpy()[:] = act
        _lib.check(env._lib.mgb_quad_step_host(env._h, *[x.data_ptr() for x in h], None, env._stream()))
        obs, rew, done, fail = (x.numpy().copy() for x in h[1:])
    else:
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        fail = env.fail_code
    out = [np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in (obs, rew, done)]
    out.append(None if fail is None else np.asarray(fail.cpu() if hasattr(fail, "cpu") else fail))
    sd = env.state_dict()
    out += [sd["state"].cpu().numpy(), sd["ct"].cpu().numpy()]
    env.close()
    return [name] + out


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8),
                                                 np.ascontiguousarray(b).view(np.uint8))


@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task", ["hovering_control", "velocity_control"])
def test_every_path_gives_the_same_bits(torch_mod, monkeypatch, task, config):
    """The envelope batch through the tile, wide (MGB_WIDE_KERNEL=1), packed (MGB_PACKED=1) kernels, rollout(1,
    actions=...) and the host zero-copy entry point, and -- tiled past the multi-wave threshold -- through the streaming
    kernel: every output and the post-step state equal the tile kernel's bit for bit (DESIGN.md section 4b)."""
    torch = torch_mod
    env_b = qe.envelope_batch(seed=13, nt=NT)
    sfx = _kernel_suffix(config)
    kernels = {"tile": "quad_step_kernel", "wide": "quad_step_wide_kernel", "packed": "quad_step2_kernel",
               "rollout": "quad_step_wide_kernel", "host_zerocopy": "quad_step_wide_kernel",   # by size at 9473 envs
               "stream": "quad_stream_kernel"}
    small = 9473                                    # a single wave of 132 SMs with >= 64 envs each: the wide kernel
    args = tuple(np.resize(x, (small,) + x.shape[1:]) for x in (env_b.state, env_b.ct, env_b.act)) + (task, config)
    ref = _run_path(torch, monkeypatch, "tile", *args)
    assert ref[0] == kernels["tile"] + sfx
    assert ref[4].any() and ref[3].any()            # some envs fail, some finish
    for path in ("wide", "packed", "rollout", "host_zerocopy"):
        got = _run_path(torch, monkeypatch, path, *args)
        assert got[0] == kernels[path] + sfx, path
        for k, (x, y) in enumerate(zip(got[1:], ref[1:])):
            assert x is None or _same_bits(x, y), (path, ("obs", "rew", "done", "fail", "state", "ct")[k])
    # past the multi-wave threshold: the streaming kernel against the tile kernel on the same tiled batch
    N = _stream_size()
    big = [np.resize(x, (N,) + x.shape[1:]) for x in (env_b.state, env_b.ct, env_b.act)]
    a = _run_path(torch, monkeypatch, "stream", *big, task, config)
    b = _run_path(torch, monkeypatch, "tile", *big, task, config)
    assert a[0] == kernels["stream"] + sfx and b[0] == kernels["tile"] + sfx
    for k, (x, y) in enumerate(zip(a[1:], b[1:])):
        assert _same_bits(x, y), ("stream", ("obs", "rew", "done", "fail", "state", "ct")[k])


# --------------------------------------------------------------------------------------------------------------------
# RK4 from the envelope states
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["tile", "rollout"])
@pytest.mark.parametrize("rk4_steps", [1, 4])
@pytest.mark.parametrize("config", ["default", "general"])
def test_rk4_step_vs_restatement(torch_mod, config, rk4_steps, path):
    """integrator="rk4" from the envelope states against qo.rk4_step(..., "f64"), within max(1e-5, 4 x the float32
    restatement's own error) per env.  Compared where the float64 step stays clear of the failure limits (RK4 stages
    from 900 rad/s overflow float32 by design of the model, and the step reports the failure); those envs must fail."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    env_b = qe.envelope_batch(seed=14, nt=NT)
    n, dt = env_b.state.shape[0], 0.01
    env = make_env(n, "hovering_control", dt=dt, nt=NT, integrator="rk4", rk4_steps=rk4_steps,
                   simulator_conf=_params(config))
    assert env.step_kernel_name() == "quad_step_kernel" + _kernel_suffix(config)
    set_state(env, env_b.state, env_b.ct)
    if path == "rollout":
        env.rollout(1, actions=torch.as_tensor(env_b.act[None]).cuda())
    else:
        env.step(torch.as_tensor(env_b.act).cuda())
        fail = env.fail_code.cpu().numpy()
    gs, _ = get_state(env)
    env.close()
    cfg = qo.make_cfg(_params(config))
    s64, s32 = (env_b.state.astype(np.float64) for _ in range(2))
    qo.rk4_step(cfg, s64, env_b.act, dt, rk4_steps, "f64")
    qo.rk4_step(cfg, s32, env_b.act, dt, rk4_steps, "f32")
    with np.errstate(invalid="ignore", over="ignore"):
        worst = np.max([np.linalg.norm(s64[:, lo:lo + 3], axis=1) / lim
                        for lo, lim in ((0, qe.FAIL_R), (3, qe.FAIL_V), (6, qe.FAIL_W))], axis=0)
    inside = np.isfinite(s64).all(axis=1) & (worst < 1 - 1e-3)
    outside = ~np.isfinite(s64).all(axis=1) | (worst > 1 + 1e-3)
    assert inside.mean() > 0.8 and outside.any()
    if path == "tile":
        assert not fail[inside].any() and fail[outside].all()
    err = group_rel_err_rows(gs[inside], s64[inside], STATE_GROUPS_W)
    own = group_rel_err_rows(s32[inside], s64[inside], STATE_GROUPS_W)
    tol = np.maximum(FLOOR, OWN * own)
    bad = np.nonzero(err > tol)[0]
    assert not bad.size, [(env_b.family[inside][i], float(err[i]), float(tol[i])) for i in bad[:8]]
    print("rk4 worst error %.3g, worst error / bound %.3g" % (err.max(), (err / tol).max()))


# --------------------------------------------------------------------------------------------------------------------
# obstacle-map edges, decided exactly
# --------------------------------------------------------------------------------------------------------------------
def _map_7x9(start):
    rng = np.random.RandomState(3)
    m = (rng.random_sample((7, 9)) < 0.5).astype(np.int64) * rng.randint(1, 9, (7, 9))
    m[:, 0] = m[:, 8] = m[0, :] = m[6, :] = 0
    m[::2, 0] = m[1::2, 8] = m[0, 1::3] = m[6, ::3] = 3         # obstacles along every edge, free cells between
    m[start] = -1
    return m


@pytest.mark.parametrize("start", [(0, 0), (3, 4)], ids=["corner", "interior"])
@pytest.mark.parametrize("task", ["no_collision", "hovering_control"])
def test_obstacle_map_edges_vs_literal_slice(torch_mod, tmp_path, task, start):
    """A 7 x 9 obstacle map with the start at a corner and in the interior.  R = I, w = 0, v_x = v_y = 0 and rotors at
    rest at the zero-thrust voltage, so x and y do not move at all, while z moves by +-3 cm in the step.  Windows that
    start negative (the numpy slice wraps once), end past the far edge, lie wholly outside the map; x, y and z on
    integers and on half cells.  done equals env.py:248-260 with a literal numpy slice, exactly."""
    torch = torch_mod
    m = _map_7x9(start)
    ys, xs = start
    path = tmp_path / "map.txt"
    path.write_text("".join(" ".join(str(int(v)) for v in row) + "\n" for row in m))
    free = m.copy()
    free[ys, xs] = 0
    cx = np.array([-12.0, -7.5, -3.0, -1.5, -1.0, -0.5, 0.0, 0.5, 1.0, 4.0, 7.5, 8.0, 8.5, 9.0, 9.5, 12.0])
    cy = np.array([-9.0, -7.0, -1.5, -1.0, -0.5, 0.0, 0.5, 3.0, 5.5, 6.0, 6.5, 7.0, 7.5, 11.0])
    zz = np.array([0.0, 1.0, 2.0, 0.5, 1.01, -0.5])
    X, Y, Z, V = [a.reshape(-1) for a in np.meshgrid(cx, cy, zz, np.array([3.0, -3.0]), indexing="ij")]
    n = X.size
    st = np.zeros((n, 22), np.float32)
    st[:, 0], st[:, 1], st[:, 2], st[:, 5] = X - xs, Y - ys, Z - 5.0, V
    st[:, 13] = st[:, 17] = st[:, 21] = 1.0
    assert np.array_equal(st[:, 0].astype(np.float64) + xs, X)
    assert np.array_equal((st[:, 2] + np.float32(5.0))[np.mod(Z, 1) == 0], Z[np.mod(Z, 1) == 0])   # z on integers
    env = make_env(n, task, dt=0.01, nt=1000, map_file=str(path))
    assert (env.x_offset, env.y_offset) == (xs, ys)
    set_state(env, st, np.zeros(n, np.int32))
    _, _, done, _ = env.step(torch.full((n, 4), float(qe.zero_thrust_voltage()), device="cuda"))
    done = done.cpu().numpy()
    assert not env.fail_code.cpu().numpy().any()
    post = env.state_dict()["state"].cpu().numpy()
    env.close()
    assert np.array_equal(post[:, :2], st[:, :2])                      # x and y did not move
    dz = post[:, 2] - st[:, 2]
    assert (np.sign(dz) == np.sign(V)).all() and (np.abs(dz) > 0.02).all()
    lit = np.array([qe.collides_literal(free, xs, ys, st[i, :3], post[i, :3]) for i in range(n)])
    bad = np.nonzero(done != lit)[0]
    assert not bad.size, [(X[i], Y[i], Z[i], V[i], bool(done[i])) for i in bad[:8]]
    assert 0.2 < lit.mean() < 0.8
