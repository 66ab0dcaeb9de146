"""GPU parity tests of the quadrotor path: libmgb200 (through the C ABI / BatchedQuadrotor) against
 (a) golden vectors recorded from the unmodified reference (tests/golden/quadrotor_golden.npz), and
 (b) the CPU oracle (oracle/quad_oracle.c) on seeded random batches,
plus size-independent properties at the BASELINE.json sizes (65 536 envs).

Tolerance: the north star asks for 1e-5 relative fp32 per step; teacher-forced single steps are asserted at 1e-5
(typically ~3e-7), free runs with an envelope that grows with the horizon (SURVEY.md 8c measured the reference's own
f32-vs-f64 drift at 7e-6 after 100 steps).
"""
import numpy as np
import pytest

from util import (OBS_GROUPS, QUAD_MAP_RUNS, QUAD_RUNS, STATE_GROUPS, golden_run, group_rel_err, group_rel_err_rows,
                  scalar_rel_err)

pytestmark = pytest.mark.gpu

RTOL_STEP = 1e-5


def _envelope(key):
    """Measured error-growth curves (tests/golden/measure_free_run_envelope.py, run on an H100): running max over the
    recorded reference episodes / oracle batches of group_rel_err at step j.  Tests assert 2x the curve."""
    import json
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "free_run_envelope.json")) as f:
        return np.asarray(json.load(f)[key], dtype=np.float64)


def _tol(curve, j, floor=5e-7):
    return max(2.0 * curve[min(j, len(curve) - 1)], floor)


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def make_env(n, task="hovering_control", **kw):
    from metagym_b200 import BatchedQuadrotor
    return BatchedQuadrotor(task=task, num_envs=n, device=0, squeeze=False, **kw)


def set_state(env, state, ct):
    import torch
    env.load_state_dict({"state": torch.as_tensor(np.asarray(state, dtype=np.float32)),
                         "ct": torch.as_tensor(np.asarray(ct, dtype=np.int32))})


def get_state(env):
    sd = env.state_dict()
    return sd["state"].cpu().numpy().astype(np.float64), sd["ct"].cpu().numpy()


def test_kat_zero_state(torch_mod, quad_golden):
    torch = torch_mod
    env = make_env(1, "no_collision")
    act = torch.tensor([[5.0, 6.0, 7.0, 8.0]], device="cuda")
    env.step(act)
    st, ct = get_state(env)
    assert group_rel_err(st, quad_golden["kat1_state"][None], STATE_GROUPS, floor=1e-12) < RTOL_STEP
    assert ct[0] == 1
    env.close()


def test_kat_200_steps(torch_mod, quad_golden):
    torch = torch_mod
    env = make_env(1, "velocity_control", nt=1000, seed=0)   # velocity_control: no floor, so the fall continues
    ref = quad_golden["kat2_states"]
    act = torch.full((1, 4), 5.0, device="cuda")
    for t in range(200):
        env.step(act)
        if t % 20 == 19:
            st, _ = get_state(env)
            assert group_rel_err(st, ref[t][None], STATE_GROUPS) < 5e-5
    env.close()


@pytest.mark.parametrize("name", QUAD_RUNS)
def test_teacher_forced_vs_reference(torch_mod, quad_golden, name):
    """Every recorded (state, ct, action) of a reference episode becomes one env of a batch; one step; compare."""
    torch = torch_mod
    r = golden_run(quad_golden, name)
    n = r["pre_state"].shape[0]
    kw = dict(dt=r["dt"], nt=r["nt"])
    if r["task"] == "velocity_control":
        kw["seed"] = r["seed"]
    env = make_env(n, r["task"], **kw)
    if r["task"] == "velocity_control":
        tbl = env.velocity_targets.cpu().numpy()[0]
        assert np.abs(tbl - r["targets"]).max() < 1e-5 * max(1.0, np.abs(r["targets"]).max())
        # use the reference's own table so the comparison below isolates the step
        env._lib.mgb_quad_set_targets(env._h, torch.as_tensor(r["targets"][None]).cuda().contiguous().data_ptr(), 1,
                                      env.env2task.data_ptr())
    set_state(env, r["pre_state"], r["pre_ct"])
    obs, rew, done, info = env.step(torch.as_tensor(r["act"]).cuda())
    st, ct = get_state(env)
    obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
    assert group_rel_err(st, r["post_state"], STATE_GROUPS) < RTOL_STEP
    assert group_rel_err(obs[:, :16], r["obs"][:, :16], OBS_GROUPS) < RTOL_STEP
    if r["task"] == "velocity_control":
        assert np.array_equal(obs[:, 16:], r["obs"][:, 16:])
    assert scalar_rel_err(rew, r["rew"]) < RTOL_STEP
    assert np.array_equal(done, r["done"])
    assert np.array_equal(ct, r["post_ct"])
    assert not env.fail_code.cpu().numpy().any()
    assert "next_target_g_v_x" in info or r["task"] != "velocity_control"     # reference test_env.py:37
    env.close()


@pytest.mark.parametrize("name", ["hover_a", "hover_fall", "nocol_a", "vel_a", "vel_c"])
def test_free_run_vs_reference(torch_mod, quad_golden, name):
    """Whole reference episodes (reset noise replayed, ct carried across episodes like the reference object)."""
    torch = torch_mod
    r = golden_run(quad_golden, name)
    kw = dict(dt=r["dt"], nt=r["nt"])
    if r["task"] == "velocity_control":
        kw["seed"] = r["seed"]
    env = make_env(1, r["task"], **kw)
    ep = r["ep"]
    curve = _envelope("curve_running_max")        # 3.9e-7 at step 1 ... 4.6e-6 at step 150 (the reference's own f32-vs-f64
    for k in range(int(ep.max()) + 1):            # drift: 7e-6 at step 100, SURVEY.md 8c)
        idx = np.nonzero(ep == k)[0]
        o0 = env.reset(noise=r["reset_noise"][k][None]).cpu().numpy()
        assert group_rel_err(o0[:, :16], r["reset_obs"][k][None, :16], OBS_GROUPS) < 1e-6
        if r["task"] == "velocity_control":
            assert np.abs(o0[0, 16:] - r["reset_obs"][k][16:]).max() < 1e-5
        for j, i in enumerate(idx):
            obs, rew, done, _ = env.step(torch.as_tensor(r["act"][i][None]).cuda())
            tol = _tol(curve, j)
            o = obs.cpu().numpy()
            assert group_rel_err(o[:, :16], r["obs"][i][None, :16], OBS_GROUPS) <= tol, (k, j)
            assert bool(done.cpu().numpy()[0]) == bool(r["done"][i]), (k, j)
            assert scalar_rel_err(rew.cpu().numpy(), r["rew"][i]) < max(tol, 1e-5), (k, j)
        _, ct = get_state(env)
        assert ct[0] == r["post_ct"][idx[-1]]
    env.close()


@pytest.mark.parametrize("task,dt", [("hovering_control", 0.01), ("velocity_control", 0.005), ("no_collision", 0.01)])
@pytest.mark.parametrize("n", [1, 127, 129, 4096])
def test_random_batch_vs_oracle(torch_mod, task, dt, n):
    """Seeded random batch: 20 free-running steps on GPU vs the CPU oracle (mixed-precision mode)."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    cfg = qo.make_cfg()
    rng = np.random.RandomState(1234 + n)
    nt = 30
    env = make_env(n, task, dt=dt, nt=nt, seed=[0, 1, 2])
    noise = rng.random_sample((n, 12))
    env.reset(noise=noise)
    state = qo.reset_state(None, noise)
    ct = np.zeros(n, np.int32)
    kw = {}
    if task == "velocity_control":
        kw = dict(targets=env.velocity_targets.cpu().numpy(), env2task=env.env2task.cpu().numpy())
    try:
        batch_curve = _envelope("random_batch_vs_oracle_running_max")     # measured, asserted x2
    except KeyError:
        batch_curve = 1.5e-6 * (1 + np.arange(20))
    for t in range(20):
        act = rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        o_ref, r_ref, d_ref, f_ref, _ = qo.env_step(cfg, state, ct, act, task, dt, nt, mode="mix", **kw)
        tol = _tol(batch_curve, t)
        assert group_rel_err(obs.cpu().numpy()[:, :16], o_ref[:, :16], OBS_GROUPS) <= tol, t
        assert scalar_rel_err(rew.cpu().numpy(), r_ref) < max(tol, 1e-5), t
        assert np.array_equal(done.cpu().numpy(), d_ref.astype(bool)), t
    st, ct_gpu = get_state(env)
    assert group_rel_err(st, state, STATE_GROUPS) < 1e-4
    assert np.array_equal(ct_gpu, ct)
    env.close()


def test_benchmark_shape_vs_oracle(torch_mod):
    """BASELINE.json configs[2] exactly as bench.py runs it -- 65 536 envs, velocity_control, dt = 0.005, nt = 1000, 64
    tasks, U(0.1, 15) actions, the 64-env tile kernel the launch rule picks for it -- stepped 20 times against the CPU
    oracle DIRECTLY (no chain through a smaller size).  Per-step error of every env, max over the batch."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    cfg = qo.make_cfg()
    n, dt, nt = 65536, 0.005, 1000
    rng = np.random.RandomState(77)
    env = make_env(n, "velocity_control", dt=dt, nt=nt, seed=list(range(64)))
    assert env.step_kernel_name().startswith("quad_step_kernel")
    noise = rng.random_sample((n, 12))
    env.reset(noise=noise)
    state = qo.reset_state(None, noise)
    ct = np.zeros(n, np.int32)
    kw = dict(targets=env.velocity_targets.cpu().numpy(), env2task=env.env2task.cpu().numpy())
    worst = 0.0
    for t in range(20):
        act = rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        o_ref, r_ref, d_ref, f_ref, _ = qo.env_step(cfg, state, ct, act, "velocity_control", dt, nt, mode="mix", **kw)
        o = obs.cpu().numpy()
        e = group_rel_err(o[:, :16], o_ref[:, :16], OBS_GROUPS)
        worst = max(worst, e)
        assert e < 3e-6 * (1 + t), t
        assert np.array_equal(o[:, 16:], o_ref[:, 16:].astype(np.float32)), t        # target rows: exact table reads
        assert scalar_rel_err(rew.cpu().numpy(), r_ref) < 1e-5, t
        assert np.array_equal(done.cpu().numpy(), d_ref.astype(bool)), t
        assert not env.fail_code.cpu().numpy().any()
    st, ct_gpu = get_state(env)
    assert group_rel_err(st, state, STATE_GROUPS) < 5e-5
    assert np.array_equal(ct_gpu, ct)
    env.close()


def test_general_config_path_vs_oracle(torch_mod, tmp_path):
    """A config that leaves the specialised kernel (off-diagonal inertia, raised rotors, cg offset, CT2 != 0), loaded
    from a file."""
    import json
    torch = torch_mod
    from oracle import quad_oracle as qo
    conf = qo.general_params()
    path = tmp_path / "conf.json"
    path.write_text(json.dumps(conf))
    cfg = qo.make_cfg(conf)
    n, dt, nt = 512, 0.01, 1000
    rng = np.random.RandomState(5)
    env = make_env(n, "hovering_control", dt=dt, nt=nt, simulator_conf=str(path))
    assert env.step_kernel_name() == "quad_step_kernel<false>"
    noise = rng.random_sample((n, 12))
    env.reset(noise=noise)
    state = qo.reset_state(conf, noise)
    ct = np.zeros(n, np.int32)
    for t in range(10):
        act = rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        o_ref, r_ref, d_ref, _, _ = qo.env_step(cfg, state, ct, act, "hovering_control", dt, nt, mode="mix")
        assert group_rel_err(obs.cpu().numpy(), o_ref, OBS_GROUPS) < 3e-6 * (1 + t)
        assert scalar_rel_err(rew.cpu().numpy(), r_ref) < 1e-5
    env.close()


def test_velocity_task_generator_vs_reference(torch_mod, quad_golden):
    """mgb_quad_make_targets == define_velocity_control_task (quadrotorsim.py:306-319) for seeds 0..5."""
    env = make_env(6, "velocity_control", dt=0.005, nt=40, seed=list(range(6)))
    tbl = env.velocity_targets.cpu().numpy()
    ref = quad_golden["veltask_tables"]
    scale = np.maximum(np.abs(ref).max(axis=2, keepdims=True), 1e-3)
    assert (np.abs(tbl - ref) / scale).max() < 2e-5
    # sample_task(seed) returns one table without touching the installed ones; set_task(seeds) installs new ones
    one = env.sample_task(3).cpu().numpy()
    assert np.array_equal(one, tbl[3]) and np.array_equal(env.velocity_targets.cpu().numpy(), tbl)
    env.set_task([5, 4])
    assert np.array_equal(env.velocity_targets.cpu().numpy(), tbl[[5, 4]])
    assert env.env2task.cpu().numpy().tolist() == [0, 1, 0, 1, 0, 1]
    env.close()


def test_velocity_task_generator_at_the_benchmarked_size(torch_mod, veltab_golden):
    """mgb_quad_make_targets at the table shape bench.py flies (nt=1000, dt=0.005, seeds 0..3) against the reference's
    define_velocity_control_task (quadrotorsim.py:306-319; tests/golden/gen_velocity_tables.py): 5000 free-running
    substeps from the zero state.  Tolerance: 2x the float32-vs-float64 drift measured along the same trajectories
    (5e-6 at t=999), floor 2e-6, relative to max(|row|, 1)."""
    ref, env_ = veltab_golden["tables"], veltab_golden["f32_vs_f64_envelope"].max(axis=0)
    seeds = [int(x) for x in veltab_golden["seeds"]]
    env = make_env(8, "velocity_control", dt=0.005, nt=1000, seed=seeds)
    tbl = env.velocity_targets.cpu().numpy()
    assert tbl.shape == ref.shape
    err = np.abs(tbl.astype(np.float64) - ref).max(axis=2) / np.maximum(np.abs(ref).max(axis=2), 1.0)      # [seed, t]
    tol = np.maximum(2.0 * env_, 2e-6)[None, :]
    assert (err <= tol).all(), (float(err.max()), np.argwhere(err > tol)[:5])
    env.close()


def test_failure_codes(torch_mod):
    torch = torch_mod
    env = make_env(4, "hovering_control")
    st = np.zeros((4, 22), np.float32)
    st[:, 13] = st[:, 17] = st[:, 21] = 1.0
    st[0, 3] = 150.0
    st[1, 6] = 2000.0
    st[2, 0] = 1500.0
    set_state(env, st, np.zeros(4, np.int32))
    obs, rew, done, _ = env.step(torch.full((4, 4), 5.0, device="cuda"))
    assert env.fail_code.cpu().tolist() == [2, 3, 1, 0]
    assert done.cpu().tolist() == [True, True, True, False]
    with pytest.raises(Exception, match="too large velocity"):
        env.raise_on_failure()
    env.close()


def test_host_path_equals_device_path(torch_mod):
    torch = torch_mod
    n = 1000
    rng = np.random.RandomState(3)
    noise = rng.random_sample((n, 12))
    a = make_env(n)
    b = make_env(n)
    a.reset(noise=noise)
    b.reset(noise=noise)
    for t in range(3):
        act = rng.uniform(0.1, 15, (n, 4)).astype(np.float32)
        o1, r1, d1, _ = a.step(torch.as_tensor(act).cuda())
        o2, r2, d2, _ = b.step(act)                       # numpy in -> host path -> numpy out
        assert isinstance(o2, np.ndarray)
        assert np.array_equal(o1.cpu().numpy(), o2) and np.array_equal(r1.cpu().numpy(), r2)
        assert np.array_equal(d1.cpu().numpy(), d2)
    a.close()
    b.close()


def test_host_step_is_ordered_after_device_work(torch_mod):
    """A numpy step right after a long asynchronous rollout() / reset() on the same env must see their results (the host
    entry point runs on the caller's stream; round-1 advice: it used a private non-blocking stream)."""
    torch = torch_mod
    n = 20000
    rng = np.random.RandomState(5)
    noise = rng.random_sample((n, 12))
    act = rng.uniform(0.1, 15, (n, 4)).astype(np.float32)
    a = make_env(n, "hovering_control", auto_reset=True)
    b = make_env(n, "hovering_control", auto_reset=True)
    for env in (a, b):
        env.reset(noise=noise)
    a.rollout(200, act_seed=3)                       # ~ms of asynchronous device work ...
    o1, r1, d1, _ = a.step(act)                      # ... immediately followed by the host path
    b.rollout(200, act_seed=3)
    torch.cuda.synchronize()
    o2, r2, d2, _ = b.step(torch.as_tensor(act).cuda())
    assert np.array_equal(o1, o2.cpu().numpy()) and np.array_equal(r1, r2.cpu().numpy())
    assert np.array_equal(d1, d2.cpu().numpy())
    a.close()
    b.close()


def test_host_path_reports_fail_codes_and_final_obs(torch_mod):
    torch = torch_mod
    st = np.zeros((4, 22), np.float32)
    st[:, 13] = st[:, 17] = st[:, 21] = 1.0
    st[0, 3] = 150.0
    st[1, 6] = 2000.0
    st[2, 0] = 1500.0
    act = np.full((4, 4), 5.0, np.float32)
    env = make_env(4, "hovering_control")
    set_state(env, st, np.zeros(4, np.int32))
    obs, rew, done, _ = env.step(act)                            # numpy in -> host path
    assert isinstance(obs, np.ndarray)
    assert list(env.fail_code) == [2, 3, 1, 0] and done.tolist() == [True, True, True, False]
    with pytest.raises(Exception, match="too large velocity"):
        env.raise_on_failure()
    env.close()
    # auto-reset: terminal observations come back through the host path too
    a = make_env(64, "hovering_control", auto_reset=True, rng_seed=2)
    b = make_env(64, "hovering_control", auto_reset=True, rng_seed=2)
    st = np.zeros((64, 22), np.float32)
    st[:, 13] = st[:, 17] = st[:, 21] = 1.0
    st[:, 2] = -4.999                                            # just above the floor: falls through it
    set_state(a, st, np.zeros(64, np.int32))
    set_state(b, st, np.zeros(64, np.int32))
    act = np.full((64, 4), 0.1, np.float32)
    for _ in range(3):
        o1, r1, d1, _ = a.step(act)
        o2, r2, d2, _ = b.step(torch.as_tensor(act).cuda())
        assert np.array_equal(o1, o2.cpu().numpy()) and np.array_equal(d1, d2.cpu().numpy())
        m = d1.astype(bool)
        assert np.array_equal(a.final_observation[m], b.final_observation.cpu().numpy()[m])
    assert d1.any() or True
    a.close()
    b.close()


def test_single_env_is_reference_shaped(torch_mod):
    from metagym_b200 import BatchedQuadrotor
    env = BatchedQuadrotor(task="velocity_control", num_envs=1, nt=10, dt=0.01)
    o = env.reset()
    assert tuple(o.shape) == (19,)
    step = 0
    done = False
    while not done:                                        # reference tests/test_env.py:31-40
        o, r, done, info = env.step(env.action_space.sample())
        assert "next_target_g_v_x" in info
        done = bool(done)
        step += 1
    assert step == env.nt
    env.close()


# ----------------------------------------------------------------------------------------------------------------
# BASELINE.json sizes: properties that do not need the oracle
# ----------------------------------------------------------------------------------------------------------------
def test_full_size_sharding_invariance_and_rollout(torch_mod):
    """65 536 envs (config 3): (i) two half-size handles with env_index_base reproduce one full handle bit for bit,
    auto-reset noise included; (ii) the fused T-step rollout kernel equals T single-step launches bit for bit."""
    torch = torch_mod
    N, T = 65536, 12
    kw = dict(dt=0.005, nt=8, seed=list(range(64)), auto_reset=True, rng_seed=77)
    full = make_env(N, "velocity_control", **kw)
    lo = make_env(N // 2, "velocity_control", env_index_base=0, **kw)
    hi = make_env(N // 2, "velocity_control", env_index_base=N // 2, **kw)
    fused = make_env(N, "velocity_control", **kw)
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = torch.rand((T, N, 4), device="cuda", generator=g) * 14.9 + 0.1
    for e in (full, lo, hi, fused):
        e.reset()
    out = fused.rollout(T, actions=acts)
    n_done = 0
    for t in range(T):
        o, r, d, _ = full.step(acts[t])
        o1, r1, d1, _ = lo.step(acts[t, : N // 2])
        o2, r2, d2, _ = hi.step(acts[t, N // 2:])
        assert torch.equal(o, torch.cat([o1, o2])) and torch.equal(r, torch.cat([r1, r2]))
        assert torch.equal(d, torch.cat([d1, d2]))
        assert torch.equal(out["obs"][t], o) and torch.equal(out["rew"][t], r)
        assert torch.equal(out["done"][t].bool(), d)
        assert torch.isfinite(o).all()
        n_done += int(d.sum())
    assert n_done == N                      # nt = 8: every env finishes exactly once in 12 steps
    s1, s2 = full.state_dict(), fused.state_dict()
    assert torch.equal(s1["state"], s2["state"]) and torch.equal(s1["ct"], s2["ct"])
    for e in (full, lo, hi, fused):
        e.close()


def test_full_size_hover_invariants(torch_mod):
    """4096- and 65 536-env hovering batches: outputs finite, done <=> floor contact or time limit, determinism, and
    the device-drawn actions equal the restated counter-based draws bit for bit."""
    torch = torch_mod
    from oracle import philox
    for N in (4096, 65536):
        a = make_env(N, "hovering_control", nt=50, auto_reset=True, rng_seed=5)
        b = make_env(N, "hovering_control", nt=50, auto_reset=True, rng_seed=5)
        a.reset()
        b.reset()
        ra = a.rollout(60, act_seed=9, want_actions=True)
        rb = b.rollout(60, act_seed=9)
        assert torch.equal(ra["obs"], rb["obs"]) and torch.equal(ra["rew"], rb["rew"])
        assert torch.isfinite(ra["obs"]).all() and torch.isfinite(ra["rew"]).all()
        drawn = ra["act"].cpu().numpy()
        for t in range(60):
            assert np.array_equal(drawn[t], philox.quad_rollout_actions(9, np.arange(N), t, 0.1, 15.0)), t
        # every env hits the nt = 50 limit once (random actions do not reach the floor 5 m below in 0.5 s)
        assert int(ra["done"].sum()) >= N
        a.close()
        b.close()


def test_auto_reset_publishes_first_obs_and_final_obs(torch_mod):
    """Every env ends its episode at once (nt = 3): the step returns the first observation of episode 2 and the state
    holds its reset state, both bit for bit against the restated draws; final_observation holds the terminal one."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    n = 256
    env = make_env(n, "no_collision", nt=3, auto_reset=True, rng_seed=1)
    ob = qo.OracleBatch(n, "no_collision", 0.01, 3, rng_seed=1, auto_reset=True)
    assert np.array_equal(env.reset().cpu().numpy(), ob.reset())
    act = np.full((n, 4), 5.0, np.float32)
    for t in range(3):
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        r = ob.step(act)
        assert group_rel_err(obs.cpu().numpy(), r.obs, OBS_GROUPS) < 1e-5
        assert scalar_rel_err(rew.cpu().numpy(), r.rew) < 1e-5
    assert bool(done.all()) and r.done.all()
    assert np.array_equal(obs.cpu().numpy(), r.obs)
    assert group_rel_err(env.final_observation.cpu().numpy(), r.final_obs, OBS_GROUPS) < 1e-5
    st, ct = get_state(env)
    assert np.all(ct == 0) and np.array_equal(st, ob.state)
    env.close()


def test_streaming_kernel_equals_tile_kernel(torch_mod, monkeypatch):
    """Multi-wave launches take the persistent TMA-pipelined kernel (quad_stream_kernel); it must reproduce the plain
    step kernel bit for bit, ragged last tile and auto-reset included (400 037 envs = 3125 full tiles + 37), in both
    SIMPLE instantiations (the default config, then the general one)."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    N = 400037
    for config in ("default", "general"):
        kw = dict(dt=0.005, nt=6, seed=list(range(16)), auto_reset=True, rng_seed=11,
                  simulator_conf=qo.general_params() if config == "general" else None)
        a = make_env(N, "velocity_control", **kw)              # streaming kernel (default for this size)
        assert a.step_kernel_name() == "quad_stream_kernel" + _kernel_suffix(config)
        monkeypatch.setenv("MGB_STREAM_KERNEL", "0")
        b = make_env(N, "velocity_control", **kw)              # plain kernel
        monkeypatch.delenv("MGB_STREAM_KERNEL")
        assert b.step_kernel_name() == "quad_step_kernel" + _kernel_suffix(config)
        g = torch.Generator(device="cuda").manual_seed(2)
        a.reset()
        b.reset()
        for t in range(9):
            act = torch.rand((N, 4), device="cuda", generator=g) * 16.0 - 0.5
            o1, r1, d1, _ = a.step(act)
            o2, r2, d2, _ = b.step(act)
            assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2), (config, t)
            if a.final_observation is not None:
                m = d1.bool()
                assert torch.equal(a.final_observation[m], b.final_observation[m])
        s1, s2 = a.state_dict(), b.state_dict()
        assert torch.equal(s1["state"], s2["state"]) and torch.equal(s1["ct"], s2["ct"])
        a.close()
        b.close()


@pytest.mark.parametrize("N,config", [pytest.param(N, c, id=str(N) + ("" if c == "default" else "-general"))
                                      for N in (9473, 65536, 67001) for c in ("default", "general")])
def test_wide_kernel_equals_tile_kernel(torch_mod, monkeypatch, N, config):
    """Single-wave launches can take the one-CTA-per-SM kernel (quad_step_wide_kernel; MGB_WIDE_KERNEL=1 selects it for
    every single-wave size); it must reproduce the 64-thread tile kernel bit for bit (ragged sizes, auto-reset, terminal
    observations).  67001 is just under the one-wave limit of an H100 (132 SMs x 512 envs)."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    kw = dict(dt=0.005, nt=5, seed=list(range(8)), auto_reset=True, rng_seed=4,
              simulator_conf=qo.general_params() if config == "general" else None)
    monkeypatch.setenv("MGB_WIDE_KERNEL", "1")
    a = make_env(N, "velocity_control", **kw)
    assert a.step_kernel_name() == "quad_step_wide_kernel" + _kernel_suffix(config)
    monkeypatch.setenv("MGB_WIDE_KERNEL", "0")
    b = make_env(N, "velocity_control", **kw)
    monkeypatch.delenv("MGB_WIDE_KERNEL")
    assert b.step_kernel_name() == "quad_step_kernel" + _kernel_suffix(config)
    g = torch.Generator(device="cuda").manual_seed(5)
    a.reset()
    b.reset()
    for t in range(8):
        act = torch.rand((N, 4), device="cuda", generator=g) * 16.0 - 0.5
        o1, r1, d1, _ = a.step(act)
        o2, r2, d2, _ = b.step(act)
        assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2), t
        m = d1.bool()
        assert torch.equal(a.final_observation[m], b.final_observation[m])
    s1, s2 = a.state_dict(), b.state_dict()
    assert torch.equal(s1["state"], s2["state"]) and torch.equal(s1["ct"], s2["ct"])
    a.close()
    b.close()


@pytest.mark.parametrize("task,dt,rk4_steps,path,config", [
    pytest.param(task, dt, k, path, c, id="%s-%s-%d" % (task, dt, k) + ("" if (path, c) == ("tile", "default") else
                                                                        "-%s-%s" % (path, c)))
    for task, dt, k in (("velocity_control", 0.005, 1), ("hovering_control", 0.01, 2))
    for path in ("tile", "wide", "stream", "rollout") for c in ("default", "general")])
def test_rk4_integrator_vs_restatement(torch_mod, monkeypatch, task, dt, rk4_steps, path, config):
    """integrator='rk4' (BASELINE config 3 wording; no reference counterpart, parity unpinned): the float32 kernel
    follows the float64 RK4 restatement of the same continuous-time model to 1e-5 over 20 free-running steps, on every
    path that integrates (the tile, wide and streaming step kernels and the rollout kernel) in both SIMPLE
    instantiations.  The packed kernel has no RK4: MGB_PACKED=1 falls back to a scalar kernel."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    params = qo.general_params() if config == "general" else None
    cfg = qo.make_cfg(params)
    n = {"wide": 9473, "stream": _stream_size()}.get(path, 2048)
    nt = 1000
    rng = np.random.RandomState(21)
    kw = dict(dt=dt, nt=nt, seed=[0, 1], integrator="rk4", rk4_steps=rk4_steps, simulator_conf=params)
    monkeypatch.setenv("MGB_WIDE_KERNEL", "1" if path == "wide" else "0")
    env = make_env(n, task, **kw)
    kname = {"wide": "quad_step_wide_kernel", "stream": "quad_stream_kernel"}.get(path, "quad_step_kernel")
    assert env.step_kernel_name() == kname + _kernel_suffix(config)
    if path == "tile":
        monkeypatch.setenv("MGB_PACKED", "1")
        packed = make_env(n, task, **kw)
        assert packed.step_kernel_name() == "quad_step_kernel" + _kernel_suffix(config)
        packed.close()
    monkeypatch.delenv("MGB_PACKED", raising=False)
    monkeypatch.delenv("MGB_WIDE_KERNEL")
    rows = _stream_subset(n) if path == "stream" else np.arange(n)
    noise = rng.random_sample((n, 12))
    env.reset(noise=noise)
    state = qo.reset_state(params, noise[rows])
    acts = [rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32) for _ in range(20)]
    if path == "rollout":
        for t0 in range(0, 20, 5):
            out = env.rollout(5, actions=torch.as_tensor(np.stack(acts[t0:t0 + 5])).cuda())
            assert torch.isfinite(out["obs"]).all() and not bool(out["done"].any())
    for t in range(20):
        if path != "rollout":
            obs, rew, done, _ = env.step(torch.as_tensor(acts[t]).cuda())
            assert torch.isfinite(obs).all() and not bool(done.any())
        qo.rk4_step(cfg, state, acts[t][rows], dt, rk4_steps, "f64")
    st, ct = get_state(env)
    assert group_rel_err(st[rows], state, STATE_GROUPS) < 2e-5
    assert np.all(ct == 20)
    env.close()


@pytest.mark.parametrize("task,dt,config", [
    pytest.param(task, dt, c, id="%s-%s" % (task, dt) + ("" if c == "default" else "-general"))
    for task, dt in (("velocity_control", 0.005), ("hovering_control", 0.01), ("no_collision", 0.003))
    for c in ("default", "general")])
@pytest.mark.parametrize("N", [1, 63, 9473, 65536, 70001, 151001])
def test_packed_kernel_equals_scalar_kernel(torch_mod, monkeypatch, N, task, dt, config):
    """The packed variant (MGB_PACKED=1: two envs per thread as two scalar chains; quad_step2_kernel) must reproduce the scalar
    one-env-per-thread instantiation of the same code bit for bit: ragged and odd sizes, auto-reset, terminal
    observations, fail codes, every task, and substep counts that do (5, 10) and do not (3) take the unrolled loop.
    Actions outside [0.1, 15] exercise the clamp; the long horizon lets hovering envs crash and velocity envs time out.
    This is also the guard against the compiler contracting multiply-add pairs in either lane (quad_lanes.cuh)."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    kw = dict(dt=dt, nt=5, auto_reset=True, rng_seed=4,
              simulator_conf=qo.general_params() if config == "general" else None)
    if task == "velocity_control":
        kw["seed"] = list(range(8))
    monkeypatch.setenv("MGB_PACKED", "1")
    a = make_env(N, task, **kw)
    monkeypatch.delenv("MGB_PACKED")
    if N > 1:
        assert a.step_kernel_name() == "quad_step2_kernel" + _kernel_suffix(config)
    b = make_env(N, task, **kw)
    assert not b.step_kernel_name().startswith("quad_step2_kernel")
    g = torch.Generator(device="cuda").manual_seed(5)
    a.reset()
    b.reset()
    steps = 8 if N > 20000 else 40
    for t in range(steps):
        act = torch.rand((N, 4), device="cuda", generator=g) * 16.0 - 0.5
        o1, r1, d1, _ = a.step(act)
        o2, r2, d2, _ = b.step(act)
        assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2), t
        assert torch.equal(a.fail_code, b.fail_code)
        m = d1.bool()
        assert torch.equal(a.final_observation[m], b.final_observation[m])
    s1, s2 = a.state_dict(), b.state_dict()
    assert torch.equal(s1["state"], s2["state"]) and torch.equal(s1["ct"], s2["ct"])
    a.close()
    b.close()


def test_packed_kernel_failing_env_does_not_disturb_its_pair_partner(torch_mod, monkeypatch):
    """Envs 2k and 2k+1 share a thread in the packed kernel.  When one of them leaves the valid zone mid-step
    (quadrotorsim.py:212-221) the other must still get exactly what the scalar kernel computes."""
    torch = torch_mod
    n = 256
    rng = np.random.RandomState(9)
    st = np.zeros((n, 22), np.float32)
    st[:, 13] = st[:, 17] = st[:, 21] = 1.0
    st[:, 3:6] = rng.uniform(-2, 2, (n, 3))
    st[:, 6:9] = rng.uniform(-5, 5, (n, 3))
    st[0::7, 3] = 99.9995        # |v| crosses 100 during the step for some of these, not for others
    st[3::11, 6] = 999.99        # |w| close to the 1000 limit
    st[5::13, 0] = 999.999       # range limit
    act = torch.as_tensor(rng.uniform(0.1, 15, (n, 4)).astype(np.float32)).cuda()
    outs = []
    for packed in ("1", "0"):
        monkeypatch.setenv("MGB_PACKED", packed)
        env = make_env(n, "hovering_control", dt=0.01)
        assert env.step_kernel_name().startswith("quad_step2_kernel") == (packed == "1")
        set_state(env, st, np.zeros(n, np.int32))
        o, r, d, _ = env.step(act)
        outs.append((o.clone(), r.clone(), d.clone(), env.fail_code.clone(), env.state_dict()["state"].clone()))
        env.close()
    monkeypatch.delenv("MGB_PACKED")
    fails = outs[0][3].cpu().numpy()
    assert (fails > 0).sum() >= 10 and (fails == 0).sum() >= 100
    pairs = fails.reshape(-1, 2)
    assert ((pairs > 0).sum(axis=1) == 1).sum() >= 5          # mixed pairs exist
    for x, y in zip(outs[0], outs[1]):
        assert torch.equal(x, y)


@pytest.mark.parametrize("name", QUAD_MAP_RUNS)
def test_obstacle_map_vs_reference(torch_mod, quad_golden, name, tmp_path):
    """map_file= (SURVEY.md 8f row 4): teacher-forced steps of reference episodes flown over an obstacle map; the
    collision / done pattern (episodes end at z + 5 < 1 over obstacle cells) must be reproduced exactly."""
    torch = torch_mod
    r = golden_run(quad_golden, name)
    path = tmp_path / "map.txt"
    path.write_text("".join(" ".join(str(int(v)).zfill(2) for v in row) + "\n" for row in quad_golden["map_obst"]))
    n = r["pre_state"].shape[0]
    env = make_env(n, r["task"], dt=r["dt"], nt=r["nt"], map_file=str(path))
    assert (env.x_offset, env.y_offset) == (5, 5)
    set_state(env, r["pre_state"], r["pre_ct"])
    obs, rew, done, _ = env.step(torch.as_tensor(r["act"]).cuda())
    assert np.array_equal(done.cpu().numpy(), r["done"]) and r["done"].sum() >= 2
    assert scalar_rel_err(rew.cpu().numpy(), r["rew"]) < RTOL_STEP
    assert group_rel_err(obs.cpu().numpy()[:, :16], r["obs"][:, :16], OBS_GROUPS) < RTOL_STEP
    _, ct = get_state(env)
    assert np.array_equal(ct, r["post_ct"])
    env.close()
    # the same states on the flat default map do NOT collide (z + 5 is ~0.98 > 0)
    flat = make_env(n, r["task"], dt=r["dt"], nt=r["nt"])
    set_state(flat, r["pre_state"], r["pre_ct"])
    _, _, done2, _ = flat.step(torch.as_tensor(r["act"]).cuda())
    assert int(done2.sum()) < int(r["done"].sum())
    flat.close()


@pytest.mark.parametrize("task,action", [("no_collision", 1.0), ("hovering_control", 0.1)])
def test_reference_smoke_episode_to_termination(torch_mod, task, action):
    """The reference's own tests (quadrotor/tests/test_env.py:20-29) fly constant actions until the env says done.
    Same here on one env, side by side with the numpy port (bit-identical to the reference): same episode length,
    observations within the free-run envelope."""
    torch = torch_mod
    from oracle.quadrotor_np import NumpyQuadrotorEnv
    rng = np.random.RandomState(8)
    noise = rng.random_sample(12)
    ref = NumpyQuadrotorEnv(task=task)
    st = np.random.get_state()
    np.random.seed(0)
    # feed the port's reset() the same 12 draws the engine replays
    import unittest.mock as mock
    draws = iter([noise[0:3], noise[3:6], noise[6:9], noise[9:12]])
    with mock.patch("numpy.random.random", side_effect=lambda n: next(draws)):
        o_ref = ref.reset()
    np.random.set_state(st)
    env = make_env(1, task)
    o = env.reset(noise=noise[None]).cpu().numpy()[0]
    assert group_rel_err(o[None, :16], o_ref[None, :16], OBS_GROUPS) < 1e-6
    act = np.full(4, action, dtype=np.float32)
    steps = 0
    while True:
        obs, rew, done, _ = env.step(torch.as_tensor(act[None]).cuda())
        o_ref, r_ref, d_ref, _ = ref.step(act)
        steps += 1
        assert bool(done[0]) == bool(d_ref), steps
        assert group_rel_err(obs.cpu().numpy()[:, :16], o_ref[None, :16], OBS_GROUPS) < 5e-6 * (1 + steps)
        if d_ref:
            break
    assert 50 < steps < 1000          # falls the 5 m to the floor
    env.close()


@pytest.mark.parametrize("name", ["c_hover", "c_nocol", "c_vel", "c_spin"])
def test_custom_simulator_config_vs_reference(torch_mod, name, tmp_path):
    """Reference episodes recorded with a NON-default config (off-diagonal inertia, centre-of-gravity offset, CT[2],
    out-of-plane rotor, initial velocities, other voltage range, healthy_reward = 2; tests/golden/gen_quadrotor_conf.py):
    the terms config.json zeroes are exercised.  Teacher-forced steps at 1e-5, reset with replayed draws, and the
    velocity-task table built from this config."""
    import json
    import os
    torch = torch_mod
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quadrotor_conf_golden.npz"))
    conf = tmp_path / "conf.json"
    conf.write_text(str(g["conf_json"]))
    assert json.loads(conf.read_text())["quality"] == 0.8
    r = golden_run(g, name)
    n = r["pre_state"].shape[0]
    kw = dict(dt=r["dt"], nt=r["nt"], simulator_conf=str(conf), healthy_reward=float(g["healthy_reward"]))
    if r["task"] == "velocity_control":
        kw["seed"] = r["seed"]
    env = make_env(n, r["task"], **kw)
    if r["task"] == "velocity_control":
        tbl = env.velocity_targets.cpu().numpy()[0]
        assert np.abs(tbl - r["targets"]).max() < 2e-5 * max(1.0, np.abs(r["targets"]).max())
        env._lib.mgb_quad_set_targets(env._h, torch.as_tensor(r["targets"][None]).cuda().contiguous().data_ptr(), 1,
                                      env.env2task.data_ptr())
    # reset with the recorded draws reproduces the recorded first observation
    noise = np.tile(r["reset_noise"][:1], (n, 1))
    o0 = env.reset(noise=noise).cpu().numpy()
    assert group_rel_err(o0[:1, :16], r["reset_obs"][:1, :16].astype(np.float64), OBS_GROUPS) < RTOL_STEP
    set_state(env, r["pre_state"], r["pre_ct"])
    obs, rew, done, info = env.step(torch.as_tensor(r["act"]).cuda())
    st, ct = get_state(env)
    obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
    assert group_rel_err(st, r["post_state"], STATE_GROUPS) < RTOL_STEP
    assert group_rel_err(obs[:, :16], r["obs"][:, :16], OBS_GROUPS) < RTOL_STEP
    assert scalar_rel_err(rew, r["rew"]) < RTOL_STEP
    assert np.array_equal(done, r["done"]) and np.array_equal(ct, r["post_ct"])
    assert not env.fail_code.cpu().numpy().any()
    env.close()


# ----------------------------------------------------------------------------------------------------------------
# Path matrix: every way the engine reaches its outputs, against the oracle batch, through auto-resets
# ----------------------------------------------------------------------------------------------------------------
MATRIX_SEED = 0x9E3779B97F4A7C15          # reset draws; both 32-bit halves non-zero
MATRIX_ACT_SEED = 0xD1B54A32D192ED03      # device-drawn rollout actions
MATRIX_TASKS = [("no_collision", "map"), ("hovering_control", "flat"), ("hovering_control", "map"),
                ("velocity_control", "flat")]
# path -> (step kernel a step of this batch launches, environment settings at creation)
MATRIX_PATHS = {
    "tile": ("quad_step_kernel", {}),
    "wide": ("quad_step_wide_kernel", {"MGB_WIDE_KERNEL": "1"}),
    "packed": ("quad_step2_kernel", {"MGB_PACKED": "1"}),
    "stream": ("quad_stream_kernel", {}),
    "rollout": ("quad_step_kernel", {}),
    "rollout_drawn": ("quad_step_kernel", {}),
    "host_copy": ("quad_step_kernel", {"MGB_HOST_ZEROCOPY": "0"}),
    "host_zerocopy": ("quad_step_kernel", {}),
    "host_zerocopy_stream": ("quad_stream_kernel", {}),
    "host_hybrid": ("quad_step_kernel", {"MGB_HOST_ZEROCOPY": "2"}),
}


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stream_size():
    """Just over the multi-wave threshold of the 64-env tile kernel: the persistent streaming kernel takes it, and the
    last 128-env state tile is ragged (37 envs)."""
    return _num_sms() * 32 * 64 + 37


def _stream_subset(n):
    """Envs the oracle follows in a streaming-size batch: the first and last two 128-env tiles and every 97th env."""
    last = ((n + 127) // 128 - 2) * 128
    return np.unique(np.concatenate([np.arange(256), np.arange(last, n), np.arange(0, n, 97)]))


def _kernel_suffix(config):
    return "<true>" if config == "default" else "<false>"


def _make_edge_states(st, ct, rows, task, terrain, rng, nt):
    """Some followed envs start next to a decision, each placed decisively on one side so that float32 error cannot
    flip it: across the range / velocity / angular-velocity limits within the first substep or not, through the floor
    or an obstacle cell's 1 m ceiling within the step or not.  Every env starts at a random ct."""
    ct[:] = rng.randint(0, nt - 1, ct.size)
    kinds = {0: ((999.999, 0, 0), (1.5, None, None), None),          # range: fails in substep 1
             1: ((999.999, 0, 0), (-1.5, None, None), None),         # range: moves away
             2: (None, (103.0, 0.0, 0.0), None),                     # |v|: 100.4 after substep 1 (drag 2.5 / substep)
             3: (None, (99.9995, 0.0, 0.0), None),                   # |v|: drag pulls it below at once
             4: (None, None, (999.99, 0.0, 0.0))}                    # |w|: angular drag overshoots past -1000
    if task != "velocity_control":
        if terrain == "map":
            kinds[5] = ((-1.5, -1.5, -3.995), (None, None, -2.0), None)    # over obstacle cells, z 1.005 -> 0.985
            kinds[6] = ((-1.5, -1.5, -3.5), (None, None, 0.0), None)       # over obstacle cells, z 1.5
            kinds[7] = ((5.5, 0.0, -4.995), (None, None, -2.0), None)      # over free cells, z 0.005 -> below 0
        else:
            kinds[5] = ((0.0, 0.0, -4.995), (None, None, -2.0), None)      # z 0.005 -> below the floor
            kinds[6] = ((0.0, 0.0, -4.9), (None, None, 0.5), None)         # z 0.1, rising
    for k, (p, v, w) in kinds.items():
        e = rows[k::17]
        for off, vals in ((0, p), (3, v), (6, w)):
            for j, x in enumerate(vals or ()):
                if x is not None:
                    st[e, off + j] = x


def _done_flip_is_marginal(ob, r, i, gpu_fail):
    """A done flag the GPU and the oracle disagree on is accepted only when the oracle's deciding quantity lies within
    1e-5 (relative) of its threshold, where the float32 error of a free run can land it: |p|^2, |v|^2, |w|^2 for a
    failure; for a collision min(z_old, z_new) against the floor, or, over an obstacle map, the altitudes and the
    swept cell window against the integers where the collision rule changes."""
    rel = 1e-5
    pre, end = r.pre_state[i], r.end_state[i]
    if r.fail[i] or gpu_fail:
        c = ob.cfg
        q = [(end[0:3] @ end[0:3], c.fail_r ** 2), (end[3:6] @ end[3:6], c.fail_v ** 2),
             (end[6:9] @ end[6:9], c.fail_w ** 2)]
        return any(abs(a / b - 1.0) <= rel for a, b in q)
    if ob.task == "velocity_control":
        return False                      # only ct == nt and a failure end its episodes
    zo = np.float32(ob.z_off)
    z = (np.float32(pre[2]) + zo, np.float32(end[2]) + zo)
    if ob.map_matrix is None:
        return abs(float(min(z))) <= rel * ob.z_off

    def near_int(q):
        return abs(q - round(q)) <= rel * max(1.0, abs(q))
    ys, xs = np.nonzero(np.asarray(ob.map_matrix) == -1)
    x = (pre[0] + xs[0], end[0] + xs[0])
    y = (pre[1] + ys[0], end[1] + ys[0])
    return any(near_int(float(q)) for q in (min(z), max(z), min(x), max(x), min(y), max(y)))


def _matrix_batch(n, task, terrain, config, map_matrix, tmp_dir):
    """The path matrix's batch, created under the caller's environment settings, and its oracle batch: episode 1 drawn
    on the device and compared bit for bit with the restatement, then the edge states loaded.  Returns (env, oracle
    batch, numpy RandomState for the actions)."""
    import os
    from oracle import quad_oracle as qo
    params = qo.general_params() if config == "general" else None
    vel = task == "velocity_control"
    dt, nt = (0.005 if vel else 0.01), 7
    base = 2 ** 32 - 50 if vel else 0
    kw = dict(dt=dt, nt=nt, auto_reset=True, rng_seed=MATRIX_SEED, env_index_base=base, simulator_conf=params)
    if vel:
        kw["seed"] = list(range(5))
    if terrain == "map":
        kw["map_file"] = os.path.join(tmp_dir, "map.txt")
        with open(kw["map_file"], "w") as f:
            f.write("".join(" ".join(str(int(v)).zfill(2) for v in row) + "\n" for row in map_matrix))
    env = make_env(n, task, **kw)
    ob = qo.OracleBatch(n, task, dt, nt, params=params, map_matrix=map_matrix if terrain == "map" else None,
                        rng_seed=MATRIX_SEED, env_index_base=base, auto_reset=True,
                        subset=_stream_subset(n) if n > 100000 else None,
                        targets=env.velocity_targets.cpu().numpy() if vel else None,
                        env2task=env.env2task.cpu().numpy() if vel else None)
    rows = ob.idx
    assert np.array_equal(env.reset().cpu().numpy()[rows], ob.reset())
    st, ct = get_state(env)
    assert np.array_equal(st[rows], ob.state)
    rng = np.random.RandomState(17)
    st = st.astype(np.float32)
    _make_edge_states(st, ct, rows, task, terrain, rng, nt)
    set_state(env, st, ct)
    ob.state[:] = st[rows]
    ob.ct[:] = ct[rows]
    return env, ob, rng


@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task,terrain", MATRIX_TASKS)
@pytest.mark.parametrize("path", list(MATRIX_PATHS))
def test_path_matrix_vs_oracle(torch_mod, quad_golden, monkeypatch, tmp_path, path, task, terrain, config):
    """Every path to the engine's outputs -- the tile, wide, packed and streaming step kernels, the rollout kernel with
    given and device-drawn actions, the host entry point by copies, zero-copy and hybrid -- in both SIMPLE
    instantiations, against the oracle batch (oracle.quad_oracle.OracleBatch) for 20 steps with nt = 7, so that every env
    auto-resets at least twice.  Per step: done and fail codes exactly; obs and reward within 2x the error envelope
    measured on these batches (tests/golden/measure_free_run_envelope.py), indexed by steps since the env's last reset; reset observations, and the state right after a reset, bit
    for bit against the restated counter-based draws; terminal observations within the same envelope.  At the end the
    whole followed state within 5e-5 and ct exactly."""
    torch = torch_mod
    from metagym_b200 import _lib
    from oracle import philox
    kname, env_vars = MATRIX_PATHS[path]
    n = {"wide": 9473, "stream": _stream_size(), "host_zerocopy_stream": _stream_size()}.get(path, 4099)
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    env, ob, rng = _matrix_batch(n, task, terrain, config, quad_golden["map_obst"], str(tmp_path))
    for k in env_vars:
        monkeypatch.delenv(k)
    assert env.step_kernel_name() == kname + _kernel_suffix(config)
    rows, vel, base = ob.idx, task == "velocity_control", int(ob.genv[0] - ob.idx[0])

    curve = _envelope("path_matrix_running_max")
    desync = np.zeros(rows.size, bool)     # envs whose done flag flipped in this launch: resynchronised after it
    since = np.zeros(rows.size, np.int64)  # steps since the env's last reset
    accepted = []

    def check_step(t, act, obs, rew, done, fail=None, final=None):
        ep_before = ob.ep.copy()
        r = ob.step(act)
        g_obs, g_rew, g_done = obs[rows], rew[rows].astype(np.float64), done[rows].astype(bool)
        g_fail = fail[rows] if fail is not None else np.zeros(rows.size, np.int32)
        live = ~desync
        flip = live & (g_done != r.done)
        for i in np.nonzero(flip)[0]:
            assert _done_flip_is_marginal(ob, r, i, g_fail[i]), (t, int(rows[i]), bool(g_done[i]), int(g_fail[i]))
            accepted.append((t, int(rows[i])))
        desync[flip] = True
        ok = live & ~flip
        tol = np.maximum(2.0 * curve[np.minimum(since, len(curve) - 1)], 5e-7)
        if fail is not None:
            assert np.array_equal(g_fail[ok], r.fail[ok]), t
        cont, fresh = ok & ~r.done, ok & r.done
        err = group_rel_err_rows(g_obs[cont, :16], r.obs[cont, :16], OBS_GROUPS)
        assert (err <= tol[cont]).all(), (t, float(err.max()), rows[cont][np.argmax(err - tol[cont])])
        if vel:
            assert np.array_equal(g_obs[ok, 16:], r.obs[ok, 16:]), t
        rerr = np.abs(g_rew - r.rew) / np.maximum(np.abs(r.rew), 1.0)
        assert (rerr[ok] <= np.maximum(tol[ok], 1e-5)).all(), (t, float(rerr[ok].max()))
        assert np.array_equal(g_obs[fresh], r.obs[fresh]), t            # reset observations, bit for bit
        if final is not None:
            ferr = group_rel_err_rows(final[rows][fresh, :16], r.final_obs[fresh, :16], OBS_GROUPS)
            assert (ferr <= tol[fresh]).all(), (t, float(ferr.max()) if ferr.size else 0.0)
        ob.ep[desync] = ep_before[desync] + g_done[desync]                 # the GPU's episode count
        since[:] = np.where(g_done, 0, since + 1)
        return fresh

    def sync(fresh):
        """After a launch: envs reset by its last step hold the restated reset state bit for bit; envs whose done
        flag flipped take the GPU's state."""
        gs, gc = get_state(env)
        gs, gc = gs[rows], gc[rows]
        assert np.array_equal(gs[fresh], ob.state[fresh]) and np.array_equal(gc[fresh], ob.ct[fresh])
        ob.state[desync] = gs[desync]
        ob.ct[desync] = gc[desync]
        desync[:] = False
        return gs, gc

    steps = 20
    acts = [rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32) for _ in range(steps)]
    if path in ("rollout", "rollout_drawn"):
        T = 5 if path == "rollout" else 10
        genv = base + np.arange(n)
        for t0 in range(0, steps, T):
            if path == "rollout":
                out = env.rollout(T, actions=torch.as_tensor(np.stack(acts[t0:t0 + T])).cuda())
            else:
                out = env.rollout(T, act_seed=MATRIX_ACT_SEED, want_actions=True)
                drawn = out["act"].cpu().numpy()
                for t in range(T):                  # t_base continues across consecutive rollouts
                    acts[t0 + t] = philox.quad_rollout_actions(MATRIX_ACT_SEED, genv, t0 + t, env._cfg.min_voltage,
                                                               env._cfg.max_voltage)
                    assert np.array_equal(drawn[t], acts[t0 + t]), t0 + t
            o, r_, d = out["obs"].cpu().numpy(), out["rew"].cpu().numpy(), out["done"].cpu().numpy()
            for t in range(T):
                fresh = check_step(t0 + t, acts[t0 + t], o[t], r_[t], d[t])
            gs, gc = sync(fresh)
    elif path.startswith("host"):
        D = env.obs_dim

        def pinned(shape, dtype):
            return torch.zeros(shape, dtype=dtype).pin_memory()
        h_act, h_obs, h_rew = pinned((n, 4), torch.float32), pinned((n, D), torch.float32), pinned((n,), torch.float32)
        h_done, h_fail, h_final = pinned((n,), torch.uint8), pinned((n,), torch.int32), pinned((n, D), torch.float32)
        for t in range(steps):
            h_act.numpy()[:] = acts[t]
            _lib.check(env._lib.mgb_quad_step_host(env._h, h_act.data_ptr(), h_obs.data_ptr(), h_rew.data_ptr(),
                                                   h_done.data_ptr(), h_fail.data_ptr(), h_final.data_ptr(),
                                                   env._stream()))
            fresh = check_step(t, acts[t], h_obs.numpy().copy(), h_rew.numpy().copy(), h_done.numpy().copy(),
                               h_fail.numpy().copy(), h_final.numpy().copy())
            gs, gc = sync(fresh)
    else:
        for t in range(steps):
            obs, rew, done, _ = env.step(torch.as_tensor(acts[t]).cuda())
            fresh = check_step(t, acts[t], obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy(),
                               env.fail_code.cpu().numpy(), env.final_observation.cpu().numpy())
            gs, gc = sync(fresh)
    assert group_rel_err(gs, ob.state, STATE_GROUPS) < 5e-5
    assert np.array_equal(gc, ob.ct)
    assert (ob.ep >= 3).all()              # the first reset and at least two auto-resets
    assert len(accepted) <= 3, accepted
    env.close()


def test_path_matrix_covers_every_step_kernel():
    """The kernels the path matrix asserts: all four step kernels, each in both SIMPLE instantiations."""
    names = {MATRIX_PATHS[p][0] + _kernel_suffix(c) for p in MATRIX_PATHS for c in ("default", "general")}
    assert names == {k + s for k in ("quad_step_kernel", "quad_step_wide_kernel", "quad_step2_kernel",
                                     "quad_stream_kernel") for s in ("<true>", "<false>")}


@pytest.mark.parametrize("task", ["hovering_control", "velocity_control"])
def test_masked_reset_vs_restatement(torch_mod, task):
    """reset(mask): masked-in envs take the restated draws of episode ep + 1, bit for bit; masked-out envs keep their
    state, ct and episode count, and their observation equals bit for bit the one their last step returned.
    reset(noise=..., mask) replays the draws without advancing the episode count, which the draws of the next
    auto-reset show."""
    torch = torch_mod
    from oracle import quad_oracle as qo
    n, nt, dt, seed, base = 1000, 5, 0.01, 0xC0FFEE1234567, 77
    kw = dict(dt=dt, nt=nt, auto_reset=True, rng_seed=seed, env_index_base=base)
    if task == "velocity_control":
        kw["seed"] = [0, 1, 2]
    env = make_env(n, task, **kw)
    vel = task == "velocity_control"
    ob = qo.OracleBatch(n, task, dt, nt, rng_seed=seed, env_index_base=base, auto_reset=True,
                        targets=env.velocity_targets.cpu().numpy() if vel else None,
                        env2task=env.env2task.cpu().numpy() if vel else None)
    assert np.array_equal(env.reset().cpu().numpy(), ob.reset())
    rng = np.random.RandomState(4)
    for _ in range(2):
        act = rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)
        obs, _, done, _ = env.step(torch.as_tensor(act).cuda())
        ob.step(act)
    assert not bool(done.any())
    last_obs = obs.cpu().numpy().copy()
    st0, ct0 = get_state(env)
    ob.state[:], ob.ct[:] = st0, ct0                  # carry on from the GPU's state: only the resets are compared
    mask = rng.random_sample(n) < 0.4
    o = env.reset(mask=torch.as_tensor(mask)).cpu().numpy()
    o_ref = ob.reset(mask=mask)
    st, ct = get_state(env)
    assert np.array_equal(o[mask], o_ref[mask]) and np.array_equal(st[mask], ob.state[mask])
    assert np.array_equal(st[~mask], st0[~mask]) and np.array_equal(ct, ct0)
    assert np.array_equal(o[~mask], last_obs[~mask])
    mask2 = rng.random_sample(n) < 0.5
    noise = rng.random_sample((n, 12))
    o = env.reset(mask=torch.as_tensor(mask2), noise=noise).cpu().numpy()
    o_ref = ob.reset(mask=mask2, noise=noise)
    st, _ = get_state(env)
    assert np.array_equal(o[mask2], o_ref[mask2]) and np.array_equal(st[mask2], ob.state[mask2])
    # ct is 2 everywhere: the third step from here ends every episode, and the auto-reset draws with ep + 1
    for t in range(nt - 2):
        act = rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)
        obs, _, done, _ = env.step(torch.as_tensor(act).cuda())
        r = ob.step(act)
        assert np.array_equal(done.cpu().numpy(), r.done), t
    assert r.done.all() and np.array_equal(np.unique(ob.ep), [2, 3])
    st, ct = get_state(env)
    assert np.array_equal(obs.cpu().numpy(), r.obs) and np.array_equal(st, ob.state) and (ct == 0).all()
    env.close()
