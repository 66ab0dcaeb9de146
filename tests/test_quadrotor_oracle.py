"""CPU: pin the oracle (oracle/quad_oracle.c) against golden vectors produced by the unmodified reference."""
import numpy as np
import pytest

from oracle import quad_oracle as qo
from util import OBS_GROUPS, QUAD_MAP_RUNS, QUAD_RUNS, STATE_GROUPS, golden_run, group_rel_err, scalar_rel_err


@pytest.fixture(scope="module")
def cfg():
    return qo.make_cfg()


def test_kat_zero_state_one_step(quad_golden, cfg):
    # never-reset simulator: all-float32 mode; agreement is at the float32 rounding level
    s = qo.zero_state(1)
    power, fail = qo.sim_step(cfg, s, np.array([[5, 6, 7, 8]], np.float32), 10, "f32")
    assert group_rel_err(s, quad_golden["kat1_state"][None], STATE_GROUPS, floor=1e-12) < 2e-6
    assert abs(power[0] - float(quad_golden["kat1_power"])) < 1e-3
    assert fail[0] == 0


def test_kat_200_steps(quad_golden, cfg):
    s = qo.zero_state(1)
    ref = quad_golden["kat2_states"]
    for t in range(200):
        qo.sim_step(cfg, s, np.array([[5, 5, 5, 5]], np.float32), 10, "f32")
        assert group_rel_err(s, ref[t][None], STATE_GROUPS) < 2e-5
    # SURVEY.md 8c quotes p_z=-2.3465273, v_z=-0.5655445, prop_w=283.22287 for this trajectory
    assert abs(ref[-1][2] - (-2.3465273)) < 1e-5 and abs(ref[-1][9] - 283.22287) < 1e-3


@pytest.mark.parametrize("name", QUAD_RUNS)
def test_teacher_forced_step(quad_golden, cfg, name):
    """One env.step from every recorded pre-step state of the reference (mixed precision after reset())."""
    r = golden_run(quad_golden, name)
    state = np.array(r["pre_state"], dtype=np.float64)
    ct = np.array(r["pre_ct"], dtype=np.int32)
    n = state.shape[0]
    kw = {}
    if r["task"] == "velocity_control":
        kw = dict(targets=r["targets"][None], env2task=np.zeros(n, np.int32))
    obs, rew, done, fail, power = qo.env_step(cfg, state, ct, r["act"], r["task"], r["dt"], r["nt"], mode="mix", **kw)
    assert group_rel_err(state, r["post_state"], STATE_GROUPS) < 1e-6
    assert group_rel_err(obs[:, :16], r["obs"][:, :16], OBS_GROUPS) < 1e-6
    if r["task"] == "velocity_control":
        assert np.array_equal(obs[:, 16:], r["obs"][:, 16:])
    assert scalar_rel_err(rew, r["rew"]) < 1e-6
    assert np.array_equal(done.astype(bool), r["done"])
    assert np.array_equal(ct, r["post_ct"])
    assert scalar_rel_err(power, r["power"]) < 1e-6
    assert not fail.any()


@pytest.mark.parametrize("name", ["hover_a", "vel_a", "nocol_a"])
def test_free_run_with_reset_replay(quad_golden, cfg, name):
    """Whole episodes from the replayed reset noise; the envelope grows with the horizon (SURVEY.md 8c)."""
    r = golden_run(quad_golden, name)
    ep = r["ep"]
    for k in range(int(ep.max()) + 1):
        idx = np.nonzero(ep == k)[0]
        state = qo.reset_state(None, r["reset_noise"][k][None])
        ct = np.array([r["reset_ct"][k]], np.int32)
        assert np.array_equal(state[0], r["pre_state"][idx[0]])
        kw = {}
        if r["task"] == "velocity_control":
            kw = dict(targets=r["targets"][None], env2task=np.zeros(1, np.int32))
        for j, i in enumerate(idx[:100]):
            obs, rew, done, fail, _ = qo.env_step(cfg, state, ct, r["act"][i][None], r["task"], r["dt"], r["nt"],
                                                  mode="mix", **kw)
            tol = 2e-6 * (1 + j)
            assert group_rel_err(obs[:, :16], r["obs"][i][None, :16], OBS_GROUPS) < tol
            assert bool(done[0]) == bool(r["done"][i])


def test_f64_arbiter_close_to_mix(quad_golden, cfg):
    r = golden_run(quad_golden, "hover_a")
    for mode, tol in (("f32", 3e-6), ("f64", 3e-6)):
        state = np.array(r["pre_state"], dtype=np.float64)
        ct = np.array(r["pre_ct"], dtype=np.int32)
        qo.env_step(cfg, state, ct, r["act"], r["task"], r["dt"], r["nt"], mode=mode)
        assert group_rel_err(state, r["post_state"], STATE_GROUPS) < tol


def test_velocity_task_tables(quad_golden, cfg):
    """define_velocity_control_task (quadrotorsim.py:306-319) re-derived: seeded actions + float32 integration."""
    from metagym_b200.quadrotor import DEFAULT_SIMULATOR_CONF, velocity_task_actions
    ref = quad_golden["veltask_tables"]
    for seed in range(ref.shape[0]):
        acts = velocity_task_actions(DEFAULT_SIMULATOR_CONF, 40, seed)
        s = qo.zero_state(1)
        for t in range(40):
            qo.sim_step(cfg, s, acts[t][None], 5, "f32")
            assert np.abs(s[0, 3:6] - ref[seed, t]).max() < 1e-5 * max(1.0, np.abs(ref[seed, t]).max())


def test_velocity_task_tables_at_the_benchmarked_size(veltab_golden, cfg):
    """The nt=1000, dt=0.005 tables bench.py's workload flies (reference: define_velocity_control_task(0.005, 1000, seed),
    seeds 0..3, tests/golden/gen_velocity_tables.py).  Asserted against 2x the float32-vs-float64 drift the generator
    measured along the same trajectories (5e-6 at t=999), floor 2e-6."""
    from metagym_b200.quadrotor import DEFAULT_SIMULATOR_CONF, velocity_task_actions
    ref, env = veltab_golden["tables"], veltab_golden["f32_vs_f64_envelope"].max(axis=0)
    for k, seed in enumerate(veltab_golden["seeds"]):
        acts = velocity_task_actions(DEFAULT_SIMULATOR_CONF, 1000, int(seed))
        s = qo.zero_state(1)
        for t in range(1000):
            qo.sim_step(cfg, s, acts[t][None], 5, "f32")
            err = np.abs(s[0, 3:6] - ref[k, t]).max() / max(1.0, np.abs(ref[k, t]).max())
            assert err <= max(2.0 * env[t], 2e-6), (seed, t, err)


def test_failure_detection(cfg):
    s = qo.zero_state(3)
    s[0, 3] = 150.0      # |v| > 100
    s[1, 6] = 2000.0     # |w| > 1000
    s[2, 0] = 1500.0     # |p| > 1000
    _, fail = qo.sim_step(cfg, s, np.full((3, 4), 5, np.float32), 10, "mix")
    assert list(fail) == [2, 3, 1]


@pytest.mark.parametrize("name,np_seed", [("hover_a", 0), ("hover_fall", 2), ("nocol_a", 4), ("vel_a", 5)])
def test_numpy_port_is_bit_identical_to_reference(quad_golden, name, np_seed):
    """oracle/quadrotor_np.py (the CPU baseline of bench.py) replays whole reference episodes, global-RNG resets
    included, to the last bit: it issues the same numpy operations on the same dtypes as the reference."""
    from oracle.quadrotor_np import NumpyQuadrotorEnv
    r = golden_run(quad_golden, name)
    env = NumpyQuadrotorEnv(dt=r["dt"], nt=r["nt"], seed=r["seed"], task=r["task"])
    if r["task"] == "velocity_control":
        assert np.array_equal(np.asarray(env.targets, dtype=np.float32), r["targets"])
    np.random.seed(np_seed)           # tests/golden/gen_quadrotor.py seeds the global RNG once per recorded run
    ep = -1
    for i in range(len(r["rew"])):
        if r["ep"][i] != ep:
            ep = int(r["ep"][i])
            assert np.array_equal(env.reset(), r["reset_obs"][ep])
        obs, rew, done, _ = env.step(r["act"][i])
        assert np.array_equal(obs, r["obs"][i]) and float(rew) == r["rew"][i] and bool(done) == bool(r["done"][i])
        assert np.array_equal(env.st.as_row(), r["post_state"][i])


def test_rk4_restatement_converges_to_the_reference_model(cfg):
    """RK4 has no reference counterpart (parity unpinned, SURVEY.md Q9).  What CAN be checked: the continuous-time
    model integrated by RK4 is the h -> 0 limit of the reference's Euler substeps -- the gap to the substep oracle
    shrinks linearly with its substep, and at 1 ms (the reference's own setting) the reference is ~100x further from
    that limit than RK4 at 5 ms."""
    import copy
    rng = np.random.RandomState(0)
    n, steps, dt = 16, 12, 0.005
    noise = rng.random_sample((n, 12))
    acts = rng.uniform(0.1, 15.0, (steps, n, 4)).astype(np.float32)
    s_rk = qo.reset_state(None, noise)
    for t in range(steps):
        qo.rk4_step(cfg, s_rk, acts[t], dt, 1, "f64")
    gaps = []
    for h in (1e-3, 1e-4, 2e-5):
        p = copy.deepcopy(qo.DEFAULT_PARAMS)
        p["precision"] = h
        c2 = qo.make_cfg(p)
        s = qo.reset_state(None, noise)
        for t in range(steps):
            qo.sim_step(c2, s, acts[t], int(round(dt / h)), "f64")
        gaps.append(group_rel_err(s_rk, s, STATE_GROUPS))
    assert gaps[0] > 5 * gaps[1] > 10 * gaps[2] / 2 and gaps[2] < 5e-4, gaps


@pytest.mark.parametrize("name", QUAD_MAP_RUNS)
def test_obstacle_map_collision_vs_reference(quad_golden, cfg, name):
    """Quadrotor(map_file=...) (env.py:248-260,293-305): with obstacle cells in the swept window the reference compares
    the integer altitude against np.any(...) == True, i.e. it ends the episode at z + 5 < 1.  Teacher-forced steps."""
    r = golden_run(quad_golden, name)
    qo.set_map(quad_golden["map_obst"])
    try:
        state = np.array(r["pre_state"], dtype=np.float64)
        ct = np.array(r["pre_ct"], dtype=np.int32)
        obs, rew, done, fail, power = qo.env_step(cfg, state, ct, r["act"], r["task"], r["dt"], r["nt"], mode="mix")
    finally:
        qo.set_map(None)
    assert np.array_equal(done.astype(bool), r["done"]) and r["done"].sum() >= 2
    assert np.all(r["obs"][r["done"], 15] > 0.9)             # ended above the floor: the obstacle rule fired
    assert scalar_rel_err(rew, r["rew"]) < 1e-6 and np.array_equal(ct, r["post_ct"])
    assert group_rel_err(obs[:, :16], r["obs"][:, :16], OBS_GROUPS) < 1e-6


@pytest.mark.parametrize("name,np_seed", [("map_hover", 11), ("map_nocol", 12)])
def test_numpy_port_with_obstacle_map(quad_golden, name, np_seed):
    from oracle.quadrotor_np import NumpyQuadrotorEnv
    r = golden_run(quad_golden, name)
    env = NumpyQuadrotorEnv(dt=r["dt"], nt=r["nt"], seed=r["seed"], task=r["task"], map_matrix=quad_golden["map_obst"])
    np.random.seed(np_seed)
    ep = -1
    for i in range(len(r["rew"])):
        if r["ep"][i] != ep:
            ep = int(r["ep"][i])
            assert np.array_equal(env.reset(), r["reset_obs"][ep])
        obs, rew, done, _ = env.step(r["act"][i])
        assert np.array_equal(obs, r["obs"][i]) and float(rew) == r["rew"][i] and bool(done) == bool(r["done"][i])


# ---------------------------------------------------------------------------------------------------------------
# non-default simulator config (tests/golden/gen_quadrotor_conf.py): off-diagonal inertia, centre-of-gravity offset,
# CT[2] != 0, an out-of-plane rotor, initial velocities, other voltage range, healthy_reward = 2
# ---------------------------------------------------------------------------------------------------------------
CONF_RUNS = ["c_hover", "c_nocol", "c_vel", "c_spin"]


@pytest.fixture(scope="module")
def conf_golden():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quadrotor_conf_golden.npz"))


@pytest.mark.parametrize("name", CONF_RUNS)
def test_custom_config_teacher_forced(conf_golden, name):
    import json
    params = json.loads(str(conf_golden["conf_json"]))
    ccfg = qo.make_cfg(params)
    r = golden_run(conf_golden, name)
    state = np.array(r["pre_state"], dtype=np.float64)
    ct = np.array(r["pre_ct"], dtype=np.int32)
    n = state.shape[0]
    kw = {}
    if r["task"] == "velocity_control":
        kw = dict(targets=r["targets"][None], env2task=np.zeros(n, np.int32))
    obs, rew, done, fail, power = qo.env_step(ccfg, state, ct, r["act"], r["task"], r["dt"], r["nt"],
                                              healthy=float(conf_golden["healthy_reward"]), mode="mix", **kw)
    assert group_rel_err(state, r["post_state"], STATE_GROUPS) < 1e-6
    assert group_rel_err(obs[:, :16], r["obs"][:, :16], OBS_GROUPS) < 1e-6
    assert scalar_rel_err(rew, r["rew"]) < 1e-6
    assert np.array_equal(done.astype(bool), r["done"]) and np.array_equal(ct, r["post_ct"])
    assert scalar_rel_err(power, r["power"]) < 1e-6 and not fail.any()
    # reset(): the recorded draws through the oracle's reset give the recorded first pre-step state
    s0 = qo.reset_state(params, r["reset_noise"][:1])
    assert group_rel_err(s0, r["pre_state"][:1], STATE_GROUPS) < 1e-7


@pytest.mark.parametrize("name,np_seed", [("c_hover", 21), ("c_nocol", 22), ("c_vel", 23)])
def test_numpy_port_with_custom_config(conf_golden, name, np_seed):
    """The numpy port (CPU baseline) stays bit-identical to the reference under the non-default config."""
    import json
    from oracle.quadrotor_np import NumpyQuadrotorEnv
    params = json.loads(str(conf_golden["conf_json"]))
    r = golden_run(conf_golden, name)
    env = NumpyQuadrotorEnv(dt=r["dt"], nt=r["nt"], seed=r["seed"], task=r["task"], params=params,
                            healthy_reward=float(conf_golden["healthy_reward"]))
    if r["task"] == "velocity_control":
        assert np.array_equal(np.asarray(env.targets, dtype=np.float32), r["targets"])
    np.random.seed(np_seed)
    ep = -1
    for i in range(len(r["rew"])):
        if r["ep"][i] != ep:
            ep = int(r["ep"][i])
            assert np.array_equal(env.reset(), r["reset_obs"][ep])
        obs, rew, done, _ = env.step(r["act"][i])
        assert np.array_equal(obs, r["obs"][i]) and float(rew) == r["rew"][i] and bool(done) == bool(r["done"][i])
        assert np.array_equal(env.st.as_row(), r["post_state"][i])


@pytest.mark.parametrize("general", [False, True])
def test_oracle_batch_reset_rules(general):
    """OracleBatch: episode counters follow the engine's rules, a reset state is float32 and within 1e-7 (relative) of
    reset_state()'s float64 expression, and a subset follows exactly the rows of the whole batch."""
    from oracle import philox
    params = qo.general_params() if general else None
    seed, base, n = (0x0123456789 << 20) | 0xABCDE, 2 ** 32 - 3, 9
    ob = qo.OracleBatch(n, "hovering_control", 0.01, 3, params=params, rng_seed=seed, env_index_base=base,
                        auto_reset=True)
    sub = qo.OracleBatch(n, "hovering_control", 0.01, 3, params=params, rng_seed=seed, env_index_base=base,
                         auto_reset=True, subset=[1, 4, 8])
    assert (ob.ep == 0).all()
    o = ob.reset()
    sub.reset()
    u = philox.quad_reset_draws(seed, base + np.arange(n), np.ones(n, np.int64))
    assert (ob.ep == 1).all() and np.array_equal(ob.state, ob.reset_rows(u))
    assert np.array_equal(ob.state, ob.state.astype(np.float32).astype(np.float64))
    ref = qo.reset_state(params, u)
    assert (np.abs(ob.state - ref) <= 1e-7 * np.maximum(np.abs(ref), 1e-30)).all()
    assert np.array_equal(o[:, 0:3], ob.state[:, 3:6]) and np.array_equal(o[:, 9:12], ob.state[:, 6:9])
    assert (o[:, 3:6] == 0).all() and (o[:, 8] == np.float32(-9.8)).all() and (o[:, 15] == 5.0).all()
    ob.reset(noise=np.full((n, 12), 0.25))
    sub.reset(noise=np.full((n, 12), 0.25))
    assert (ob.ep == 1).all()
    mask = np.arange(n) % 2 == 0
    ob.reset(mask=mask)
    sub.reset(mask=mask)
    assert np.array_equal(ob.ep, np.where(mask, 2, 1)) and np.array_equal(sub.ep, ob.ep[[1, 4, 8]])
    # nt = 3 steps end every episode; the auto-reset draws with ep + 1
    for _ in range(3):
        r = ob.step(np.full((n, 4), 5.0, np.float32))
        rs = sub.step(np.full((n, 4), 5.0, np.float32))
    assert r.done.all() and np.isfinite(r.final_obs).all() and np.array_equal(rs.obs, r.obs[[1, 4, 8]])
    assert np.array_equal(ob.ep, np.where(mask, 3, 2))
    u = philox.quad_reset_draws(seed, base + np.arange(n), ob.ep)
    assert np.array_equal(ob.state, ob.reset_rows(u)) and np.array_equal(sub.state, ob.state[[1, 4, 8]])
    assert np.array_equal(r.obs, ob.reset_obs(np.ones(n, bool)))
