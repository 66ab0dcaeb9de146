"""GPU: whole-episode evaluation (mgb_quad_evaluate, mgb_maze_evaluate; DESIGN.md "Whole-episode evaluation").

Every check runs against twin handles built the same way as the evaluated one:
- one policy rollout of T = B steps that outputs only rew / done / truncated, split into episodes by the float64
  restatement of tests/episode_ref.py: return bit for bit, length and truncated exactly;
- a chain of T = 1 policy rollouts with a snapshot after each: env e's record (and carried state row) after step L_e
  must equal what evaluate left;
- the step counter, populations against member-by-member evaluations on twin handles, value rows, the mean mode, graph
  capture, refusals and one full-size quadrotor run."""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import test_lstm_policy_rollout_maze_gpu as lstm_t  # noqa: E402
import test_policy_rollout_gpu as quad_t  # noqa: E402
import test_policy_rollout_maze_gpu as mlp_t  # noqa: E402
import test_quad_rnn_rollout_gpu as qrnn_t  # noqa: E402
import test_rnn_policy_rollout_maze_gpu as gru_t  # noqa: E402
from episode_ref import split_episodes  # noqa: E402
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = 0x9E3779B97F4A7C15          # both 32-bit halves set
LOG_STD = (-0.5, 0.0, 0.3, -1.0)
NT = 50                            # quadrotor time limit
MAX_STEPS = 45                     # maze time limit
MAZE_N = 9
TRIAL_K = 3


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


# ---------------------------------------------------------------------------------------------------------------
# handles and policies
# ---------------------------------------------------------------------------------------------------------------

def quad_env(n, task="velocity_control", conf=None, base=0, nt=NT):
    """A quadrotor handle a few steps in: ct != 0 (a partial first episode) and t_base != 0."""
    from metagym_b200 import BatchedQuadrotor
    kw = dict(seed=[0, 1, 2]) if task == "velocity_control" else {}
    e = BatchedQuadrotor(task=task, dt=0.005, nt=nt, num_envs=n, device=0, squeeze=False, auto_reset=True,
                         rng_seed=5, env_index_base=base, simulator_conf=conf, **kw)
    e.reset()
    e.rollout(7)
    return e


def quad_policy(env, kind, seed=0, value=False):
    if kind == "mlp":
        from metagym_b200.policy import MLPPolicy
        m = quad_t.make_module(env.obs_dim, (32, 32), nn.Tanh, seed)
        vh = None
        if value:
            vh = nn.Linear(32, 1)
            with torch.no_grad():
                vh.weight.normal_(0, 0.3)
        return MLPPolicy(m, log_std=torch.tensor(LOG_STD), device=env.device, value=vh)
    return qrnn_t.make_policy(env, kind, H=24, width=16 if kind == "gru" else 0, value=value, seed=seed)


def maze_env(n, rec=True, k=TRIAL_K, base=0, table=None):
    """A MetaMaze2D trial handle (one table slot per env) a few steps in."""
    from metagym_b200 import BatchedMetaMaze2D
    e = BatchedMetaMaze2D(max_steps=MAX_STEPS, task_type="SURVIVAL", view_grid=1, num_envs=n, squeeze=False,
                          auto_reset=True, env_index_base=base, record_path=rec, episodes_per_task=k)
    table = table if table is not None else slot_table(MAZE_N, n)[0]
    e.set_task(table, env2task=np.arange(n))
    e.reset()
    e.rollout(3)
    return e


def maze_policy(env, kind, seed=0, value=False):
    vh = None
    if kind == "mlp":
        from metagym_b200.policy import MLPPolicy
        m = mlp_t.make_module(env._obs[0].numel(), (32,), nn.Tanh, seed)
        if value:
            vh = nn.Linear(32, 1)
        return MLPPolicy(m, device=env.device, value=vh)
    make = gru_t.make_policy if kind == "gru" else lstm_t.make_policy
    pol = make(env, 16, 8 if kind == "gru" else 0, nn.Tanh, True, "task", seed=seed)
    if value:       # the same cell and head with a value head
        vh = nn.Linear(pol.head_width or pol.hidden, 1)
        pol = type(pol)(pol._cell, pol._head, feedback=True, hidden_reset="task", device=env.device, value=vh)
    return pol


def initial_state(pol, n, quad):
    from metagym_b200 import GRUPolicy, LSTMPolicy, PolicyPopulation
    if not (isinstance(pol, (GRUPolicy, LSTMPolicy)) or (isinstance(pol, PolicyPopulation) and pol.recurrent)):
        return None
    return (qrnn_t.random_state if quad else gru_t.random_state)(pol, n)


def limit(env):
    return env.nt if hasattr(env, "nt") else env.max_steps


def rs_args(rs):
    return dict(seed=SEED, **CFG) if rs else None


def evaluate(env, pol, episodes, state, rs=False, det=False):
    kw = dict(resample=rs_args(rs)) if not hasattr(env, "nt") else {}
    return env.evaluate(pol, episodes, act_seed=SEED, deterministic=det, state=state, **kw)


def rollout(env, pol, T, state, rs=False, det=False):
    """A policy rollout that outputs only rew / done / truncated."""
    n = env.num_envs
    rew_t = torch.float32 if hasattr(env, "nt") else torch.float64
    out = {"rew": torch.empty((T, n), dtype=rew_t, device=env.device),
           "done": torch.empty((T, n), dtype=torch.uint8, device=env.device),
           "truncated": torch.empty((T, n), dtype=torch.uint8, device=env.device)}
    kw = dict(resample=rs_args(rs)) if not hasattr(env, "nt") else {}
    return env.rollout(T, policy=pol, act_seed=SEED, deterministic=det, state=state, out=out, **kw)


def counter(env):
    lib, c = env._lib, ctypes.c_uint64()
    fn = lib.mgb_quad_counters if hasattr(env, "nt") else lib.mgb_maze_counters
    assert fn(env._h, ctypes.byref(c), 0) == 0
    return c.value


def assert_equal_to_restatement(res, ref, episodes):
    ret, length, trunc, steps = split_episodes(ref["rew"].cpu().numpy(), ref["done"].cpu().numpy(),
                                               ref["truncated"].cpu().numpy(), episodes)
    assert np.array_equal(res["return"].cpu().numpy(), ret)           # bit for bit: float64 == compares exactly
    assert np.array_equal(res["length"].cpu().numpy(), length)
    assert np.array_equal(res["truncated"].cpu().numpy(), trunc)
    return steps


def assert_post_state(evaluated, state, chain, chain_state, pol, steps, rs=False, det=False):
    """Run `chain` as T = 1 rollouts; after step L_e env e's record (and state row) must equal what evaluate left."""
    got = evaluated.snapshot()["records"]
    rec = getattr(evaluated, "record_path", False)
    paths = evaluated.trajectory() if rec else None
    seen = np.zeros(len(steps), bool)
    for t in range(1, int(steps.max()) + 1):
        rollout(chain, pol, 1, chain_state, rs, det)
        here = np.nonzero(steps == t)[0]
        if not len(here):
            continue
        idx = torch.as_tensor(here, device=got.device)
        assert torch.equal(chain.snapshot()["records"][idx], got[idx]), t
        if state is not None:
            assert torch.equal(chain_state[idx], state[idx]), t
        if rec:
            cells, lens = chain.trajectory()
            assert torch.equal(cells[idx], paths[0][idx]) and torch.equal(lens[idx], paths[1][idx]), t
        seen[here] = True
    assert seen.all()


def check_against_twins(make, make_pol, quad, episodes, rs=False, det=False):
    env, twin, chain = make(), make(), make()
    pol = make_pol(env)
    state = initial_state(pol, env.num_envs, quad)
    st_twin = st_chain = None
    if state is not None:
        st_twin, st_chain = state.clone(), state.clone()
    B = episodes * limit(env)
    c0 = counter(env)
    res = evaluate(env, pol, episodes, state, rs, det)
    assert counter(env) == c0 + B
    ref = rollout(twin, pol, B, st_twin, rs, det)
    steps = assert_equal_to_restatement(res, ref, episodes)
    assert_post_state(env, state, chain, st_chain, pol, steps, rs, det)
    return env, pol, state, res


# ---------------------------------------------------------------------------------------------------------------
# 1. equal to the rollout, and 5. the mean mode
# ---------------------------------------------------------------------------------------------------------------

QUAD_CASES = [(kind, task, simple, episodes) for kind in ("mlp", "gru", "lstm")
              for task in ("velocity_control", "hovering_control") for simple in (True, False)
              for episodes in ((1, 3) if kind == "mlp" else (3,))]


@pytest.mark.parametrize("kind,task,simple,episodes", QUAD_CASES,
                         ids=["%s-%s-%s-ep%d" % (k, t, "default" if s else "general", e) for k, t, s, e in QUAD_CASES])
def test_quad_equals_rollout(kind, task, simple, episodes):
    conf = None if simple else qrnn_t.general()
    check_against_twins(lambda: quad_env(200, task, conf), lambda e: quad_policy(e, kind), True, episodes)


MAZE_CASES = [(kind, rs) for kind in ("mlp", "gru", "lstm") for rs in (False, True)]


@pytest.mark.parametrize("kind,rs", MAZE_CASES, ids=["%s-rs%d" % c for c in MAZE_CASES])
@pytest.mark.parametrize("episodes", [1, 3])
def test_maze_equals_rollout(kind, rs, episodes):
    _, _, _, res = check_against_twins(lambda: maze_env(300), lambda e: maze_policy(e, kind), False, episodes, rs)
    assert res["length"].min() < res["length"].max()        # envs stop at different steps


@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm"])
def test_deterministic_mode(kind):
    check_against_twins(lambda: quad_env(200), lambda e: quad_policy(e, kind), True, 2, det=True)
    check_against_twins(lambda: maze_env(300), lambda e: maze_policy(e, kind), False, 2, rs=True, det=True)


def test_consecutive_calls_score_consecutive_episodes():
    # the mean mode draws nothing, so the step counter (which advances by the bound, not by the steps taken) does not
    # enter the results; the auto-reset noise is keyed by each env's episode counter
    a, b = quad_env(200), quad_env(200)
    pol = quad_policy(a, "lstm")
    sa = qrnn_t.random_state(pol, 200)
    sb = sa.clone()
    first, second = evaluate(a, pol, 1, sa, det=True), evaluate(a, pol, 2, sa, det=True)
    both = evaluate(b, pol, 3, sb, det=True)
    assert torch.equal(torch.cat([first["return"], second["return"]]), both["return"])
    assert torch.equal(torch.cat([first["length"], second["length"]]), both["length"])
    assert torch.equal(sa, sb)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])


# ---------------------------------------------------------------------------------------------------------------
# 2. the counter
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
def test_counter_and_a_following_rollout(quad):
    make = (lambda: quad_env(200)) if quad else (lambda: maze_env(300, rec=False))
    env, twin = make(), make()
    pol = quad_policy(env, "mlp") if quad else maze_policy(env, "mlp")
    c0 = counter(env)
    evaluate(env, pol, 2, None)
    assert counter(env) == c0 + 2 * limit(env)
    twin.restore(env.snapshot(), mask=torch.ones(twin.num_envs, dtype=torch.bool))     # a masked restore keeps counters
    assert counter(twin) == c0
    fn = twin._lib.mgb_quad_counters if quad else twin._lib.mgb_maze_counters
    assert fn(twin._h, ctypes.byref(ctypes.c_uint64(c0 + 2 * limit(env))), 1) == 0
    a, b = rollout(env, pol, 30, None), rollout(twin, pol, 30, None)
    for k in ("rew", "done", "truncated"):
        assert torch.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------
# 3. populations
# ---------------------------------------------------------------------------------------------------------------

def assert_same_result(a, b):
    for k in ("return", "length", "truncated"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm"])
def test_one_member_is_the_single_policy(quad, kind):
    from metagym_b200 import PolicyPopulation
    make = (lambda: quad_env(200)) if quad else (lambda: maze_env(300))
    a, b = make(), make()
    pol = quad_policy(a, kind) if quad else maze_policy(a, kind)
    sa = initial_state(pol, a.num_envs, quad)
    sb = sa.clone() if sa is not None else None
    ref = evaluate(a, pol, 2, sa, rs=not quad)
    out = evaluate(b, PolicyPopulation([pol]), 2, sb, rs=not quad)
    assert_same_result(out, ref)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])
    if sa is not None:
        assert torch.equal(sa, sb)


POP_CASES = [(True, "mlp", 64, 4), (True, "gru", 64, 3), (True, "lstm", 128, 2),
             (False, "mlp", 32, 4), (False, "gru", 128, 2), (False, "lstm", 64, 3)]


@pytest.mark.parametrize("quad,kind,E,M", POP_CASES,
                         ids=["%s-%s-E%d-M%d" % ("quad" if q else "maze", k, E, M) for q, k, E, M in POP_CASES])
def test_population_against_twin_handles(quad, kind, E, M):
    from metagym_b200 import PolicyPopulation
    n = E * M
    table = None if quad else [slot_table(MAZE_N, 1)[0][0]] * n     # every slice of the table has the same food cap
    big = quad_env(n) if quad else maze_env(n, table=table)
    pop = PolicyPopulation([quad_policy(big, kind, seed=3 + 7 * m) if quad else maze_policy(big, kind, seed=3 + 7 * m)
                            for m in range(M)])
    state = initial_state(pop, n, quad)
    twin_state = state.clone() if state is not None else None
    out = evaluate(big, pop, 2, state, rs=not quad)
    fitness = out["return"].mean(0).view(M, -1).mean(1)
    recs = big.snapshot()["records"]
    for m in range(M):
        sl = slice(m * E, (m + 1) * E)
        tw = quad_env(E, base=m * E) if quad else maze_env(E, base=m * E, table=table[sl])
        ts = twin_state[sl].clone() if state is not None else None
        ref = evaluate(tw, pop.policies[m], 2, ts, rs=not quad)
        for k in ("return", "length", "truncated"):
            assert torch.equal(out[k][:, sl], ref[k]), (m, k)
        assert fitness[m].item() == ref["return"].mean(0).mean().item()
        mine, twin = recs[sl].clone(), tw.snapshot()["records"]
        if not quad:            # the task slot (bytes 28..31 of a maze record) is local: e here, e - m E on the twin
            assert torch.equal(mine[:, 28:32].view(torch.int32)[:, 0] - m * E, twin[:, 28:32].view(torch.int32)[:, 0])
            mine[:, 28:32] = twin[:, 28:32]
        assert torch.equal(mine, twin), m
        if state is not None:
            assert torch.equal(state[sl], ts), m


# ---------------------------------------------------------------------------------------------------------------
# 4. value rows are skipped
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm"])
def test_value_row_is_skipped(quad, kind):
    make = (lambda: quad_env(200)) if quad else (lambda: maze_env(300))
    a, b = make(), make()
    with_v = quad_policy(a, kind, value=True) if quad else maze_policy(a, kind, value=True)
    assert with_v.has_value
    without = quad_policy(a, kind) if quad else maze_policy(a, kind)     # the same actor, from the same seed
    assert not without.has_value
    sa = initial_state(with_v, a.num_envs, quad)
    sb = sa.clone() if sa is not None else None
    ra = evaluate(a, with_v, 2, sa, rs=not quad)
    rb = evaluate(b, without, 2, sb, rs=not quad)
    assert_same_result(ra, rb)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])


# ---------------------------------------------------------------------------------------------------------------
# 6. graph capture
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
def test_graph_capture_sees_policy_update(quad):
    from metagym_b200.policy import MLPPolicy
    make = (lambda: quad_env(200)) if quad else (lambda: maze_env(300, rec=False))
    env, eager = make(), make()
    D = env.obs_dim if quad else env._obs[0].numel()
    build = quad_t.make_module if quad else mlp_t.make_module
    m0, m1 = build(D, (32, 32), nn.Tanh, 0), build(D, (32, 32), nn.Tanh, 1)
    kw = dict(log_std=torch.tensor(LOG_STD)) if quad else {}
    pol = MLPPolicy(m0, device=env.device, **kw)
    ref_pol = MLPPolicy(m1, device=env.device, **kw)
    snap = env.snapshot()
    evaluate(env, pol, 2, None, rs=not quad)        # warm-up: module load and the shared-memory attribute
    env.restore(snap)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            res = evaluate(env, pol, 2, None, rs=not quad)
    torch.cuda.synchronize()
    env.restore(snap)
    pol.update(module=m1)
    g.replay()
    torch.cuda.synchronize()
    ref = evaluate(eager, ref_pol, 2, None, rs=not quad)
    assert_same_result(res, ref)
    assert torch.equal(env.snapshot()["records"], eager.snapshot()["records"])


# ---------------------------------------------------------------------------------------------------------------
# 7. refusals leave the handle, its counter and the state untouched
# ---------------------------------------------------------------------------------------------------------------

def fingerprint(env):
    lib, w = env._lib, (ctypes.c_uint64 * 4)()
    fn = lib.mgb_quad_fingerprint if hasattr(env, "nt") else lib.mgb_maze_fingerprint
    assert fn(env._h, w) == 0
    return list(w)


@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
def test_refusals_from_c(quad):
    from metagym_b200 import _lib
    env = quad_env(128) if quad else maze_env(128, rec=False)
    mlp = quad_policy(env, "mlp") if quad else maze_policy(env, "mlp")
    gru = quad_policy(env, "gru") if quad else maze_policy(env, "gru")
    n, dev = env.num_envs, env.device
    state = initial_state(gru, n, quad)
    ret = torch.zeros((3, n), dtype=torch.float64, device=dev)
    ln = torch.zeros((3, n), dtype=torch.int32, device=dev)
    tr = torch.zeros((3, n), dtype=torch.uint8, device=dev)
    pm, pr = ctypes.byref(mlp.struct()), ctypes.byref(gru.struct())
    fn = env._lib.mgb_quad_evaluate if quad else env._lib.mgb_maze_evaluate
    cfg = env._sampler_cfg(**CFG)[0] if not quad else None

    def call(episodes=1, m=pm, r=None, value_row=0, members=1, stride=0, st=None, outs=(ret, ln, tr)):
        args = [env._h, episodes, m, r, value_row, members, stride, SEED]
        if not quad:
            args += [ctypes.byref(cfg), SEED]
        return fn(*args, _lib.ptr(st), *[_lib.ptr(o) for o in outs], env._stream())

    big = 2 ** 31 // limit(env) + 1
    refusals = {"episodes 0": dict(episodes=0), "episodes -1": dict(episodes=-1), "B > 2^31 - 1": dict(episodes=big),
                "both": dict(r=pr, st=state), "neither": dict(m=None), "rnn without state": dict(m=None, r=pr),
                "mlp with state": dict(st=state), "value_row 2": dict(value_row=2), "value_row -1": dict(value_row=-1),
                "null return": dict(outs=(None, ln, tr)), "null length": dict(outs=(ret, None, tr)),
                "null truncated": dict(outs=(ret, ln, None)), "population E": dict(members=3, stride=mlp.numel),
                "short stride": dict(members=2, stride=1)}
    st0, fp0, c0, rec0 = state.clone(), fingerprint(env), counter(env), env.snapshot()["records"]
    for what, kw in refusals.items():
        assert call(**kw) == MGB_ERR_ARG, what
        torch.cuda.synchronize()
        assert fingerprint(env) == fp0 and counter(env) == c0, what
        assert torch.equal(env.snapshot()["records"], rec0) and torch.equal(state, st0), what
        assert not ret.any() and not ln.any() and not tr.any(), what
    # auto_reset off (quad_env's rng_seed is 5)
    opt = env._lib.mgb_quad_set_options if quad else env._lib.mgb_maze_set_options
    assert (opt(env._h, 0, 5) if quad else opt(env._h, 0)) == 0
    assert call() == MGB_ERR_ARG
    assert (opt(env._h, 1, 5) if quad else opt(env._h, 1)) == 0
    # output mirrors, then multicast (set on the handle only: the refused call launches nothing)
    pre = "mgb_quad" if quad else "mgb_maze"
    mir, mc = getattr(env._lib, pre + "_set_mirrors"), getattr(env._lib, pre + "_set_multicast")
    assert mir(env._h, 1, (ctypes.c_int64 * 1)(1 << 20)) == 0
    assert call() == MGB_ERR_ARG
    assert mir(env._h, 0, None) == 0
    assert mc(env._h, 1 << 20) == 0
    assert call() == MGB_ERR_ARG
    assert mc(env._h, 0) == 0
    torch.cuda.synchronize()
    assert counter(env) == c0 and fingerprint(env) == fp0
    assert torch.equal(env.snapshot()["records"], rec0) and not ret.any()
    assert call() == 0              # and the same call with nothing wrong runs


def test_maze_3d_refused():
    from metagym_b200 import BatchedMetaMazeDiscrete3D, _lib
    from metagym_b200.textures import synthetic_textures
    env = BatchedMetaMazeDiscrete3D(resolution=(16, 16), max_steps=MAX_STEPS, num_envs=32, squeeze=False,
                                    textures=synthetic_textures(seed=0))
    env.set_task(slot_table(MAZE_N, 1)[0][0])
    env.reset()
    pol = maze_policy(maze_env(32, rec=False), "mlp")
    out = [torch.zeros((1, 32), dtype=d, device="cuda") for d in (torch.float64, torch.int32, torch.uint8)]
    c0 = counter(env)
    assert env._lib.mgb_maze_evaluate(env._h, 1, ctypes.byref(pol.struct()), None, 0, 1, 0, SEED, None, 0, None,
                                      *[_lib.ptr(o) for o in out], env._stream()) == MGB_ERR_ARG
    assert counter(env) == c0
    assert not hasattr(env, "evaluate")


@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
def test_refusals_from_python(quad):
    from metagym_b200 import PolicyPopulation
    env = quad_env(128) if quad else maze_env(128, rec=False)
    mlp = quad_policy(env, "mlp") if quad else maze_policy(env, "mlp")
    gru = quad_policy(env, "gru") if quad else maze_policy(env, "gru")
    state = initial_state(gru, env.num_envs, quad)
    st0, fp0, c0, rec0 = state.clone(), fingerprint(env), counter(env), env.snapshot()["records"]
    bad = [lambda: env.evaluate(mlp, 0), lambda: env.evaluate(mlp, 2 ** 31 // limit(env) + 1),
           lambda: env.evaluate(gru), lambda: env.evaluate(mlp, state=state),
           lambda: env.evaluate(gru, state=state[:-1]), lambda: env.evaluate(gru, state=state.double()),
           lambda: env.evaluate(PolicyPopulation.from_template(mlp, 3), state=None)]
    if quad:
        from metagym_b200.policy import MLPPolicy
        bad.append(lambda: env.evaluate(MLPPolicy(quad_t.make_module(env.obs_dim), device=env.device)))
    for f in bad:
        with pytest.raises(ValueError):
            f()
    assert fingerprint(env) == fp0 and counter(env) == c0
    assert torch.equal(env.snapshot()["records"], rec0) and torch.equal(state, st0)
    # output mirrors, then multicast, set on the handle: the library refuses (set only on the handle, nothing launches)
    from metagym_b200 import MgbError
    for on, off in ((lambda: env.set_mirrors([1 << 20]), lambda: env.set_mirrors([])),
                    (lambda: env.set_multicast(1 << 20), lambda: env.set_multicast(0))):
        on()
        for f in (lambda: env.evaluate(mlp, 2), lambda: env.evaluate(gru, 2, state=state)):
            with pytest.raises(MgbError, match="mirrors"):
                f()
        off()
    torch.cuda.synchronize()
    assert fingerprint(env) == fp0 and counter(env) == c0
    assert torch.equal(env.snapshot()["records"], rec0) and torch.equal(state, st0)


@pytest.mark.parametrize("quad", [True, False], ids=["quad", "maze"])
def test_auto_reset_off_refused_from_python(quad):
    from metagym_b200 import BatchedMetaMaze2D, BatchedQuadrotor, MgbError
    if quad:
        env = BatchedQuadrotor(task="velocity_control", dt=0.005, nt=NT, seed=[0, 1, 2], num_envs=128, device=0,
                               squeeze=False, auto_reset=False, rng_seed=5)
    else:
        env = BatchedMetaMaze2D(max_steps=MAX_STEPS, view_grid=1, num_envs=128, squeeze=False, auto_reset=False)
        env.set_task(slot_table(MAZE_N, 128)[0], env2task=np.arange(128))
    env.reset()
    mlp = quad_policy(env, "mlp") if quad else maze_policy(env, "mlp")
    gru = quad_policy(env, "gru") if quad else maze_policy(env, "gru")
    state = initial_state(gru, env.num_envs, quad)
    st0, fp0, c0, rec0 = state.clone(), fingerprint(env), counter(env), env.snapshot()["records"]
    for f in (lambda: env.evaluate(mlp, 2), lambda: env.evaluate(gru, 2, state=state)):
        with pytest.raises(MgbError, match="auto_reset"):
            f()
    torch.cuda.synchronize()
    assert fingerprint(env) == fp0 and counter(env) == c0
    assert torch.equal(env.snapshot()["records"], rec0) and torch.equal(state, st0)


# ---------------------------------------------------------------------------------------------------------------
# 8. full size, once
# ---------------------------------------------------------------------------------------------------------------

def test_full_size_quadrotor():
    from metagym_b200 import BatchedQuadrotor
    from metagym_b200.policy import MLPPolicy
    n, nt = 65536, 1000
    envs = []
    for _ in range(2):
        e = BatchedQuadrotor(task="velocity_control", dt=0.005, nt=nt, seed=[0, 1, 2, 3], num_envs=n, device=0,
                             squeeze=False, auto_reset=True, rng_seed=11)
        e.reset()
        envs.append(e)
    pol = MLPPolicy(quad_t.make_module(19, (64, 64), nn.Tanh, 0), log_std=torch.tensor(LOG_STD), device=envs[0].device)
    res = envs[0].evaluate(pol, 1, act_seed=SEED)
    ref = rollout(envs[1], pol, nt, None)
    assert_equal_to_restatement(res, ref, 1)
