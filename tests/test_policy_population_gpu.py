"""GPU: policy populations (DESIGN.md "Populations").  One launch drives each block of E = N / M envs with its own
member, and every output of member m's block must equal, bit for bit, what a handle of those E envs alone (env_index_base
m E, the same tasks) computes with member m through the single-policy path.  Also: members = 1 against the existing
entry points, identical members against the single policy, locality of a perturbed row, the refusals with nothing
touched, graph capture of a write into pop.params, and unroll() against the kernel's log-probabilities."""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import test_lstm_policy_rollout_maze_gpu as lstm_t  # noqa: E402
import test_policy_rollout_gpu as quad_t  # noqa: E402
import test_policy_rollout_maze_gpu as mlp_t  # noqa: E402
import test_rnn_policy_rollout_maze_gpu as gru_t  # noqa: E402
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_policy_rollout_matrix_gpu import LOG_STD, MATRIX, SEED, Shape, mlp_staged, smem_bytes  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
MAZE_N = 9


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def maze_env(n, shape, rec=False, fin=True, base=0, table=None, k=None):
    from metagym_b200 import BatchedMetaMaze2D
    e = BatchedMetaMaze2D(max_steps=mlp_t.MAX_STEPS, task_type=shape.task_type, view_grid=shape.view_grid, num_envs=n,
                          squeeze=False, auto_reset=True, final_obs=fin, env_index_base=base, record_path=rec,
                          episodes_per_task=k)
    table = table if table is not None else food_table(n)
    e.set_task(table, env2task=np.arange(n))
    e.reset()
    e.rollout(3)                         # t_base != 0
    return e


def food_table(n):
    """One slot per env, every task with food, so that every slice of the table has the same food cap (the sampler
    draws food up to the table's cap, and a twin handle holds a slice)."""
    return [slot_table(MAZE_N, 1)[0][0]] * n


def members(shape, env, M, seed=0):
    return [shape.policy(env, seed=seed + 7 * m)[1] for m in range(M)]


def run_maze(shape, env, pol, T, state, rs):
    rs = dict(seed=SEED, **CFG) if rs else None
    if shape.kind == "mlp":
        return env.rollout(T, policy=pol, act_seed=SEED, resample=rs)
    return env.rollout(T, policy=pol, state=state, act_seed=SEED, resample=rs, want_hidden=True)


def assert_same(a, b, what=""):
    """Every entry equal; final_obs on the rows where done (the others are never written)."""
    assert set(a) == set(b), (what, set(a) ^ set(b))
    for k in a:
        if k == "final_obs":
            d = a["done"].bool()
            assert torch.equal(a[k][d], b[k][d]), (what, k)
        elif isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), (what, k)
        else:
            assert a[k] == b[k], (what, k)


def env_state(env):
    return [x.clone() for x in env.agent_state()]


# ---------------------------------------------------------------------------------------------------------------
# 1. members = 1 is the existing call, bit for bit
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,fin,rec,rs,shape", MATRIX,
                         ids=["%s-fin%d-rec%d-rs%d" % (k, f, r, s) for k, f, r, s, _ in MATRIX])
def test_maze_one_member_is_the_single_policy(kind, fin, rec, rs, shape):
    from metagym_b200 import PolicyPopulation
    n, T = 300, 20
    a, b = maze_env(n, shape, rec, bool(fin)), maze_env(n, shape, rec, bool(fin))
    pol = members(shape, a, 1)[0]
    sa = sb = None
    if kind != "mlp":
        sa = gru_t.random_state(pol, n)
        sb = sa.clone()
    ref = run_maze(shape, a, pol, T, sa, rs)
    pop = PolicyPopulation([pol])
    out = run_maze(shape, b, pop, T, sb, rs)
    assert_same(out, ref)
    if kind != "mlp":
        assert torch.equal(sa, sb)
    for x, y in zip(env_state(a), env_state(b)):
        assert torch.equal(x, y)
    if rec:
        for x, y in zip(a.trajectory(), b.trajectory()):
            assert torch.equal(x, y)


def quad_env(n, task="velocity_control", base=0, fin=True, conf=None):
    from metagym_b200 import BatchedQuadrotor
    kw = dict(seed=[0, 1, 2]) if task == "velocity_control" else {}
    e = BatchedQuadrotor(task=task, dt=0.005, nt=20, num_envs=n, device=0, squeeze=False, auto_reset=True,
                         final_obs=fin, rng_seed=5, env_index_base=base, simulator_conf=conf, **kw)
    e.reset()
    e.rollout(5)
    return e


def quad_members(env, M, widths=(64, 64), seed=0):
    return [quad_t.make_policy(env, widths, nn.Tanh, seed + 7 * m, LOG_STD)[1] for m in range(M)]


@pytest.mark.parametrize("fin", [False, True], ids=["fin0", "fin1"])
@pytest.mark.parametrize("simple", [True, False], ids=["default", "general"])
def test_quad_one_member_is_the_single_policy(simple, fin):
    from metagym_b200 import PolicyPopulation
    from oracle import quad_oracle as qo
    conf = None if simple else qo.general_params()
    task = "velocity_control" if fin else "hovering_control"
    a, b = quad_env(300, task, fin=fin, conf=conf), quad_env(300, task, fin=fin, conf=conf)
    pol = quad_members(a, 1)[0]
    ref = a.rollout(32, policy=pol, act_seed=SEED)
    out = b.rollout(32, policy=PolicyPopulation([pol]), act_seed=SEED)
    assert ref["done"].any()
    assert_same(out, ref)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])


# ---------------------------------------------------------------------------------------------------------------
# 2. identical members equal the single policy, E below and above the CTA
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm"])
@pytest.mark.parametrize("E", [32, 256])
def test_maze_identical_members(kind, E):
    from metagym_b200 import PolicyPopulation
    shape = {"mlp": Shape("mlp", (17, 64)), "gru": Shape("gru", H=17, width=5), "lstm": Shape("lstm", H=8, width=33)}[kind]
    n = 512
    a, b = maze_env(n, shape), maze_env(n, shape)
    pol = members(shape, a, 1)[0]
    sa = sb = None
    if kind != "mlp":
        sa = gru_t.random_state(pol, n)
        sb = sa.clone()
    ref = run_maze(shape, a, pol, 24, sa, True)
    out = run_maze(shape, b, PolicyPopulation.from_template(pol, n // E), 24, sb, True)
    assert_same(out, ref)
    if kind != "mlp":
        assert torch.equal(sa, sb)


@pytest.mark.parametrize("E", [32, 128])
def test_quad_identical_members(E):
    from metagym_b200 import PolicyPopulation
    a, b = quad_env(512), quad_env(512)
    pol = quad_members(a, 1)[0]
    ref = a.rollout(32, policy=pol, act_seed=SEED)
    out = b.rollout(32, policy=PolicyPopulation.from_template(pol, 512 // E), act_seed=SEED)
    assert_same(out, ref)


# ---------------------------------------------------------------------------------------------------------------
# 3. twin handles: member m's block against a handle of its E envs alone
# ---------------------------------------------------------------------------------------------------------------

TWIN_SHAPES = {"mlp": Shape("mlp", (33, 17)), "gru": Shape("gru", H=17, width=13, reset="task"),
               "lstm": Shape("lstm", H=8, width=5, reset="task")}
KINDS = ("mlp", "gru", "lstm")
TWINS = ([(kind, E, M, False, None, True) for kind in KINDS for E, M in ((32, 6), (64, 4), (128, 3), (256, 2))]
         + [(kind, 32, 3, False, None, True) for kind in ("mlp", "lstm")]     # n = 96: one partial CTA of 3 members
         + [(kind, E, M, True, 2, True) for kind in KINDS for E, M in ((32, 6), (256, 2))]
         # without resampling: the RS-off instantiations, with and without path recording
         + [(kind, E, M, rec, None, False) for kind in KINDS for E, M, rec in ((32, 4, False), (64, 2, True),
                                                                              (32, 3, True), (256, 2, False))])


@pytest.mark.parametrize("kind,E,M,rec,k,rs", TWINS, ids=["%s-E%d-M%d-rec%d-k%s-rs%d" % t for t in TWINS])
def test_maze_twin_handles(kind, E, M, rec, k, rs):
    from metagym_b200 import PolicyPopulation
    shape = TWIN_SHAPES[kind]
    n, T = E * M, 24
    table = food_table(n)
    big = maze_env(n, shape, rec=rec, table=table, k=k)
    pop = PolicyPopulation(members(shape, big, M, seed=3))
    state = gru_t.random_state(pop, n) if kind != "mlp" else None
    twins_state = state.clone() if state is not None else None
    out = run_maze(shape, big, pop, T, state, rs)
    assert out["done"].any()
    st_big = env_state(big)
    for m in range(M):
        tw = maze_env(E, shape, rec=rec, base=m * E, table=table[m * E:(m + 1) * E], k=k)
        ts = twins_state[m * E:(m + 1) * E].clone() if state is not None else None
        ref = run_maze(shape, tw, pop.policies[m], T, ts, rs)
        assert_same(pop.member_slice(out, m), ref, "member %d" % m)
        if state is not None:
            assert torch.equal(pop.member_slice(state, m), ts)
        for x, y in zip(st_big, env_state(tw)):
            assert torch.equal(x[m * E:(m + 1) * E], y), m
        if rec:
            for x, y in zip(big.trajectory(), tw.trajectory()):
                assert torch.equal(x[m * E:(m + 1) * E], y), m
        if k is not None:
            assert torch.equal(big.task_episodes[m * E:(m + 1) * E], tw.task_episodes)
        tw.close()
    big.close()


@pytest.mark.parametrize("E", [32, 64, 128])
def test_quad_twin_handles(E):
    from metagym_b200 import PolicyPopulation
    M = 4
    n = E * M
    big = quad_env(n)
    pop = PolicyPopulation(quad_members(big, M, widths=(64, 17), seed=3))
    out = big.rollout(32, policy=pop, act_seed=SEED)
    assert out["done"].any()
    for m in range(M):
        tw = quad_env(E, base=m * E)
        ref = tw.rollout(32, policy=pop.policies[m], act_seed=SEED)
        assert_same(pop.member_slice(out, m), ref, "member %d" % m)
        tw.close()
    big.close()


# ---------------------------------------------------------------------------------------------------------------
# 4. locality: a perturbed row moves only its member's block
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,E", [("mlp", 32), ("lstm", 64), ("gru", 256)])
def test_maze_locality(kind, E):
    from metagym_b200 import PolicyPopulation
    shape = TWIN_SHAPES[kind]
    M, T = 4, 24
    n = E * M
    outs = []
    for perturb in (False, True):
        env = maze_env(n, shape)
        pop = PolicyPopulation.from_template(members(shape, env, 1)[0], M)
        if perturb:
            pop.params[2] += 0.5 * torch.randn(pop.numel, generator=torch.Generator().manual_seed(1)).to(pop.device)
        state = gru_t.random_state(pop, n) if kind != "mlp" else None
        outs.append(run_maze(shape, env, pop, T, state, False))
        env.close()
    for m in range(M):
        a, b = pop.member_slice(outs[0], m), pop.member_slice(outs[1], m)
        same = all(torch.equal(a[x], b[x]) for x in ("act", "logp", "obs"))
        assert same == (m != 2), m


@pytest.mark.parametrize("E", [32, 64])
def test_quad_locality(E):
    from metagym_b200 import PolicyPopulation
    M = 4
    outs = []
    for perturb in (False, True):
        env = quad_env(E * M)
        pop = PolicyPopulation.from_template(quad_members(env, 1)[0], M)
        if perturb:
            pop.params[1, :100] += 0.3
        outs.append(env.rollout(16, policy=pop, act_seed=SEED))
        env.close()
    for m in range(M):
        a, b = pop.member_slice(outs[0], m), pop.member_slice(outs[1], m)
        assert torch.equal(a["act"], b["act"]) == (m != 1), m


# ---------------------------------------------------------------------------------------------------------------
# 5. refusals, with the handle, its step counter and the state untouched
# ---------------------------------------------------------------------------------------------------------------

def rnn_staged(kind, D, H, width, feedback=True):
    NG = 3 if kind == "gru" else 4
    Hp, n_in = (H + 7) // 8 * 8, D + 5 * feedback
    return NG * Hp * n_in + NG * Hp * H + 2 * NG * Hp + mlp_staged(H, (width,) if width else ())


def lstm_pop_bytes(view_grid, H, width, copies, threads=128):
    """A population CTA of the LSTM: the two tiles, `copies` staged members, and the columns x, c, h0, h1."""
    D = (2 * view_grid + 1) ** 2
    n_in, Hr = D + 5, max(H, width)
    return 2 * threads * D * 4 + (rnn_staged("lstm", D, H, width) * copies + (n_in + H + 2 * Hr) * threads) * 4


def test_refusals_leave_everything_untouched():
    from metagym_b200 import MgbError, PolicyPopulation, _lib
    lib = _lib.load()
    shape = Shape("lstm", H=8, width=5)
    n = 256
    env = maze_env(n, shape)
    pol = members(shape, env, 1)[0]
    pop = PolicyPopulation.from_template(pol, 4)
    state = gru_t.random_state(pol, n)
    before, counters, st = state.clone(), env._counters(), env_state(env)
    st_pol = pop.struct()

    def call(members, stride, struct=st_pol):
        return lib.mgb_maze_rollout_rnn_population(env._h, 4, ctypes.byref(struct), members, stride, SEED, None, 0,
                                                   state.data_ptr(), None, None, None, None, None, None, None, None,
                                                   None, None, env._stream())

    for members_, stride, why in ((0, pop.numel, "members must be at least 1"),
                                  (3, pop.numel, "multiple of members"),
                                  (16, pop.numel, "envs per member"),             # E = 16
                                  (4, pop.numel - 1, "member_stride is shorter")):
        assert call(members_, stride) == MGB_ERR_ARG
        assert why in lib.mgb_last_error().decode()
    env2 = maze_env(96 * 2, shape)                       # E = 96: neither divides 128 nor is a multiple of it
    s2 = gru_t.random_state(pol, 192)
    rc = lib.mgb_maze_rollout_rnn_population(env2._h, 4, ctypes.byref(st_pol), 2, pop.numel, SEED, None, 0,
                                             s2.data_ptr(), None, None, None, None, None, None, None, None, None, None,
                                             env2._stream())
    assert rc == MGB_ERR_ARG and "envs per member" in lib.mgb_last_error().decode()
    with pytest.raises(ValueError, match="envs per member"):
        env2.rollout(4, policy=PolicyPopulation.from_template(pol, 2), state=s2)
    env2.close()
    torch.cuda.synchronize()
    assert torch.equal(state, before) and env._counters() == counters
    for x, y in zip(st, env_state(env)):
        assert torch.equal(x, y)
    # the footprint of H = 48 at view_grid 1: two members per CTA (E = 64) fit, four (E = 32) are refused
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    big = Shape("lstm", H=48, width=0)
    assert lstm_pop_bytes(1, 48, 0, 2) <= optin < lstm_pop_bytes(1, 48, 0, 4)
    e3 = maze_env(128, big)
    p3 = members(big, e3, 1)[0]
    s3 = gru_t.random_state(p3, 128)
    out = e3.rollout(4, policy=PolicyPopulation.from_template(p3, 2), state=s3)
    assert out["done"].shape == (4, 128)
    s_before, cnt = s3.clone(), e3._counters()
    with pytest.raises(MgbError, match="needs %d bytes of shared memory" % lstm_pop_bytes(1, 48, 0, 4)):
        e3.rollout(4, policy=PolicyPopulation.from_template(p3, 4), state=s3)
    torch.cuda.synchronize()
    assert torch.equal(s3, s_before) and e3._counters() == cnt
    e3.close()
    env.close()


def test_python_refusals():
    from metagym_b200 import PolicyPopulation
    q = quad_env(128)
    pol = quad_members(q, 1)[0]
    with pytest.raises(ValueError, match="envs per member"):
        q.rollout(4, policy=PolicyPopulation.from_template(pol, 8))          # E = 16
    with pytest.raises(ValueError, match="multiple of it"):
        q.rollout(4, policy=PolicyPopulation.from_template(pol, 3))
    q.close()


def test_quad_short_stride_leaves_everything_untouched():
    """The quadrotor's packed length includes the 4 log_std floats, so numel - 1 is one float short."""
    from metagym_b200 import PolicyPopulation, _lib
    lib = _lib.load()
    q = quad_env(128)
    pop = PolicyPopulation.from_template(quad_members(q, 1)[0], 4)
    snap = q.snapshot()["records"].clone()
    counters = q._counters()
    st = pop.struct()
    act = torch.zeros((4, 128, 4), device=q.device)
    for members_, stride, why in ((4, pop.numel - 1, "member_stride is shorter"), (0, pop.numel, "at least 1"),
                                  (3, pop.numel, "multiple of members"), (8, pop.numel, "envs per member")):
        rc = lib.mgb_quad_rollout_population(q._h, 4, ctypes.byref(st), members_, stride, SEED, act.data_ptr(), None,
                                             None, None, None, None, None, None, q._stream())
        assert rc == MGB_ERR_ARG and why in lib.mgb_last_error().decode(), members_
    torch.cuda.synchronize()
    assert torch.equal(act, torch.zeros_like(act)) and q._counters() == counters
    assert torch.equal(q.snapshot()["records"], snap)
    assert lib.mgb_quad_rollout_population(q._h, 4, ctypes.byref(st), 4, pop.numel, SEED, act.data_ptr(), None, None,
                                           None, None, None, None, None, q._stream()) == 0
    q.close()


def test_maze_mlp_refusals_leave_everything_untouched():
    """mgb_maze_rollout_population: a short stride, and the footprint of (64, 64, 64) at view_grid 4, where one staged
    member fits and two (E = 64) are refused with the byte count restated in Python."""
    from metagym_b200 import MgbError, PolicyPopulation, _lib
    lib = _lib.load()
    shape = Shape("mlp", (64, 64, 64), view_grid=4)
    env = maze_env(128, shape)
    pol = members(shape, env, 1)[0]
    D = pol.obs_dim
    two = smem_bytes("mlp", 4, widths=(64, 64, 64)) + mlp_staged(D, (64, 64, 64)) * 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert smem_bytes("mlp", 4, widths=(64, 64, 64)) <= optin < two
    counters, st = env._counters(), env_state(env)
    pop = PolicyPopulation.from_template(pol, 2)
    rc = lib.mgb_maze_rollout_population(env._h, 4, ctypes.byref(pop.struct()), 2, pop.numel - 5, SEED, None, 0,
                                         *[None] * 8, env._stream())
    assert rc == MGB_ERR_ARG and "member_stride is shorter" in lib.mgb_last_error().decode()
    with pytest.raises(MgbError, match="needs %d bytes of shared memory" % two):
        env.rollout(4, policy=pop)
    torch.cuda.synchronize()
    assert env._counters() == counters
    for x, y in zip(st, env_state(env)):
        assert torch.equal(x, y)
    out = env.rollout(4, policy=PolicyPopulation.from_template(pol, 1))
    assert out["done"].shape == (4, 128)
    env.close()


# ---------------------------------------------------------------------------------------------------------------
# 6. graph capture sees writes into pop.params; 7. unroll
# ---------------------------------------------------------------------------------------------------------------

def test_graph_capture_sees_new_params():
    from metagym_b200 import PolicyPopulation
    shape = TWIN_SHAPES["gru"]
    n, M, T = 256, 8, 16
    a, b = maze_env(n, shape), maze_env(n, shape)
    pop = PolicyPopulation(members(shape, a, M))
    sa = gru_t.random_state(pop, n)
    sb = sa.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        snap = a.snapshot()
        run_maze(shape, a, pop, T, sa, False)                     # warm-up outside the capture
        a.restore(snap)
        sa.copy_(sb)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = run_maze(shape, a, pop, T, sa, False)
    torch.cuda.synchronize()
    new = pop.params + 0.1 * torch.randn(pop.params.shape, generator=torch.Generator().manual_seed(2)).to(pop.device)
    a.restore(snap)
    sa.copy_(sb)
    pop.params.copy_(new)
    g.replay()
    torch.cuda.synchronize()
    ref_pop = PolicyPopulation(members(shape, b, M))
    ref_pop.params.copy_(new)
    ref = run_maze(shape, b, ref_pop, T, sb, False)
    for k in ("obs", "rew", "done", "act", "logp", "hid"):
        assert torch.equal(out[k], ref[k]), k
    assert torch.equal(sa, sb)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_unroll_agrees_with_the_kernel(kind):
    from metagym_b200 import PolicyPopulation
    shape = TWIN_SHAPES[kind]
    n, M = 256, 4
    env = maze_env(n, shape)
    pop = PolicyPopulation(members(shape, env, M, seed=11))
    state = pop.initial_state(n)
    out = run_maze(shape, env, pop, 24, state, True)
    _, logp = pop.unroll(out)
    err = (logp.double().cpu() - out["logp"].double().cpu()).abs().max().item()
    assert err < 1e-4, err           # the bound of the single-policy unroll test
    env.close()
