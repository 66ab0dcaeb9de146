"""GPU: value heads and GAE in the policy rollouts (DESIGN.md "Value heads and GAE").

A policy with a value head must leave every other output bit-identical to the same policy without one; value must lie
within the float32 error bound of a float64 reference (teacher-forced on the kernel's h_t for the cells); value_last
must be the next launch's value[0] bit for bit; final_value must be written exactly where the cut fires on a truncated
step, and match the float64 terminal value from the memory before the wipe; adv and ret must equal the float32 NumPy
restatement bit for bit.  Also: population twins, graph capture of a write into the value row, and the refusals."""
import ctypes
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import test_lstm_policy_rollout_maze_gpu as lstm_t  # noqa: E402
import test_policy_rollout_gpu as quad_t  # noqa: E402
import test_rnn_policy_rollout_maze_gpu as gru_t  # noqa: E402
from critic_ref import gae_f32  # noqa: E402
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402
from test_policy_rollout_matrix_gpu import LOG_STD, SEED, Shape  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
U = 2.0 ** -24
GAE = (0.97, 0.9)
MAX_STEPS = 9           # short episodes: truncations within a launch


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def maze_env(n, shape, base=0, k=None, auto_reset=True):
    from metagym_b200 import BatchedMetaMaze2D
    e = BatchedMetaMaze2D(max_steps=MAX_STEPS, task_type=shape.task_type, view_grid=shape.view_grid, num_envs=n,
                          squeeze=False, auto_reset=auto_reset, final_obs=auto_reset, env_index_base=base,
                          episodes_per_task=k)
    e.set_task([slot_table(9, 1)[0][0]] * n, env2task=np.arange(n))
    e.reset()
    e.rollout(3)                         # t_base != 0
    return e


def quad_env(n, task="velocity_control", base=0):
    from metagym_b200 import BatchedQuadrotor
    kw = dict(seed=[0, 1, 2]) if task == "velocity_control" else {}
    e = BatchedQuadrotor(task=task, dt=0.005, nt=11, num_envs=n, device=0, squeeze=False, auto_reset=True,
                         final_obs=True, rng_seed=5, env_index_base=base, **kw)
    e.reset()
    e.rollout(5)
    return e


def value_layer(k, seed, device):
    g = torch.Generator().manual_seed(1000 + seed)
    v = nn.Linear(k, 1)
    with torch.no_grad():
        v.weight.copy_(torch.randn(v.weight.shape, generator=g) / k ** 0.5)
        v.bias.copy_(torch.randn(1, generator=g))
    return v


def with_value(pol, seed=0):
    """The same policy (the same torch modules) with a value head."""
    from metagym_b200.policy import MLPPolicy
    if isinstance(pol, MLPPolicy):
        k = pol.widths[-1] if pol.widths else pol.obs_dim
        return MLPPolicy(pol._module, log_std=pol._log_std, obs_mean=pol._mean, obs_std=pol._std, device=pol.device,
                         value=value_layer(k, seed, pol.device))
    k = pol.head_width or pol.hidden
    return type(pol)(pol._cell, pol._head, feedback=pol.feedback, hidden_reset=pol.hidden_reset, device=pol.device,
                     value=value_layer(k, seed, pol.device))


def run(env, pol, T, state=None, rs=False, gae=None, out=None):
    rs = dict(seed=SEED, **CFG) if rs else None
    kw = dict(state=state, want_hidden=True) if state is not None else {}
    return env.rollout(T, policy=pol, act_seed=SEED, resample=rs, gae=gae, out=out, **kw)


def nan_out(ref, T, N, dev):
    """An out dict shaped like `ref` whose final_value starts as NaN."""
    out = {k: (torch.empty_like(v) if isinstance(v, torch.Tensor) else v) for k, v in ref.items()}
    out["final_value"] = torch.full((T, N), float("nan"), device=dev)
    return out


def cut_mask(pol, out):
    from metagym_b200.metamaze import new_tasks
    if getattr(pol, "hidden_reset", "episode") == "task":
        return new_tasks(out).bool() & out["done"].bool()
    return out["done"].bool()


def assert_rest_equal(a, b):
    """Every output of the value-less rollout `a` equals that of `b`; final_obs where done."""
    for k, v in a.items():
        if k == "final_obs":
            d = a["done"].bool()
            assert torch.equal(v[d], b[k][d]), k
        elif isinstance(v, torch.Tensor):
            assert torch.equal(v, b[k]), k
        else:
            assert v == b[k], k


def check_gae(pol, out):
    cut = cut_mask(pol, out).cpu().numpy()
    adv, ret = gae_f32(out["rew"].cpu().numpy(), cut, out["truncated"].cpu().numpy(), out["value"].cpu().numpy(),
                       out["value_last"].cpu().numpy(), out["final_value"].cpu().numpy(), *GAE)
    assert np.array_equal(out["adv"].cpu().numpy(), adv)
    assert np.array_equal(out["ret"].cpu().numpy(), ret)


def check_final_written(pol, out):
    """final_value is written exactly where cut & truncated (NaN elsewhere); returns that mask."""
    where = cut_mask(pol, out) & out["truncated"].bool()
    fv = out["final_value"]
    assert not torch.isnan(fv[where]).any()
    assert torch.isnan(fv[~where]).all()
    return where


def bound_from(module, x, err):
    """forward_bound with an input error `err` (1-Lipschitz activations; tanhf adds 2 ulp)."""
    h, e = x, err
    mods = list(module)
    for k in range(0, len(mods), 2):
        lin = mods[k]
        W, b = lin.weight.detach().double().to(x.device), lin.bias.detach().double().to(x.device)
        y = h @ W.T + b
        e = (lin.in_features + 1) * U * (h.abs() @ W.abs().T + b.abs()) + e @ W.abs().T
        if k + 1 < len(mods):
            y = torch.tanh(y) if isinstance(mods[k + 1], nn.Tanh) else torch.relu(y)
            if isinstance(mods[k + 1], nn.Tanh):
                e = e + 2 * U * y.abs()
        h = y
    return h, e


def value_net(pol, head):
    """nn.Sequential from the input the output layer reads... to V: the hidden layers of `head` then the value layer."""
    mods = list(head) if isinstance(head, nn.Sequential) else [head]
    return nn.Sequential(*mods[:-1], pol._value)


def within(got, ref, bound, slack=1.0):
    err = ((got.double() - ref).abs() / (bound + 1e-30)).max().item() if got.numel() else 0.0
    assert err <= slack, err
    return err


# ---------------------------------------------------------------------------------------------------------------
# 1-5. the quadrotor, MLP, all three tasks
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("task", ["velocity_control", "hovering_control", "no_collision"])
def test_quad_critic(task):
    n, T = 300, 32
    a, b = quad_env(n, task), quad_env(n, task)
    module, plain = quad_t.make_policy(a, (64, 17), nn.Tanh, 3, LOG_STD)
    critic = with_value(plain, 1)
    ref = a.rollout(T, policy=plain, act_seed=SEED)
    out = b.rollout(T, policy=critic, act_seed=SEED, gae=GAE, out=nan_out(ref, T, n, b.device))
    assert_rest_equal(ref, out)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])
    net = value_net(critic, module)
    pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).double()
    with torch.no_grad():
        v, vb = forward_bound(net, pre)
        within(out["value"], v[..., 0], vb[..., 0])
        where = check_final_written(critic, out)
        assert where.any()
        fv, fb = forward_bound(net, out["final_obs"][where].double())
        within(out["final_value"][where], fv[..., 0], fb[..., 0])
    check_gae(critic, out)
    nxt = b.rollout(4, policy=critic, act_seed=SEED)
    assert torch.equal(nxt["value"][0], out["value_last"])
    assert set(nxt) >= {"value", "value_last"} and "adv" not in nxt and "final_value" in nxt


# ---------------------------------------------------------------------------------------------------------------
# 1-5. MetaMaze2D: MLP, GRU and LSTM, with and without resampling, and the task rule on a k = 2 trial handle
# ---------------------------------------------------------------------------------------------------------------

MAZE_CASES = [("mlp", False, None), ("mlp", True, None), ("gru", False, None), ("gru", True, None),
              ("lstm", False, None), ("lstm", True, None), ("gru", True, 2), ("lstm", True, 2), ("mlp", True, 2)]
SHAPES = {"mlp": Shape("mlp", (33, 17)), "gru": Shape("gru", H=17, width=13), "lstm": Shape("lstm", H=8, width=5),
          "gru-task": Shape("gru", H=17, width=0, reset="task"), "lstm-task": Shape("lstm", H=8, width=11, reset="task")}


def maze_shape(kind, k):
    return SHAPES[kind + "-task"] if k and kind != "mlp" else SHAPES[kind]


def maze_reference(kind, plain, critic, module, out):
    """(worst value error / bound, the final_value check) against float64: the MLP on the inputs, a cell teacher-forced
    on the kernel's h_t (and, for the LSTM, on the float64 c with its propagated bound)."""
    T, N = out["act"].shape
    where = check_final_written(critic, out)
    fvo = out["final_obs"].reshape(T, N, -1).double()
    if kind == "mlp":
        net = value_net(critic, module)
        pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, N, -1).double()
        v, vb = forward_bound(net, pre)
        within(out["value"], v[..., 0], vb[..., 0])
        fv, fb = forward_bound(net, fvo[where])
        within(out["final_value"][where], fv[..., 0], fb[..., 0])
        return where
    hid = out["hid"].double()
    if kind == "gru":
        Wi, Wh, bi, bh, head = gru_t.unpack(plain)
    else:
        Wi, Wh, bi, bh, head = lstm_t.unpack(plain)
    net = value_net(critic, head)
    v, vb = forward_bound(net, hid)
    within(out["value"], v[..., 0], vb[..., 0])
    # the terminal step: the cell once more on [final window, onehot(a_t), (float)r_t] from h_t (and c'_t)
    H = plain.hidden
    fbk = torch.cat([torch.nn.functional.one_hot(out["act"].long(), 4).double(),
                     out["rew"].float().double()[..., None]], -1)
    x = torch.cat([fvo, fbk], -1) if plain.feedback else fvo
    if kind == "gru":
        h, eb = gru_t.gru_bound(Wi, Wh, bi, bh, x[where], hid[where])
    else:
        # c'_t in float64 with its bound, teacher-forced on the kernel's h as lstm_t.teacher_forced carries it
        obs = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, N, -1).double()
        s0 = out["state0"].double()
        wipe = cut_mask(critic, out)
        hp, c, fb = s0[:, :H], s0[:, H:2 * H], s0[:, 2 * H:]
        ec = torch.zeros_like(c)
        cs, ecs = [], []
        for t in range(T):
            xt = torch.cat([obs[t], fb], -1) if plain.feedback else obs[t]
            _, _, c, ec = lstm_t.lstm_bound(Wi, Wh, bi, bh, xt, hp, c, ec)
            cs.append(c)
            ecs.append(ec)
            keep = ~wipe[t][:, None]
            hp = torch.where(keep, hid[t], 0.0)
            c, ec = torch.where(keep, c, 0.0), torch.where(keep, ec, 0.0)
            fb = torch.where(keep, fbk[t], 0.0)
        c_all, ec_all = torch.stack(cs), torch.stack(ecs)
        h, eb, _, _ = lstm_t.lstm_bound(Wi, Wh, bi, bh, x[where], hid[where], c_all[where], ec_all[where])
    fv, fb_ = bound_from(net, h, eb)
    within(out["final_value"][where], fv[..., 0], fb_[..., 0])
    return where


@pytest.mark.parametrize("kind,rs,k", MAZE_CASES, ids=["%s-rs%d-k%s" % c for c in MAZE_CASES])
def test_maze_critic(kind, rs, k):
    shape = maze_shape(kind, k)
    n, T = 300, 24
    a, b = maze_env(n, shape, k=k), maze_env(n, shape, k=k)
    module, plain = shape.policy(a, seed=5)
    critic = with_value(plain, 2)
    sa = sb = None
    if kind != "mlp":
        sa = gru_t.random_state(plain, n)
        sb = sa.clone()
    wrote = 0
    for launch in range(3):
        ref = run(a, plain, T, sa, rs)
        out = run(b, critic, T, sb, rs, gae=GAE, out=nan_out(ref, T, n, b.device))
        assert_rest_equal(ref, out)
        if sa is not None:
            assert torch.equal(sa, sb)
        for x, y in zip(a.agent_state(), b.agent_state()):
            assert torch.equal(x, y)
        with torch.no_grad():
            wrote += int(maze_reference(kind, plain, critic, module, out).sum())
        check_gae(critic, out)
        if launch:
            assert torch.equal(out["value"][0], last)
        last = out["value_last"].clone()
    assert wrote > 0
    if k and kind != "mlp":
        cut = cut_mask(critic, out)
        assert (out["done"].bool() & ~cut).any()         # the task rule: some episodes end without a cut


# ---------------------------------------------------------------------------------------------------------------
# 6. populations: member m's block against a handle of its E envs alone
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,E", [("mlp", 32), ("mlp", 256), ("lstm", 32), ("gru", 256), ("lstm-task", 64)])
def test_maze_population_twins(kind, E):
    from metagym_b200 import PolicyPopulation
    shape = SHAPES[kind]
    k = 2 if kind.endswith("task") else None
    M = 3
    n, T = E * M, 24
    big = maze_env(n, shape, k=k)
    pop = PolicyPopulation([with_value(shape.policy(big, seed=3 + 7 * m)[1], m) for m in range(M)])
    state = gru_t.random_state(pop, n) if shape.kind != "mlp" else None
    st0 = state.clone() if state is not None else None
    out = run(big, pop, T, state, True, gae=GAE)
    for m in range(M):
        tw = maze_env(E, shape, base=m * E, k=k)
        ts = st0[m * E:(m + 1) * E].clone() if state is not None else None
        ref = run(tw, pop.policies[m], T, ts, True, gae=GAE)
        mine = pop.member_slice(out, m)
        where = cut_mask(pop.policies[m], ref) & ref["truncated"].bool()
        for key in ("value", "value_last", "adv", "ret", "act", "logp", "rew", "done", "truncated"):
            assert torch.equal(mine[key], ref[key]), (m, key)
        assert torch.equal(mine["final_value"][where], ref["final_value"][where]), m
        if state is not None:
            assert torch.equal(pop.member_slice(state, m), ts)
        tw.close()
    big.close()


@pytest.mark.parametrize("E", [32, 128])
def test_quad_population_twins(E):
    from metagym_b200 import PolicyPopulation
    M = 3
    big = quad_env(E * M)
    pop = PolicyPopulation([with_value(quad_t.make_policy(big, (64, 17), nn.Tanh, 3 + 7 * m, LOG_STD)[1], m)
                            for m in range(M)])
    out = big.rollout(32, policy=pop, act_seed=SEED, gae=GAE)
    for m in range(M):
        tw = quad_env(E, base=m * E)
        ref = tw.rollout(32, policy=pop.policies[m], act_seed=SEED, gae=GAE)
        mine = pop.member_slice(out, m)
        where = ref["done"].bool() & ref["truncated"].bool()
        for key in ("value", "value_last", "adv", "ret", "act", "logp", "rew", "done", "truncated"):
            assert torch.equal(mine[key], ref[key]), (m, key)
        assert torch.equal(mine["final_value"][where], ref["final_value"][where]), m
        tw.close()
    big.close()


# ---------------------------------------------------------------------------------------------------------------
# 7. graph capture sees a write into the value row of pop.params
# ---------------------------------------------------------------------------------------------------------------

def test_graph_capture_sees_the_value_row():
    from metagym_b200 import PolicyPopulation
    shape = SHAPES["lstm"]
    n, M, T = 256, 2, 16
    a, b = maze_env(n, shape), maze_env(n, shape)
    pop = PolicyPopulation([with_value(shape.policy(a, seed=m)[1], m) for m in range(M)])
    sa = gru_t.random_state(pop, n)
    sb = sa.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        snap = a.snapshot()
        run(a, pop, T, sa, False, gae=GAE)                       # warm-up outside the capture
        a.restore(snap)
        sa.copy_(sb)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = run(a, pop, T, sa, False, gae=GAE)
    torch.cuda.synchronize()
    k = shape.width
    row = pop.numel - 5 * (k + 1)            # the output layer: W [5][k], then b [5]
    new = pop.params.clone()
    new[:, row + 4 * k:row + 5 * k] += 0.25  # the value row's weights
    new[:, -1] += 1.5                        # and its bias
    a.restore(snap)
    sa.copy_(sb)
    pop.params.copy_(new)
    g.replay()
    torch.cuda.synchronize()
    ref_pop = PolicyPopulation([with_value(shape.policy(b, seed=m)[1], m) for m in range(M)])
    ref_pop.params.copy_(new)
    ref = run(b, ref_pop, T, sb, False, gae=GAE)
    for key in ("value", "value_last", "adv", "ret", "act", "logp", "hid"):
        assert torch.equal(out[key], ref[key]), key


# ---------------------------------------------------------------------------------------------------------------
# 8. refusals leave the handle, its counter and the state untouched
# ---------------------------------------------------------------------------------------------------------------

def critic_struct(T, n, dev, gamma=0.99, lam=0.95, value=True, final=True, adv=True, ret=True):
    from metagym_b200 import _lib
    bufs = [torch.zeros((T, n), device=dev) if on else None for on in (value, True, final, adv, ret)]
    bufs[1] = torch.zeros(n, device=dev)
    return _lib.Critic(*[_lib.ptr(x) for x in bufs], gamma, lam), bufs


BAD = [dict(value=False), dict(adv=False), dict(ret=False), dict(final=False), dict(gamma=float("nan")),
       dict(gamma=1.5), dict(gamma=-0.1), dict(lam=float("inf")), dict(lam=-1e-3)]
WHY = ["null value_dev", "go together", "go together", "need rew", "gamma", "gamma", "gamma", "lambda", "lambda"]


def test_maze_refusals_leave_everything_untouched():
    from metagym_b200 import MgbError, PolicyPopulation, _lib
    lib = _lib.load()
    T, n = 4, 256
    for kind in ("mlp", "lstm"):
        shape = SHAPES[kind]
        env = maze_env(n, shape)
        critic = with_value(shape.policy(env, seed=1)[1], 0)
        pop = PolicyPopulation([critic])
        state = gru_t.random_state(critic, n) if kind != "mlp" else None
        before = state.clone() if state is not None else None
        counters, st = env._counters(), [x.clone() for x in env.agent_state()]
        rew = torch.zeros((T, n), dtype=torch.float64, device=env.device)
        done = torch.zeros((T, n), dtype=torch.uint8, device=env.device)
        trunc = torch.zeros((T, n), dtype=torch.uint8, device=env.device)

        def call(cr, r=rew, d=done, tr=trunc):
            outs = [None, None, None, None, _lib.ptr(r), _lib.ptr(d), None, _lib.ptr(tr)]
            if kind == "mlp":
                return lib.mgb_maze_rollout_critic(env._h, T, ctypes.byref(pop.struct()), 1, 0, SEED, None, 0, *outs,
                                                   ctypes.byref(cr), env._stream())
            return lib.mgb_maze_rollout_rnn_critic(env._h, T, ctypes.byref(pop.struct()), 1, 0, SEED, None, 0,
                                                   state.data_ptr(), None, None, *outs, ctypes.byref(cr),
                                                   env._stream())
        for bad, why in zip(BAD, WHY):
            cr, bufs = critic_struct(T, n, env.device, **bad)
            assert call(cr) == MGB_ERR_ARG, bad
            assert why in lib.mgb_last_error().decode(), (bad, lib.mgb_last_error())
        cr, bufs = critic_struct(T, n, env.device)
        assert call(cr, tr=None) == MGB_ERR_ARG and "need rew" in lib.mgb_last_error().decode()
        assert call(cr, r=None) == MGB_ERR_ARG and "need rew" in lib.mgb_last_error().decode()
        torch.cuda.synchronize()
        assert env._counters() == counters
        for x, y in zip(st, env.agent_state()):
            assert torch.equal(x, y)
        if state is not None:
            assert torch.equal(state, before)
        assert all(float(x.abs().sum()) == 0 for x in bufs if x is not None)
        env.close()
    # auto_reset off
    shape = SHAPES["mlp"]
    env = maze_env(128, shape, auto_reset=False)
    critic = with_value(shape.policy(env, seed=1)[1], 0)
    counters = env._counters()
    with pytest.raises(MgbError, match="auto_reset"):
        env.rollout(T, policy=critic, act_seed=SEED)
    assert env._counters() == counters
    env.close()
    # the footprint: an LSTM of H = 64 with a 64-wide head at view_grid 4 does not fit
    big = Shape("lstm", H=64, width=64, view_grid=4)
    env = maze_env(128, big)
    critic = with_value(big.policy(env, seed=1)[1], 0)
    state = critic.initial_state(128)
    counters = env._counters()
    with pytest.raises(MgbError, match="bytes of shared memory"):
        env.rollout(T, policy=critic, state=state, act_seed=SEED)
    torch.cuda.synchronize()
    assert env._counters() == counters and float(state.abs().sum()) == 0
    env.close()


def test_quad_refusals_leave_everything_untouched():
    from metagym_b200 import BatchedQuadrotor, PolicyPopulation, _lib
    lib = _lib.load()
    T, n = 4, 128
    q = quad_env(n)
    critic = with_value(quad_t.make_policy(q, (64, 17), nn.Tanh, 3, LOG_STD)[1], 0)
    pop = PolicyPopulation([critic])
    snap, counters = q.snapshot()["records"].clone(), q._counters()
    rew = torch.zeros((T, n), device=q.device)
    done = torch.zeros((T, n), dtype=torch.uint8, device=q.device)
    trunc = torch.zeros((T, n), dtype=torch.uint8, device=q.device)
    for bad, why in zip(BAD, WHY):
        cr, bufs = critic_struct(T, n, q.device, **bad)
        rc = lib.mgb_quad_rollout_critic(q._h, T, ctypes.byref(pop.struct()), 1, 0, SEED, None, None, None, None,
                                         _lib.ptr(rew), _lib.ptr(done), None, _lib.ptr(trunc), ctypes.byref(cr),
                                         q._stream())
        assert rc == MGB_ERR_ARG and why in lib.mgb_last_error().decode(), bad
    torch.cuda.synchronize()
    assert q._counters() == counters and torch.equal(q.snapshot()["records"], snap)
    q.close()
    q2 = BatchedQuadrotor(task="hovering_control", dt=0.005, nt=11, num_envs=n, device=0, squeeze=False,
                          auto_reset=False)
    q2.reset()
    counters = q2._counters()
    c2 = with_value(quad_t.make_policy(q2, (64, 17), nn.Tanh, 3, LOG_STD)[1], 0)
    with pytest.raises(Exception, match="auto_reset"):
        q2.rollout(T, policy=c2, act_seed=SEED)
    assert q2._counters() == counters
    with pytest.raises(ValueError, match="value head"):
        q2.rollout(T, policy=quad_t.make_policy(q2, (64, 17), nn.Tanh, 3, LOG_STD)[1], gae=GAE)
    q2.close()


# ---------------------------------------------------------------------------------------------------------------
# unroll(value=True) and evaluate() against the kernel
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gru", "lstm-task"])
def test_unroll_value_agrees_with_the_kernel(kind):
    from metagym_b200 import PolicyPopulation
    shape = SHAPES[kind]
    k = 2 if kind.endswith("task") else None
    n = 256
    env = maze_env(n, shape, k=k)
    pop = PolicyPopulation([with_value(shape.policy(env, seed=11 + m)[1], m) for m in range(2)])
    state = pop.initial_state(n)
    out = run(env, pop, 24, state, True, gae=GAE)
    logits, logp, value = pop.unroll(out, value=True)
    assert value.shape == out["value"].shape and value.requires_grad
    err = (value.detach().double().cpu() - out["value"].double().cpu()).abs().max().item()
    assert err < 1e-4, err
    env.close()


def test_evaluate_agrees_with_the_kernel():
    q = quad_env(256)
    critic = with_value(quad_t.make_policy(q, (64, 64), nn.Tanh, 3, LOG_STD)[1], 0)
    out = q.rollout(16, policy=critic, act_seed=SEED, gae=GAE)
    pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0)
    with torch.no_grad():
        _, v = critic.evaluate(pre)
    assert (v - out["value"].cpu()).abs().max().item() < 1e-4
    assert math.isfinite(float(out["adv"].abs().max()))
    q.close()

