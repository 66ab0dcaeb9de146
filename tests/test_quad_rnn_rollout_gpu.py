"""GPU: quadrotor rollouts driven by an on-device GRU or LSTM policy with a Gaussian head (mgb_quad_rollout_rnn,
BatchedQuadrotor.rollout(policy=GRUPolicy/LSTMPolicy(dist="gaussian"), state=); DESIGN.md "Recurrent quadrotor
policies").

1. Every task, both physics paths, both cells, FIN off and on: the env side is bit for bit the open-loop rollout fed
   the actions taken; every h_t, teacher-forced, lies within the header's float32 bound of a float64 cell (the LSTM's
   c carried in float64 with its bound); the actions are mean + exp(log_std) z with z restated from Philox and logp
   within bound; deterministic mode takes the mean; the final state is the restated carry, zero after a done and
   (a_t, r_t) in the feedback otherwise.
2. Two launches of T are one launch of 2T; two handles split by env_index_base are one handle; a captured rollout sees
   policy.update().
3. Populations: one member is the single call, and twin handles match per member for E = 32, 64, 128 and 256.
4. Critic: every other output is the value-less policy's; value and final_value within the float32 bound;
   final_value written exactly where done & truncated; value_last is the next launch's value[0]; adv and ret are
   gae_f32 bit for bit.
5. Unroll: the fused cell sequence's h is the rollout's hid bit for bit, logp within bound of the rollout's, gradients
   (log_std included) match _unroll_reference to float32 tolerance.
6. Footprint: the restated byte count gives the largest H that fits and H + 1 is refused with that exact count; every
   refusal leaves t_base, the state and the outputs untouched.
"""
import ctypes
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from critic_ref import gae_f32  # noqa: E402
from policy_draws import quad_policy_normals  # noqa: E402
from test_lstm_policy_rollout_maze_gpu import lstm_bound  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402
from test_rnn_policy_rollout_maze_gpu import gru_bound  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SEED = 0x9E3779B97F4A7C15
LOG_STD = (-0.5, 0.0, 0.3, -1.0)
TASKS = ("velocity_control", "no_collision", "hovering_control")
CTA = 128                   # MGB_QUAD_RNN_CTA_ENVS
TILES = 2 * CTA * 19 * 4    # the kernel's static observation tiles


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def make_env(n, task="velocity_control", base=0, fin=True, conf=None, nt=20, auto_reset=True):
    from metagym_b200 import BatchedQuadrotor
    kw = dict(seed=[0, 1, 2]) if task == "velocity_control" else {}
    e = BatchedQuadrotor(task=task, dt=0.005, nt=nt, num_envs=n, device=0, squeeze=False, auto_reset=auto_reset,
                         final_obs=fin, rng_seed=5, env_index_base=base, simulator_conf=conf, **kw)
    e.reset()
    e.rollout(5)                                    # t_base != 0
    return e


def general():
    from oracle import quad_oracle as qo
    return qo.general_params()


def make_policy(env, kind="gru", H=24, width=0, value=False, seed=0, log_std=LOG_STD):
    from metagym_b200 import GRUPolicy, LSTMPolicy
    g = torch.Generator().manual_seed(seed)
    Cell, Pol = (nn.GRUCell, GRUPolicy) if kind == "gru" else (nn.LSTMCell, LSTMPolicy)
    cell = Cell(env.obs_dim + 5, H)
    head = nn.Linear(H, 4) if not width else nn.Sequential(nn.Linear(H, width), nn.Tanh(), nn.Linear(width, 4))
    vh = nn.Linear(width or H, 1) if value else None
    mods = list(cell.parameters()) + list(head.parameters()) + (list(vh.parameters()) if value else [])
    with torch.no_grad():
        for p in mods:
            p.copy_(torch.randn(p.shape, generator=g) * (1.2 / p.shape[-1] ** 0.5 if p.dim() == 2 else 0.3))
        # the feedback columns see voltages near 7.5: keep their weights small so the gates do not saturate
        cell.weight_ih[:, env.obs_dim:env.obs_dim + 4].mul_(0.05)
        (head if width == 0 else head[-1]).bias.add_(7.5)     # mid-range voltages, so that episodes last
    ls = None if log_std is None else torch.tensor(log_std)
    return Pol(cell, head, log_std=ls, dist="gaussian", device=env.device, value=vh)


def unpack(pol):
    """float64 cell weights, the head as an nn.Sequential, the value row (W, b) or None and log_std, read from the
    packed float32 buffer (what the kernel reads)."""
    buf = pol.params.double()
    G = 3 if pol._cell_code == 0 else 4
    H, n_in = pol.hidden, pol.obs_dim + 5
    o = 0

    def take(k):
        nonlocal o
        o += k
        return buf[o - k:o]
    Wi, Wh = take(G * H * n_in).reshape(G * H, n_in), take(G * H * H).reshape(G * H, H)
    bi, bh = take(G * H), take(G * H)
    dims = [H] + ([pol.head_width] if pol.head_width else []) + [4]
    layers, vrow = [], None
    for k in range(len(dims) - 1):
        last = k == len(dims) - 2
        rows = dims[k + 1] + (1 if last and pol.has_value else 0)
        W, b = take(dims[k] * rows).reshape(rows, dims[k]), take(rows)
        lin = nn.Linear(dims[k], dims[k + 1]).double().to(buf.device)
        with torch.no_grad():
            lin.weight.copy_(W[:dims[k + 1]])
            lin.bias.copy_(b[:dims[k + 1]])
        if last and pol.has_value:
            vrow = nn.Sequential(nn.Linear(dims[k], 1).double().to(buf.device))
            with torch.no_grad():
                vrow[0].weight.copy_(W[4:5])
                vrow[0].bias.copy_(b[4:5])
        layers.append(lin)
        if not last:
            layers.append(nn.ReLU() if pol.activation == 1 else nn.Tanh())
    ls = take(4)
    assert o == buf.numel()
    return Wi, Wh, bi, bh, nn.Sequential(*layers), vrow, ls


def teacher_forced(pol, out, cs=None):
    """(worst |hid - h_ref| / bound over every t, the restated final state row [N, S] float64 with its bound).  x_t is
    [obs_t, a_{t-1}, r_{t-1}] (state0's feedback at t = 0, zeros after a done); h_{t-1} is state0's at t = 0, the
    kernel's hid[t-1], zeros after a done; the LSTM's c is carried in float64 with a bound, and each step's c'_t
    (before the wipe) with its bound is appended to the list cs when one is given."""
    Wi, Wh, bi, bh = unpack(pol)[:4]
    lstm = pol._cell_code == 1
    H = pol.hidden
    hid = out["hid"].double()
    T, N = hid.shape[:2]
    obs = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).double()
    done = out["done"].bool()
    s0 = out["state0"].double()
    nm = 2 * H if lstm else H
    hp, fb = s0[:, :H], s0[:, nm:]
    c, ec = (s0[:, H:2 * H], torch.zeros((N, H), dtype=torch.float64, device=hid.device)) if lstm else (None, None)
    worst = 0.0
    for t in range(T):
        x = torch.cat([obs[t], fb], 1)
        if lstm:
            h, eh, c2, ec2 = lstm_bound(Wi, Wh, bi, bh, x, hp, c, ec)
            if cs is not None:
                cs.append((c2, ec2))
        else:
            h, eh = gru_bound(Wi, Wh, bi, bh, x, hp)
        worst = max(worst, float(((hid[t] - h).abs() / eh).max()))
        d = done[t][:, None]
        hp = torch.where(d, 0., hid[t])
        fb = torch.where(d, 0., torch.cat([out["act"][t].double(), out["rew"][t].double()[:, None]], 1))
        if lstm:
            c, ec = torch.where(d, 0., c2), torch.where(d, 0., ec2)
    if lstm:
        return worst, torch.cat([hp, c, fb], 1), torch.cat([torch.zeros_like(hp), ec, torch.zeros_like(fb)], 1)
    return worst, torch.cat([hp, fb], 1), torch.zeros_like(torch.cat([hp, fb], 1))


def check_actions(env, pol, out, t0, deterministic=False):
    """act and logp against the float64 head on the kernel's hid with the Philox normals; worst error / bound."""
    head, ls = unpack(pol)[4], unpack(pol)[6]
    hid = out["hid"].double()
    mean, bound = forward_bound(head, hid)
    act = out["act"].double()
    if deterministic:
        return float(((act - mean).abs() / (bound + U * mean.abs() + 1e-30)).max())
    T, N = hid.shape[:2]
    genv = env.env_index_base + np.arange(N)
    std = torch.exp(ls)
    worst = 0.0
    for t in range(T):
        z = torch.as_tensor(quad_policy_normals(SEED, genv, t0 + t), device=act.device)
        want = mean[t] + std * z
        tol = bound[t] + 8 * U * std * (z.abs() + 1) + U * want.abs()
        worst = max(worst, float(((act[t] - want).abs() / tol).max()))
        # the kernel's logp depends on z alone: sum_k (-z_k^2 / 2 - log_std_k) - 2 log(2 pi)
        lp = (-0.5 * z * z - ls).sum(-1) - 2 * math.log(2 * math.pi)
        lp_tol = ((z.abs() / std) * tol).sum(-1) + 16 * U * ((z * z / 2 + ls.abs()).sum(-1) + 4)
        worst = max(worst, float(((out["logp"][t].double() - lp).abs() / lp_tol).max()))
    return worst


def value_bound(pol, h, eh=None):
    """float64 V on cell outputs h [..., H] and the bound on the float32 kernel's V: the head's hidden layer and the
    value row as fma chains (forward_bound), plus an error eh of h itself carried through |W|."""
    head, vrow = unpack(pol)[4:6]
    eh = torch.zeros_like(h) if eh is None else eh
    if pol.head_width:
        hidden = nn.Sequential(*list(head)[:-1])
        z, ez = forward_bound(hidden, h)
        ez = ez + eh @ list(head)[0].weight.detach().abs().T
    else:
        z, ez = h, eh
    v, ev = forward_bound(vrow, z)
    return v[..., 0], (ev + ez @ vrow[0].weight.detach().abs().T)[..., 0]


def assert_env_side_equal(a, b, fin=True):
    for k in ("obs", "rew", "done"):
        assert torch.equal(a[k], b[k]), k
    if fin:
        assert torch.equal(a["truncated"], b["truncated"])
        d = a["done"].bool()
        assert torch.equal(a["final_obs"][d], b["final_obs"][d])


def random_state(pol, N, seed=1):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn((N, pol.state_dim), generator=g) * 0.5
    s[:, -5:-1] = 7.5 + torch.randn((N, 4), generator=g)      # a plausible previous action
    return s.to(pol.device)


# ---------------------------------------------------------------------------------------------------------------
# 1. the matrix
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fin", [False, True], ids=["fin0", "fin1"])
@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task", TASKS)
def test_rollout_against_references(task, config, kind, fin):
    n, T = 500, 40
    env = make_env(n, task, fin=fin, conf=None if config == "default" else general())
    pol = make_policy(env, kind, H=24, seed=len(task))
    state = random_state(pol, n)
    s0 = state.clone()
    snap = env.snapshot()
    t0 = env._counters()
    out = env.rollout(T, policy=pol, act_seed=SEED, state=state, want_hidden=True)
    assert out["done"].any(), "no episode ended: the carry's wipe is not exercised"
    assert torch.equal(out["state0"], s0)
    assert env._counters() == t0 + T
    env.restore(snap)
    ref = env.rollout(T, actions=out["act"])
    assert_env_side_equal(out, ref, fin)
    worst, st_ref, st_bound = teacher_forced(pol, out)
    assert worst <= 1.0, worst
    assert check_actions(env, pol, out, t0) <= 1.0
    # the final state: the h rows are hid[T - 1] bit for bit, the feedback (a, r) bit for bit, zero after a done
    H = pol.hidden
    d = out["done"][-1].bool()
    assert torch.equal(state[:, :H], torch.where(d[:, None], 0., out["hid"][-1]))
    fb = torch.where(d[:, None], 0., torch.cat([out["act"][-1], out["rew"][-1][:, None]], 1))
    assert torch.equal(state[:, -5:], fb)
    assert not state[d].any()
    assert bool(((state.double() - st_ref).abs() <= st_bound * 1.0 + 1e-30).all())
    # deterministic: a = mean, no logp
    env.restore(snap)
    det_state = s0.clone()
    det = env.rollout(T, policy=pol, deterministic=True, state=det_state, want_hidden=True)
    assert det["logp"] is None
    assert check_actions(env, pol, det, t0, deterministic=True) <= 1.0
    env.restore(snap)
    assert_env_side_equal(det, env.rollout(T, actions=det["act"]), fin)
    env.close()


# ---------------------------------------------------------------------------------------------------------------
# 2. continuity, sharding, graph capture
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_two_launches_are_one(kind):
    n, T = 300, 24
    a, b = make_env(n), make_env(n)
    pol = make_policy(a, kind, H=32, width=16)
    sa = random_state(pol, n)
    sb = sa.clone()
    one = a.rollout(2 * T, policy=pol, act_seed=SEED, state=sa, want_hidden=True)
    p1 = b.rollout(T, policy=pol, act_seed=SEED, state=sb, want_hidden=True)
    p2 = b.rollout(T, policy=pol, act_seed=SEED, state=sb, want_hidden=True)
    assert one["done"].any()
    for k in ("obs", "rew", "done", "act", "logp", "hid", "truncated"):
        assert torch.equal(one[k], torch.cat([p1[k], p2[k]], 0)), k
    d = one["done"].bool()
    assert torch.equal(one["final_obs"][d], torch.cat([p1["final_obs"], p2["final_obs"]], 0)[d])
    assert torch.equal(sa, sb)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_sharded_handles_are_one_handle(kind):
    n, T, cut = 384, 24, 160
    whole = make_env(n)
    parts = [make_env(cut), make_env(n - cut, base=cut)]
    pol = make_policy(whole, kind)
    s = random_state(pol, n)
    s_parts = [s[:cut].clone(), s[cut:].clone()]
    out = whole.rollout(T, policy=pol, act_seed=SEED, state=s, want_hidden=True)
    outs = [p.rollout(T, policy=pol, act_seed=SEED, state=sp, want_hidden=True) for p, sp in zip(parts, s_parts)]
    for k in ("obs", "rew", "done", "act", "logp", "hid", "truncated"):
        assert torch.equal(out[k], torch.cat([o[k] for o in outs], 1)), k
    assert torch.equal(s, torch.cat(s_parts, 0))


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_graph_capture_sees_update(kind):
    n, T = 256, 16
    a, b = make_env(n), make_env(n)
    pol = make_policy(a, kind, value=False)
    sa = random_state(pol, n)
    sb = sa.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        snap = a.snapshot()
        a.rollout(T, policy=pol, act_seed=SEED, state=sa, want_hidden=True)      # warm-up outside the capture
        a.restore(snap)
        sa.copy_(sb)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = a.rollout(T, policy=pol, act_seed=SEED, state=sa, want_hidden=True)
    torch.cuda.synchronize()
    new = make_policy(a, kind, seed=9, log_std=(0.2, -0.2, 0.1, -0.3))
    pol.update(new._cell, new._head, log_std=torch.tensor((0.2, -0.2, 0.1, -0.3)))
    a.restore(snap)
    sa.copy_(sb)
    g.replay()
    torch.cuda.synchronize()
    ref = b.rollout(T, policy=new, act_seed=SEED, state=sb, want_hidden=True)
    for k in ("obs", "rew", "done", "act", "logp", "hid"):
        assert torch.equal(out[k], ref[k]), k
    assert torch.equal(sa, sb)


# ---------------------------------------------------------------------------------------------------------------
# 3. populations
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_one_member_is_the_single_policy(kind):
    from metagym_b200 import PolicyPopulation
    n, T = 300, 24
    a, b = make_env(n), make_env(n)
    pol = make_policy(a, kind, value=True)
    sa = random_state(pol, n)
    sb = sa.clone()
    ref = a.rollout(T, policy=pol, act_seed=SEED, state=sa, want_hidden=True, gae=(0.99, 0.95))
    out = b.rollout(T, policy=PolicyPopulation([pol]), act_seed=SEED, state=sb, want_hidden=True, gae=(0.99, 0.95))
    d = ref["done"].bool()
    written = {"final_obs": d, "final_value": d & ref["truncated"].bool()}     # other rows are not written
    for k in ref:
        if isinstance(ref[k], torch.Tensor):
            m = written.get(k)
            assert torch.equal(out[k] if m is None else out[k][m], ref[k] if m is None else ref[k][m]), k
    assert torch.equal(sa, sb)


@pytest.mark.parametrize("kind,E", [("gru", 32), ("lstm", 64), ("gru", 128), ("lstm", 256)])
def test_twin_handles_per_member(kind, E):
    from metagym_b200 import PolicyPopulation
    M = 512 // E
    n, T = E * M, 24
    big = make_env(n)
    pop = PolicyPopulation([make_policy(big, kind, H=20, width=8, seed=3 + 7 * m) for m in range(M)])
    s = random_state(pop.policies[0], n)
    s_ref = s.clone()
    out = big.rollout(T, policy=pop, act_seed=SEED, state=s, want_hidden=True)
    assert out["done"].any()
    for m in range(M):
        tw = make_env(E, base=m * E)
        sm = s_ref[m * E:(m + 1) * E].clone()
        ref = tw.rollout(T, policy=pop.policies[m], act_seed=SEED, state=sm, want_hidden=True)
        got = pop.member_slice(out, m)
        for k in ("obs", "rew", "done", "act", "logp", "hid", "state0", "truncated"):
            assert torch.equal(got[k], ref[k]), (m, k)
        assert torch.equal(s[m * E:(m + 1) * E], sm), m
        tw.close()
    with pytest.raises(ValueError):
        PolicyPopulation([make_policy(big, kind) for _ in range(2)]).check_envs(2 * 96, CTA)


# ---------------------------------------------------------------------------------------------------------------
# 4. critic
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("config", ["default", "general"])
def test_critic(kind, config):
    n, T = 400, 40
    conf = None if config == "default" else general()
    a, b = make_env(n, "hovering_control", conf=conf), make_env(n, "hovering_control", conf=conf)
    pol = make_policy(a, kind, H=24, width=12, value=True)
    sa = random_state(pol, n)
    sb = sa.clone()
    f32 = lambda *sh: torch.empty(sh, dtype=torch.float32, device=a.device)      # noqa: E731
    out = {"obs": f32(T, n, a.obs_dim), "rew": f32(T, n), "done": torch.empty((T, n), dtype=torch.uint8, device=a.device),
           "act": f32(T, n, 4), "logp": f32(T, n), "obs0": f32(n, a.obs_dim), "state0": f32(n, pol.state_dim),
           "hid": f32(T, n, pol.hidden), "final_obs": f32(T, n, a.obs_dim),
           "truncated": torch.empty((T, n), dtype=torch.uint8, device=a.device),
           "final_value": torch.full((T, n), float("nan"), device=a.device)}
    a.rollout(T, policy=pol, act_seed=SEED, state=sa, want_hidden=True, gae=(0.99, 0.95), out=out)
    # the value-less policy's outputs, bit for bit
    plain = make_policy(b, kind, H=24, width=12, value=False)
    plain.update(pol._cell, pol._head)
    ref = b.rollout(T, policy=plain, act_seed=SEED, state=sb, want_hidden=True)
    for k in ("obs", "rew", "done", "act", "logp", "hid", "truncated"):
        assert torch.equal(out[k], ref[k]), k
    done, trunc = out["done"].bool(), out["truncated"].bool()
    assert torch.equal(out["final_obs"][done], ref["final_obs"][done])
    assert torch.equal(sa, sb)
    assert (done & trunc).any()
    # value within the float32 bound of the float64 value row on the head's input
    head, vrow = unpack(pol)[4:6]
    v, ev = value_bound(pol, out["hid"].double())
    assert bool(((out["value"].double() - v).abs() <= ev * 1.01 + 1e-30).all())
    # final_value: written exactly where done & truncated; there, the cell from (h_t, c'_t) on [terminal obs, a_t, r_t]
    fv = out["final_value"]
    assert bool(torch.isnan(fv[~(done & trunc)]).all())
    assert not torch.isnan(fv[done & trunc]).any()
    Wi, Wh, bi, bh = unpack(pol)[:4]
    H = pol.hidden
    t_idx, e_idx = torch.nonzero(done & trunc, as_tuple=True)
    x = torch.cat([out["final_obs"][t_idx, e_idx].double(), out["act"][t_idx, e_idx].double(),
                   out["rew"][t_idx, e_idx].double()[:, None]], 1)
    hp = out["hid"][t_idx, e_idx].double()
    if kind == "gru":
        h, eh = gru_bound(Wi, Wh, bi, bh, x, hp)
    else:       # c'_t is not reported: the teacher-forced carry restates it, with its bound
        cs = []
        assert teacher_forced(pol, out, cs)[0] <= 1.0
        c2 = torch.stack([c for c, _ in cs])[t_idx, e_idx]
        ec2 = torch.stack([e for _, e in cs])[t_idx, e_idx]
        h, eh = lstm_bound(Wi, Wh, bi, bh, x, hp, c2, ec2)[:2]
    vf, evf = value_bound(pol, h, eh)
    assert bool(((fv[t_idx, e_idx].double() - vf).abs() <= evf * 1.01 + 1e-30).all())
    # value_last is the next launch's value[0]; adv and ret are gae_f32 bit for bit
    nxt = a.rollout(1, policy=pol, act_seed=SEED, state=sa)
    assert torch.equal(out["value_last"], nxt["value"][0])
    c = lambda k: out[k].cpu().numpy()                          # noqa: E731
    adv, ret = gae_f32(c("rew"), c("done"), c("truncated"), c("value"), c("value_last"),
                       np.nan_to_num(c("final_value")), 0.99, 0.95)
    assert np.array_equal(c("adv"), adv) and np.array_equal(c("ret"), ret)


# ---------------------------------------------------------------------------------------------------------------
# 5. unroll
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_unroll(kind):
    from metagym_b200 import cell_seq
    n, T = 256, 32
    env = make_env(n, "hovering_control")
    pol = make_policy(env, kind, H=24, width=8, value=True)
    s = random_state(pol, n)
    out = env.rollout(T, policy=pol, act_seed=SEED, state=s, want_hidden=True, gae=(0.99, 0.95))
    assert out["done"].any()
    for m in (pol._cell, pol._head, pol._value):        # the fused path runs a float32 cell on the device
        m.cuda()
    obs, act, rew, wipe, state0 = pol._unroll_inputs(out)
    X = pol._cell_input(obs, act, rew, wipe, state0).detach().transpose(1, 2).contiguous()
    with torch.no_grad():
        h = cell_seq.run(pol._cell, pol._cell_code, X, wipe.contiguous(), state0[:, :pol._memory * pol.hidden])
    assert torch.equal(h, out["hid"])
    ls = torch.tensor(LOG_STD, device=env.device, requires_grad=True)
    pol.update(log_std=ls)
    mean, logp, v = pol.unroll(out, value=True)
    # both sides are float32 on the same h: each mean within twice the head's bound, so z = (a - mean) / sigma within
    # tol (plus the roundings of a and the subtraction), and logp within sum (|z| + tol) tol and its own roundings
    head = unpack(pol)[4]
    m64, mb = forward_bound(head, out["hid"].double())
    assert bool(((mean.detach().double() - m64).abs() <= mb * 1.01 + 1e-30).all())
    sigma = torch.tensor(LOG_STD, dtype=torch.float64, device=env.device).exp()
    a = out["act"].double()
    tol = (2 * mb + 4 * U * (a.abs() + m64.abs())) / sigma
    z = (a - m64) / sigma
    lp_tol = ((z.abs() + tol) * tol).sum(-1) + 16 * U * ((z * z / 2).sum(-1) + 8)
    assert bool(((logp.detach().double() - out["logp"].double()).abs() <= lp_tol).all())
    vb, evb = value_bound(pol, out["hid"].double())
    assert bool(((v.detach().double() - out["value"].double()).abs() <= 2 * evb + 1e-30).all())
    # gradients against the float64 reference loop
    params = list(pol._cell.parameters()) + list(pol._head.parameters()) + list(pol._value.parameters()) + [ls]
    (logp.sum() + v.sum() + mean.pow(2).mean()).backward()
    got = [p.grad.clone() for p in params]
    for p in params:
        p.grad = None
    import copy
    ref_pol = copy.copy(pol)
    ref_pol._cell, ref_pol._head = copy.deepcopy(pol._cell).double(), copy.deepcopy(pol._head).double()
    ref_pol._value = copy.deepcopy(pol._value).double()
    ls64 = ls.detach().double().requires_grad_(True)
    ref_pol._log_std_arg = ls64
    m2, l2, v2 = ref_pol._unroll_reference(out, value=True)
    (l2.sum() + v2.sum() + m2.pow(2).mean()).backward()
    refs = (list(ref_pol._cell.parameters()) + list(ref_pol._head.parameters()) + list(ref_pol._value.parameters())
            + [ls64])
    for g, r in zip(got, refs):
        err = (g.double() - r.grad).abs().max()
        assert float(err) <= 1e-3 * float(r.grad.abs().max()) + 1e-4, float(err)


# ---------------------------------------------------------------------------------------------------------------
# 6. footprint and refusals
# ---------------------------------------------------------------------------------------------------------------

def footprint(gates, H, D, width, value):
    """Bytes of shared memory per CTA of MGB_QUAD_RNN_CTA_ENVS envs, restated from mgb_rnn_plan / mgb_mlp_plan: the cell
    (units rounded up to 8) and its biases, the head (hidden layer rows in groups of 8, the output layer in groups of 4:
    5 rows pad to 8), log_std in a slot of 8, then the columns x, c, h0, h1 and w, plus the static tiles."""
    r8 = lambda k: -(-k // 8) * 8                             # noqa: E731
    Hp, n_in = r8(H), D + 5
    staged = gates * Hp * n_in + gates * Hp * H + 2 * gates * Hp
    head = 0
    k = H
    if width:
        head += r8(r8(width) * H + r8(width))
        k = width
    rows = 8 if value else 4
    head += r8(rows * k + rows) + 8
    C = H if gates == 4 else 0
    Hr = max(H, width) if gates == 4 else H
    Hw = 0 if gates == 4 else width
    return 4 * (staged + head + (n_in + C + 2 * Hr + Hw) * CTA) + TILES


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("width", [0, 64])
@pytest.mark.parametrize("value", [False, True])
def test_footprint_boundary(kind, width, value):
    from metagym_b200 import MgbError
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    gates = 3 if kind == "gru" else 4
    env = make_env(CTA)
    fits = [H for H in range(1, 65) if footprint(gates, H, env.obs_dim, width, value) <= optin]
    Hmax = max(fits)
    assert fits == list(range(1, Hmax + 1))
    pol = make_policy(env, kind, H=Hmax, width=width, value=value)
    s = pol.initial_state(CTA)
    env.rollout(2, policy=pol, act_seed=SEED, state=s, gae=(0.99, 0.95) if value else None)
    if Hmax == 64:
        return
    big = make_policy(env, kind, H=Hmax + 1, width=width, value=value)
    s = random_state(big, CTA)
    s0 = s.clone()
    T = 2
    out = {k: torch.full((T, CTA) + sh, 3.0, device=env.device) for k, sh in
           (("obs", (env.obs_dim,)), ("rew", ()), ("act", (4,)), ("logp", ()), ("hid", (Hmax + 1,)))}
    out["done"] = torch.full((T, CTA), 7, dtype=torch.uint8, device=env.device)
    out["obs0"] = torch.full((CTA, env.obs_dim), 3.0, device=env.device)
    out["state0"] = torch.full((CTA, big.state_dim), 3.0, device=env.device)
    before = {k: v.clone() for k, v in out.items()}
    t0 = env._counters()
    with pytest.raises(MgbError, match=r"needs %d bytes" % footprint(gates, Hmax + 1, env.obs_dim, width, value)):
        env.rollout(T, policy=big, act_seed=SEED, state=s, want_hidden=True, out=out,
                    gae=(0.99, 0.95) if value else None)
    assert env._counters() == t0 and torch.equal(s, s0)
    for k in before:
        assert torch.equal(out[k], before[k]), k


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_refusals_touch_nothing(kind):
    from metagym_b200 import _lib
    env = make_env(CTA)
    lib = _lib.load()
    pol = make_policy(env, kind)
    s = random_state(pol, CTA)
    s0 = s.clone()
    act = torch.full((4, CTA, 4), 3.0, device=env.device)
    t0 = env._counters()

    def call(st=None, state=s.data_ptr(), h=env._h):
        st = st or pol.struct()
        return lib.mgb_quad_rollout_rnn(h, 4, ctypes.byref(st), SEED, state, None, None, act.data_ptr(), None, None,
                                        None, None, None, None, None, env._stream())
    bad_reset = pol.struct()
    bad_reset.reset = _lib.RNN_RESET_TASK
    bad_cell = pol.struct()
    bad_cell.cell = 7
    for rc in (call(bad_reset), call(bad_cell), call(state=None), call(state=s.data_ptr() + 2)):
        assert rc == -1
    off = make_env(CTA, fin=False, auto_reset=False)
    assert lib.mgb_quad_rollout_rnn(off._h, 4, ctypes.byref(pol.struct()), SEED, s.data_ptr(), None, None,
                                    act.data_ptr(), None, None, None, None, None, None, None, off._stream()) == -1
    assert "auto_reset" in lib.mgb_last_error().decode()
    torch.cuda.synchronize()
    assert env._counters() == t0 and torch.equal(s, s0) and bool((act == 3.0).all())
