"""GPU: every compiled cell-sequence kernel (rnn_seq.cu), on the raw operation, at the shapes and edges the unroll
tests skip.

The library compiles rnn_seq_forward_kernel<NG, SAVE> (GRU / LSTM, with and without the saved gates) and
rnn_seq_backward_kernel<NG, HA> with HA = 16, 32, 64, the weight_hh rows rounded up for the warp-uniform float4 reads.
Each backward instantiation runs here at H on both sides of its HA boundary and at padded sizes, over synthetic X, wipe,
state0 and dh with no policy and no rollout, and is checked against a float64 restatement of the masked-reset cell whose
pre-activations x W_ih^T + b_ih and h W_hh^T + b_hh are retained-grad tensors: dgi, the GRU's dghn, dstate0 (the
LSTM's c columns too) and CellSequence's four parameter gradients, each no worse than 4x the error of the same
restatement in float32 plus the floor of test_rnn_unroll_gpu.  Then exact structural checks of the reset rule in the
backward, and PolicyPopulation.unroll's gradients against each member's own unroll.
"""
import pytest
import torch

from test_rnn_unroll_gpu import f64_twin, grads, make_env, make_policy

pytestmark = pytest.mark.gpu

OPTIN_H100 = 232448
HS = (1, 15, 16, 17, 31, 32, 33, 48, 63, 64)
NS = (1, 127, 128, 129, 300)
T = 6


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    pass


def code_of(kind):
    from metagym_b200 import _lib
    return _lib.RNN_CELL_GRU if kind == "gru" else _lib.RNN_CELL_LSTM


def largest_in(kind, H, optin=OPTIN_H100):
    """The largest input width whose forward footprint fits (the backward's does not depend on it)."""
    from metagym_b200 import cell_seq
    G = 3 if kind == "gru" else 4
    n_in = 1
    while cell_seq.smem_bytes(G, H, n_in + 1)[0] <= optin:
        n_in += 1
    assert max(cell_seq.smem_bytes(G, H, n_in)) <= optin < cell_seq.smem_bytes(G, H, n_in + 1)[0]
    return n_in


def inputs(kind, H, n_in, n, bias=True, scale=1.0, seed=0, p_wipe=0.25):
    """Synthetic (X [T, in, N], wipe [T, N] bool, state0 [N, HC], dh [T, N, H], [W_ih, W_hh, b_ih, b_hh]) float32."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = 3 if kind == "gru" else 4
    HC = H if kind == "gru" else 2 * H
    rn = lambda *s: torch.randn(s, generator=g, device="cuda")           # noqa: E731
    X = rn(T, n_in, n)
    wipe = torch.rand((T, n), generator=g, device="cuda") < p_wipe
    s0 = rn(n, HC) * 0.5
    dh = rn(T, n, H)
    params = [rn(G * H, n_in) * (scale * 1.5 / n_in ** 0.5), rn(G * H, H) * (scale * 1.5 / H ** 0.5)]
    params += [rn(G * H) * 0.3 * scale, rn(G * H) * 0.3 * scale] if bias else [None, None]
    return X, wipe, s0, dh, params


def restated(kind, X, wipe, s0, Wi, Wh, bi, bh):
    """h [T, N, H] of the masked-reset cell in the dtype of its arguments, and per step the pre-activations gi = x W_ih^T
    + b_ih and gh = h_{t-1} W_hh^T + b_hh [N, G H] with retained gradients."""
    H = Wh.shape[1]
    hp, cp = s0[:, :H], (s0[:, H:] if kind == "lstm" else None)
    hs, gis, ghs = [], [], []
    for t in range(X.shape[0]):
        if t:
            hp = h.masked_fill(wipe[t - 1][:, None], 0.)
            if kind == "lstm":
                cp = c.masked_fill(wipe[t - 1][:, None], 0.)
        gi = X[t].T @ Wi.T
        gh = hp @ Wh.T
        if bi is not None:
            gi = gi + bi
        if bh is not None:
            gh = gh + bh
        gi.retain_grad()
        gh.retain_grad()
        if kind == "gru":
            r = torch.sigmoid(gi[:, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * hp
        else:
            a = gi + gh
            i, f, gg, o = (a[:, k * H:(k + 1) * H] for k in range(4))
            c = torch.sigmoid(f) * cp + torch.sigmoid(i) * torch.tanh(gg)
            h = torch.sigmoid(o) * torch.tanh(c)
        hs.append(h)
        gis.append(gi)
        ghs.append(gh)
    return torch.stack(hs), gis, ghs


def reference_grads(kind, X, wipe, s0, dh, params, dtype):
    """[dgi [T, G H, N], dghn [T, H, N] (GRU) or None, dstate0, dW_ih, dW_hh, db_ih, db_hh (None without bias), h]."""
    leaves = [s0.to(dtype).clone().requires_grad_()] + [None if p is None else p.to(dtype).clone().requires_grad_()
                                                        for p in params]
    h, gis, ghs = restated(kind, X.to(dtype), wipe, *leaves)
    H = leaves[2].shape[1]
    live = [x for x in leaves if x is not None]
    gs = iter(torch.autograd.grad((h * dh.to(dtype)).sum(), live + gis + ghs, allow_unused=True))
    lg = [None if x is None else next(gs) for x in leaves]
    dgi = torch.stack([next(gs) for _ in gis]).transpose(1, 2)
    dgh = torch.stack([next(gs) for _ in ghs]).transpose(1, 2)
    dghn = dgh[:, 2 * H:] if kind == "gru" else None
    return [dgi, dghn] + lg + [h.detach()]


def kernel_grads(kind, X, wipe, s0, dh, params):
    """The same list from the kernels: dgi, dghn and dstate0 of mgb_rnn_seq_backward, the parameter gradients of
    CellSequence and h of the forward, which saving the gates must not change; also (h, gates)."""
    from metagym_b200 import _lib, cell_seq
    code = code_of(kind)
    H = params[1].shape[1]
    n = X.shape[2]
    packed = cell_seq._packed(*params)
    h, gates = cell_seq.forward(code, H, packed, X, wipe, s0, save=True)
    assert torch.equal(cell_seq.forward(code, H, packed, X, wipe, s0)[0], h)
    G = 3 if kind == "gru" else 4
    dgi = torch.full((X.shape[0], G * H, n), 7.25, device="cuda")
    dghn = torch.full((X.shape[0], H, n), 7.25, device="cuda") if kind == "gru" else None
    ds0 = torch.full_like(s0, 7.25)
    seq = cell_seq._struct(code, H, packed, X, wipe, s0, h, gates)
    seq.dh_dev, seq.dgi_dev, seq.dghn_dev, seq.dstate0_dev = dh.data_ptr(), dgi.data_ptr(), _lib.ptr(dghn), ds0.data_ptr()
    cell_seq._call(_lib.load().mgb_rnn_seq_backward, seq, X.device)
    leaves = [s0.clone().requires_grad_()] + [None if p is None else p.clone().requires_grad_() for p in params]
    hh = cell_seq.CellSequence.apply(code, H, X, wipe, *leaves)
    assert torch.equal(hh, h)
    live = [x for x in leaves if x is not None]
    gs = iter(torch.autograd.grad((hh * dh).sum(), live))
    lg = [None if x is None else next(gs) for x in leaves]
    assert torch.equal(lg[0], ds0)
    return [dgi, dghn] + lg + [h], (h, gates)


NAMES = ("dgi", "dghn", "dstate0", "dW_ih", "dW_hh", "db_ih", "db_hh", "h")


def assert_within_criterion(kind, X, wipe, s0, dh, params):
    got, _ = kernel_grads(kind, X, wipe, s0, dh, params)
    r32 = reference_grads(kind, X, wipe, s0, dh, params, torch.float32)
    r64 = reference_grads(kind, X, wipe, s0, dh, params, torch.float64)
    for name, a, r, ref in zip(NAMES, got, r32, r64):
        assert (a is None) == (ref is None), name
        if a is None:
            continue
        ef, er = float((a.double() - ref).abs().max()), float((r.double() - ref).abs().max())
        floor = 1e-6 * (1. + float(ref.abs().max()))
        assert ef <= 4 * er + floor, (name, ef, er)


def matrix():
    cases, k = [], 0
    for kind in ("gru", "lstm"):
        for H in HS:
            for n_in in (1, 14, None):
                cases.append((kind, H, n_in, NS[k % len(NS)], k % 2 == 0))
                k += 1
    return cases


MATRIX = matrix()


@pytest.mark.parametrize("kind,H,n_in,n,bias", MATRIX,
                         ids=["%s-H%d-in%s-n%d-bias%d" % (c[0], c[1], c[2] or "max", c[3], c[4]) for c in MATRIX])
def test_backward_matrix(kind, H, n_in, n, bias):
    n_in = n_in or largest_in(kind, H, torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    X, wipe, s0, dh, params = inputs(kind, H, n_in, n, bias, seed=H * 7 + n_in + n)
    assert_within_criterion(kind, X, wipe, s0, dh, params)


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("H", [16, 33])
def test_backward_saturated_gates(kind, H):
    """Weights and biases scaled by 8: most gates sit in the flat tails of sigmoid and tanh."""
    X, wipe, s0, dh, params = inputs(kind, H, 14, 300, True, scale=8.0, seed=3)
    assert_within_criterion(kind, X, wipe, s0, dh, params)


# ---------------------------------------------------------------------------------------------------------------
# exact structural checks of the reset rule in the backward
# ---------------------------------------------------------------------------------------------------------------

STRUCT = [(kind, H) for kind in ("gru", "lstm") for H in (7, 16, 32, 48)]


def raw(kind, X, wipe, s0, dh, params):
    """(h, gates, dgi, dghn, dstate0) of one forward and one backward launch."""
    g, (h, gates) = kernel_grads(kind, X, wipe, s0, dh, params)
    return h, gates, g[0], g[1], g[2]


@pytest.mark.parametrize("kind,H", STRUCT, ids=["%s-H%d" % s for s in STRUCT])
def test_gradient_stops_at_wipes(kind, H):
    """dh non-zero at one step t* only: dgi[t] (and the GRU's dghn[t]) is exactly zero for t > t* and for t < t* with a
    wipe in wipe[t .. t*-1], and dstate0 is exactly zero where a wipe precedes t*."""
    n = 300
    X, wipe, s0, dh, params = inputs(kind, H, 14, n, seed=H)
    for ts in (0, 2, T - 1):
        d = torch.zeros_like(dh)
        d[ts] = dh[ts]
        _, _, dgi, dghn, ds0 = raw(kind, X, wipe, s0, d, params)
        steps = torch.arange(T, device="cuda")[:, None]
        # the last wipe before t* (-1: none); step t's gradient is cut where t <= that wipe
        before = torch.where(wipe[:ts], steps[:ts], -1).max(0).values if ts else torch.full((n,), -1, device="cuda")
        dead = (steps > ts) | (steps <= before[None])                         # [T, N]
        for name, v in (("dgi", dgi), ("dghn", dghn)):
            if v is not None:
                assert bool((v.transpose(1, 2)[dead] == 0).all()), (name, ts)
                assert bool((v.transpose(1, 2)[~dead] != 0).any()), (name, ts)
        cut = before >= 0
        assert bool((ds0[cut] == 0).all()), ts
        if bool((~cut).any()):
            assert bool((ds0[~cut] != 0).any()), ts


@pytest.mark.parametrize("kind,H", STRUCT, ids=["%s-H%d" % s for s in STRUCT])
def test_last_wipe_changes_nothing(kind, H):
    X, wipe, s0, dh, params = inputs(kind, H, 14, 300, seed=H + 1)
    a = raw(kind, X, wipe, s0, dh, params)
    flipped = wipe.clone()
    flipped[-1] = ~flipped[-1]
    b = raw(kind, X, flipped, s0, dh, params)
    for name, x, y in zip(("h", "gates", "dgi", "dghn", "dstate0"), a, b):
        assert (x is None and y is None) or torch.equal(x, y), name


@pytest.mark.parametrize("kind,H", STRUCT, ids=["%s-H%d" % s for s in STRUCT])
def test_every_step_wiped_equals_single_steps(kind, H):
    """With every step wiped, the T-step launches equal T launches of T = 1 bit for bit: step 0 from the real state0,
    every later step from a zero state."""
    X, wipe, s0, dh, params = inputs(kind, H, 14, 129, seed=H + 2)
    wipe[:] = True
    h, gates, dgi, dghn, ds0 = raw(kind, X, wipe, s0, dh, params)
    for t in range(T):
        st = s0 if t == 0 else torch.zeros_like(s0)
        h1, g1, dgi1, dghn1, ds01 = raw(kind, X[t:t + 1].contiguous(), wipe[t:t + 1].contiguous(), st,
                                         dh[t:t + 1].contiguous(), params)
        assert torch.equal(h1[0], h[t]) and torch.equal(g1[0], gates[t]), t
        assert torch.equal(dgi1[0], dgi[t]), t
        if dghn is not None:
            assert torch.equal(dghn1[0], dghn[t]), t
        if t == 0:
            assert torch.equal(ds01, ds0)


# ---------------------------------------------------------------------------------------------------------------
# PolicyPopulation.unroll
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,H,width,E", [("gru", 17, 8, 128), ("lstm", 33, 0, 64)])
def test_population_unroll_gradients(kind, H, width, E):
    """Gradients of PolicyPopulation.unroll on every member's modules equal, bit for bit, that member's own unroll over
    member_slice(out, m), and meet the float64 criterion of test_rnn_unroll_gpu."""
    from metagym_b200 import PolicyPopulation
    M = 3
    N = E * M
    env = make_env(N)
    D = env._obs[0].numel()
    pop = PolicyPopulation([make_policy(kind, D, H, width, True, "episode", True, True, seed=10 + m) for m in range(M)])
    st = torch.randn((N, pop.state_dim), generator=torch.Generator(device="cuda").manual_seed(1), device="cuda") * 0.5
    env.rollout(5, policy=pop, state=st, act_seed=1)
    out = env.rollout(16, policy=pop, state=st, act_seed=2, want_hidden=True)
    g = torch.Generator(device="cuda").manual_seed(11)
    weights = [torch.randn((16, N, 4), generator=g, device="cuda"), torch.randn((16, N), generator=g, device="cuda"),
               torch.randn((16, N), generator=g, device="cuda")]
    mods = [[mm for mm in (p._cell, p._head, p._value)] for p in pop.policies]
    params = [q for ms in mods for mm in ms for q in mm.parameters()]
    res = pop.unroll(out, True)
    gp = torch.autograd.grad(sum((r * w).sum() for r, w in zip(res, weights)), params)
    k = 0
    for m, p in enumerate(pop.policies):
        sl = slice(m * E, (m + 1) * E)
        wm = [w[:, sl] for w in weights]
        om = pop.member_slice(out, m)
        gf = grads(p, om, lambda o: p.unroll(o, True), wm, False)
        mine = [x.double() for x in gp[k:k + len(gf)]]
        k += len(gf)
        for a, b in zip(mine, gf):
            assert torch.equal(a, b), m
        gr = grads(p, om, lambda o: p._unroll_reference(o, True), wm, False)
        p64 = f64_twin(p)
        g64 = grads(p64, om, lambda o: p64._unroll_reference(o, True), [w.double() for w in wm], False)
        for j, (a, r, ref) in enumerate(zip(gf, gr, g64)):
            ef, er = float((a - ref).abs().max()), float((r - ref).abs().max())
            assert ef <= 4 * er + 1e-6 * (1. + float(ref.abs().max())), (m, j, ef, er)
    assert k == len(params)
    env.close()
