"""GPU: the fused unroll of GRUPolicy / LSTMPolicy (mgb_rnn_seq_forward / mgb_rnn_seq_backward through
metagym_b200.cell_seq; DESIGN.md "Fused unroll").

1. Forward: h equals the rollout's hid bit for bit (with and without saving for the backward), and logp / value match
   the kernel's; with normalisation, h lies within the header's float32 bound of a float64 cell on the same inputs.
2. Gradients of every cell, head and value-head parameter and of state0, against float64 autograd through
   _unroll_reference: no worse than 4x the float32 torch loop's error.
3. Two eager runs give bit-identical gradients; a forward + backward captured in one CUDA graph replays them bit for
   bit, also after an optimiser step on the cell.
4. Under no_grad nothing is saved.
5. Fallback past the footprint, every C refusal with its outputs untouched, the footprint boundary against a restated
   byte count.
6. Offsets past 2^31 elements against a twin run on an env slice.
"""
import copy
import ctypes

import pytest
import torch
from torch import nn

from test_maze2d_resample_rollout_gpu import CFG, slot_table
import test_lstm_policy_rollout_maze_gpu as lstm_tests
import test_rnn_policy_rollout_maze_gpu as gru_tests

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = (0xbeef << 32) | 5


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    pass


def make_env(N, k=None, max_steps=5, view_grid=1):
    import numpy as np
    from metagym_b200 import BatchedMetaMaze2D
    table, _ = slot_table(7, N)
    env = BatchedMetaMaze2D(num_envs=N, squeeze=False, auto_reset=True, max_steps=max_steps, view_grid=view_grid,
                            episodes_per_task=k)
    env.set_task(table, env2task=np.arange(N))
    env.reset()
    return env


def make_policy(kind, D, H=16, width=0, feedback=True, reset="episode", bias=True, value=False, seed=0, mean=None,
                std=None):
    from metagym_b200 import GRUPolicy, LSTMPolicy
    g = torch.Generator().manual_seed(seed)
    cell = (nn.GRUCell if kind == "gru" else nn.LSTMCell)(D + 5 * feedback, H, bias=bias)
    head = nn.Linear(H, 4) if not width else nn.Sequential(nn.Linear(H, width), nn.Tanh(), nn.Linear(width, 4))
    vh = nn.Linear(width or H, 1) if value else None
    mods = [cell, head] + ([vh] if vh is not None else [])
    with torch.no_grad():
        for m in mods:
            for p in m.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * (1.5 / p.shape[-1] ** 0.5 if p.dim() == 2 else 0.3))
    for m in mods:
        m.cuda()
    cls = GRUPolicy if kind == "gru" else LSTMPolicy
    return cls(cell, head, feedback=feedback, hidden_reset=reset, obs_mean=mean, obs_std=std, device="cuda", value=vh)


def collect(env, pol, T, mode="none", state=None, act_seed=3):
    """A rollout dict with hid; mode: "none", "resample" (in-launch resampling) or a trial handle's resampling."""
    st = pol.initial_state(env.num_envs) if state is None else state
    rs = dict(seed=SEED, **CFG) if mode != "none" else None
    return env.rollout(T, policy=pol, state=st, act_seed=act_seed, want_hidden=True, resample=rs), st


def fused(pol, out, save):
    """(h, gates or None) of the cell over out's inputs, through the forward kernel directly."""
    from metagym_b200 import cell_seq
    obs, act, rew, wipe, state0 = pol._unroll_inputs(out)
    X = pol._cell_input(obs, act, rew, wipe, state0).transpose(1, 2).contiguous()
    c = pol._cell
    with torch.no_grad():
        params = cell_seq._packed(c.weight_ih, c.weight_hh, c.bias_ih, c.bias_hh)
        return cell_seq.forward(pol._cell_code, pol.hidden, params, X, wipe.contiguous(),
                                state0[:, :pol._memory * pol.hidden].contiguous(), save)


# (kind, H, head width, feedback, reset, collection, value head, bias, N)
CASES = [
    ("gru", 64, 0, True, "episode", "none", False, True, 200),
    ("gru", 5, 8, False, "task", "resample", True, True, 130),
    ("gru", 17, 0, True, "task", "trial", True, True, 256),
    ("gru", 1, 8, True, "episode", "resample", True, False, 1),
    ("lstm", 64, 0, True, "episode", "none", True, True, 200),
    ("lstm", 1, 8, False, "task", "resample", False, True, 129),
    ("lstm", 5, 8, True, "task", "trial", True, True, 256),
    ("lstm", 64, 0, True, "episode", "resample", True, False, 1),
]
IDS = ["-".join(str(v) for v in c) for c in CASES]


def case_setup(case, T=12, seed=0):
    kind, H, width, fb, reset, mode, value, bias, N = case
    env = make_env(N, k=2 if mode == "trial" else None)
    pol = make_policy(kind, env._obs[0].numel(), H, width, fb, reset, bias, value, seed)
    # a non-zero state0 carried from a previous launch
    st = pol.initial_state(N)
    collect(env, pol, 7, mode, state=st, act_seed=1)
    out, _ = collect(env, pol, T, mode, state=st, act_seed=2)
    return env, pol, out


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_forward_bit_exact_against_the_rollout(case):
    env, pol, out = case_setup(case)
    assert bool(out["state0"].abs().sum() > 0)
    for save in (False, True):
        h, _ = fused(pol, out, save)
        assert torch.equal(h, out["hid"]), save
    res = pol.unroll(out, value=pol.has_value)
    assert res[1].requires_grad
    assert float((res[1].detach() - out["logp"]).abs().max()) < 1e-4
    if pol.has_value:
        assert float((res[2].detach() - out["value"]).abs().max()) < 1e-4
    env.close()


@pytest.mark.parametrize("T", [1, 9])
@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_edge_wipes_and_T1(kind, T):
    """T = 1, and wipes at t = 0, at t = T-1, everywhere and nowhere on synthetic inputs: the forward equals a rollout-
    free restatement of the reset rule through the same kernel cell stepwise (the T = 1 launch per step)."""
    from metagym_b200 import cell_seq
    N, D, H = 300, 9, 12
    pol = make_policy(kind, D, H, seed=3)
    G = torch.Generator(device="cuda").manual_seed(4)
    nm = pol._memory * H
    for pattern in ("t0", "last", "all", "none", "random"):
        wipe = torch.zeros((T, N), dtype=torch.bool, device="cuda")
        if pattern == "t0":
            wipe[0] = True
        elif pattern == "last":
            wipe[-1] = True
        elif pattern == "all":
            wipe[:] = True
        elif pattern == "random":
            wipe = torch.rand((T, N), generator=G, device="cuda") < 0.3
        X = torch.randn((T, D + 5, N), generator=G, device="cuda")
        s0 = torch.randn((N, nm), generator=G, device="cuda")
        with torch.no_grad():
            h = cell_seq.run(pol._cell, pol._cell_code, X, wipe, s0)
            # one launch per step, the memory carried and wiped here
            mem = s0.clone()
            for t in range(T):
                ht, gates = cell_seq.forward(pol._cell_code, H, cell_seq._packed(
                    pol._cell.weight_ih, pol._cell.weight_hh, pol._cell.bias_ih, pol._cell.bias_hh),
                    X[t:t + 1].contiguous(), wipe[t:t + 1].contiguous(), mem, save=True)
                assert torch.equal(ht[0], h[t]), (pattern, t)
                new = ht[0] if kind == "gru" else torch.cat([ht[0], gates[0, 4].T], 1)
                mem = new.masked_fill(wipe[t][:, None], 0.).contiguous()


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_normalised_forward_within_the_float32_bound(kind):
    """With obs_mean / obs_std the rollout folds the normalisation into the weights and unroll normalises in torch, so h
    is checked teacher-forced against a float64 cell on the fused path's own inputs, to the header's bound."""
    env = make_env(200)
    D = env._obs[0].numel()
    g = torch.Generator().manual_seed(8)
    pol = make_policy(kind, D, 24, 8, True, "episode", True, True, seed=6, mean=torch.rand(D, generator=g),
                      std=0.5 + torch.rand(D, generator=g))
    out, _ = collect(env, pol, 10)
    obs, act, rew, wipe, state0 = pol._unroll_inputs(out)
    x = pol._cell_input(obs, act, rew, wipe, state0).double()
    h, gates = fused(pol, out, True)
    c = pol._cell
    Wi, Wh = c.weight_ih.double(), c.weight_hh.double()
    bi, bh = c.bias_ih.double(), c.bias_hh.double()
    H = pol.hidden
    hp = state0[:, :H].double()
    cp = state0[:, H:2 * H].double() if kind == "lstm" else None
    worst = 0.
    for t in range(h.shape[0]):
        if t:
            hp = h[t - 1].double().masked_fill(wipe[t - 1][:, None], 0.)
            if kind == "lstm":
                cp = gates[t - 1, 4].T.double().masked_fill(wipe[t - 1][:, None], 0.)
        if kind == "gru":
            ref, bound = gru_tests.gru_bound(Wi, Wh, bi, bh, x[t], hp)
        else:
            ref, bound, _, _ = lstm_tests.lstm_bound(Wi, Wh, bi, bh, x[t], hp, cp, torch.zeros_like(cp))
        worst = max(worst, float(((h[t].double() - ref).abs() / bound).max()))
    assert worst <= 1.0, worst
    _, logp = pol.unroll(out)
    assert float((logp.detach() - out["logp"]).abs().max()) < 1e-3
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. gradients
# ---------------------------------------------------------------------------------------------------------------------
def loss_of(res, weights):
    return sum((r * w).sum() for r, w in zip(res, weights))


def grads(pol, out, fn, weights, state_grad):
    params = [p for m in pol_modules(pol) for p in m.parameters()]
    o = dict(out)
    if state_grad:
        o["state0"] = out["state0"].to(params[0].dtype).clone().requires_grad_()
    res = fn(o)
    gs = torch.autograd.grad(loss_of(res, weights), params + ([o["state0"]] if state_grad else []))
    gs = [g.double() for g in gs]
    if state_grad:
        gs[-1] = gs[-1][:, :pol._memory * pol.hidden]      # the feedback columns are data
    return gs


def pol_modules(pol):
    return [pol._cell, pol._head] + ([pol._value] if pol.has_value else [])


def f64_twin(pol):
    cls = type(pol)
    cell, head = copy.deepcopy(pol._cell).double(), copy.deepcopy(pol._head).double()
    vh = copy.deepcopy(pol._value).double() if pol.has_value else None
    return cls(cell, head, feedback=pol.feedback, hidden_reset=pol.hidden_reset, device="cuda", value=vh)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_gradients_against_float64(case):
    env, pol, out = case_setup(case, T=16)
    T, N = out["act"].shape
    g = torch.Generator(device="cuda").manual_seed(11)
    weights = [torch.randn((T, N, 4), generator=g, device="cuda"), torch.randn((T, N), generator=g, device="cuda")]
    if pol.has_value:
        weights.append(torch.randn((T, N), generator=g, device="cuda"))
    v = pol.has_value
    p64 = f64_twin(pol)
    w64 = [w.double() for w in weights]
    for state_grad in (False, True):
        gf = grads(pol, out, lambda o: pol.unroll(o, v), weights, state_grad)
        gr = grads(pol, out, lambda o: pol._unroll_reference(o, v), weights, state_grad)
        g64 = grads(p64, out, lambda o: p64._unroll_reference(o, v), w64, state_grad)
        assert len(gf) == len(gr) == len(g64)
        for k, (a, r, ref) in enumerate(zip(gf, gr, g64)):
            ef, er = float((a - ref).abs().max()), float((r - ref).abs().max())
            floor = 1e-6 * (1. + float(ref.abs().max()))
            assert ef <= 4 * er + floor, (k, state_grad, ef, er)
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. determinism and graph capture
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_deterministic_and_graph_capture(kind):
    env = make_env(300)
    pol = make_policy(kind, env._obs[0].numel(), 32, 8, True, "episode", True, True, seed=9)
    out, _ = collect(env, pol, 12)
    params = [p for m in pol_modules(pol) for p in m.parameters()]
    T, N = out["act"].shape
    g = torch.Generator(device="cuda").manual_seed(12)
    weights = [torch.randn((T, N, 4), generator=g, device="cuda"), torch.randn((T, N), generator=g, device="cuda"),
               torch.randn((T, N), generator=g, device="cuda")]

    def step():
        return torch.autograd.grad(loss_of(pol.unroll(out, True), weights), params)

    a, b = step(), step()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    assert all(torch.equal(x, y) for x, y in zip(captured, a))
    opt = torch.optim.SGD(pol._cell.parameters(), lr=0.05)
    for p, gp in zip(pol._cell.parameters(), a):
        p.grad = gp.clone()
    opt.step()
    eager = step()
    assert not torch.equal(eager[0], a[0])
    graph.replay()
    assert all(torch.equal(x, y) for x, y in zip(captured, eager))
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. no grad
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_no_grad_saves_nothing(kind):
    env = make_env(512)
    pol = make_policy(kind, env._obs[0].numel(), 64, 0, True, "episode", True, True, seed=2)
    out, _ = collect(env, pol, 16)
    with torch.no_grad():
        pol.unroll(out, True)        # library workspaces of the first calls
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.no_grad():
        res = pol.unroll(out, True)
    torch.cuda.synchronize()
    grown = torch.cuda.memory_allocated() - before
    allowed = sum(-(-r.untyped_storage().nbytes() // 512) * 512 for r in res)
    assert not any(r.requires_grad for r in res)
    assert grown <= allowed, (grown, allowed)
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. fallback, refusals, footprint
# ---------------------------------------------------------------------------------------------------------------------
def synthetic_out(pol, T, N, g):
    D = pol.obs_dim
    return {"obs0": torch.randn((N, D), generator=g, device="cuda"),
            "obs": torch.randn((T, N, D), generator=g, device="cuda"),
            "act": torch.randint(0, 4, (T, N), generator=g, device="cuda", dtype=torch.int32),
            "rew": torch.randn((T, N), generator=g, device="cuda", dtype=torch.float64),
            "done": torch.rand((T, N), generator=g, device="cuda") < 0.2,
            "state0": torch.randn((N, pol.state_dim), generator=g, device="cuda")}


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_fallback_beyond_the_footprint(kind):
    from metagym_b200 import cell_seq
    pol = make_policy(kind, 400, 64, seed=1)
    assert not cell_seq.fits(pol._cell)
    out = synthetic_out(pol, 5, 70, torch.Generator(device="cuda").manual_seed(1))
    a, b = pol.unroll(out), pol._unroll_reference(out)
    assert torch.equal(a[1], b[1]) and a[1].requires_grad


def seq_buffers(kind, H, n_in, T=3, n=5):
    from metagym_b200 import _lib
    G = 3 if kind == "gru" else 4
    HC = H if kind == "gru" else 2 * H
    S = 4 if kind == "gru" else 5
    f = lambda *s: torch.full(s, 7.25, device="cuda")          # noqa: E731
    bufs = dict(params=torch.randn(G * H * (n_in + H + 2), device="cuda") * 0.1, x=torch.randn((T, n_in, n), device="cuda"),
                wipe=torch.zeros((T, n), dtype=torch.uint8, device="cuda"), state0=torch.randn((n, HC), device="cuda"),
                h=f(T, n, H), gates=f(T, S, H, n), dh=torch.randn((T, n, H), device="cuda"), dgi=f(T, G * H, n),
                dghn=f(T, H, n), dstate0=f(n, HC))
    seq = _lib.RnnSeq(_lib.RNN_CELL_GRU if kind == "gru" else _lib.RNN_CELL_LSTM, H, n_in, T, n,
                      *[bufs[k].data_ptr() for k in ("params", "x", "wipe", "state0", "h", "gates", "dh", "dgi",
                                                     "dghn", "dstate0")])
    return seq, bufs


def call(name, seq):
    from metagym_b200 import _lib
    lib = _lib.load()
    rc = getattr(lib, name)(ctypes.byref(seq) if seq is not None else None,
                            _lib.current_stream(torch, torch.device("cuda", 0)))
    torch.cuda.synchronize()
    return rc, lib.mgb_last_error().decode()


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_refusals_touch_nothing(kind):
    outs = {"mgb_rnn_seq_forward": ("h", "gates"), "mgb_rnn_seq_backward": ("dgi", "dghn", "dstate0")}
    bad = [("cell", 7), ("hidden", 0), ("hidden", 65), ("in_", 0), ("T", 0), ("n", 0), ("params_dev", None),
           ("wipe_dev", None), ("state0_dev", None)]
    per_call = {"mgb_rnn_seq_forward": bad + [("x_dev", None), ("h_dev", None)],
                "mgb_rnn_seq_backward": bad + [("gates_dev", None), ("dh_dev", None), ("dgi_dev", None),
                                               ("dstate0_dev", None)]
                + ([("dghn_dev", None), ("h_dev", None)] if kind == "gru" else [])}
    for name, cases in per_call.items():
        assert call(name, None)[0] == MGB_ERR_ARG
        for field, val in cases:
            seq, bufs = seq_buffers(kind, 8, 6)
            setattr(seq, field, val)
            rc, msg = call(name, seq)
            assert rc == MGB_ERR_ARG, (name, field)
            assert name in msg
            for k in outs[name]:
                assert bool((bufs[k] == 7.25).all()), (name, field, k)
    seq, bufs = seq_buffers(kind, 8, 6)
    assert call("mgb_rnn_seq_forward", seq)[0] == 0
    assert call("mgb_rnn_seq_backward", seq)[0] == 0


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_footprint_boundary(kind):
    from metagym_b200 import cell_seq
    G = 3 if kind == "gru" else 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    n_in = 300
    fit = max(H for H in range(1, 65) if cell_seq.smem_bytes(G, H, n_in)[0] <= optin)
    assert fit < 64
    seq, bufs = seq_buffers(kind, fit, n_in)
    assert call("mgb_rnn_seq_forward", seq)[0] == 0
    seq, bufs = seq_buffers(kind, fit + 1, n_in)
    rc, msg = call("mgb_rnn_seq_forward", seq)
    assert rc == MGB_ERR_ARG and ("needs %d bytes" % cell_seq.smem_bytes(G, fit + 1, n_in)[0]) in msg, msg
    assert bool((bufs["h"] == 7.25).all())
    cells = [(nn.GRUCell if kind == "gru" else nn.LSTMCell)(n_in, H).cuda() for H in (fit, fit + 1)]
    assert cell_seq.fits(cells[0]) and not cell_seq.fits(cells[1])


# ---------------------------------------------------------------------------------------------------------------------
# 6. large offsets
# ---------------------------------------------------------------------------------------------------------------------
def test_offsets_past_2_31_against_an_env_slice():
    """LSTM H = 64, T = 8, N = 2^20 + 1000: the saved gates hold 2.7e9 floats and dgi 2.15e9.  The last envs' h, gates,
    dgi and dstate0 equal those of a twin run on that slice, bit for bit."""
    T, N, H, n_in, m = 8, 2 ** 20 + 1000, 64, 14, 300
    free, _ = torch.cuda.mem_get_info()
    if free < 32 * 2 ** 30:
        pytest.skip("needs 32 GiB of free device memory")
    from metagym_b200 import _lib, cell_seq
    g = torch.Generator(device="cuda").manual_seed(5)
    cell = nn.LSTMCell(n_in, H).cuda()
    params = cell_seq._packed(cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh).detach()

    def run(X, wipe, s0, dh):
        h, gates = cell_seq.forward(_lib.RNN_CELL_LSTM, H, params, X, wipe, s0, save=True)
        dgi = torch.empty((T, 4 * H, X.shape[2]), device="cuda")
        ds0 = torch.empty_like(s0)
        seq = cell_seq._struct(_lib.RNN_CELL_LSTM, H, params, X, wipe, s0, h, gates)
        seq.dh_dev, seq.dgi_dev, seq.dstate0_dev = dh.data_ptr(), dgi.data_ptr(), ds0.data_ptr()
        cell_seq._call(_lib.load().mgb_rnn_seq_backward, seq, X.device)
        sl = slice(X.shape[2] - m, X.shape[2])
        return h[:, sl].clone(), gates[..., sl].clone(), dgi[..., sl].clone(), ds0[sl].clone()

    X = torch.randn((T, n_in, N), generator=g, device="cuda")
    wipe = torch.rand((T, N), generator=g, device="cuda") < 0.2
    s0 = torch.randn((N, 2 * H), generator=g, device="cuda")
    dh = torch.randn((T, N, H), generator=g, device="cuda")
    big = run(X, wipe, s0, dh)
    small = run(X[..., -m:].contiguous(), wipe[:, -m:].contiguous(), s0[-m:].contiguous(), dh[:, -m:].contiguous())
    del X, dh
    for a, b in zip(big, small):
        assert torch.equal(a, b)
