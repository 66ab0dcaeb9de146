"""CPU: LSTMPolicy packs an nn.LSTMCell and its head into the layout the recurrent MetaMaze2D rollout reads
(include/mgb200.h, mgb_rnn_policy with cell = MGB_RNN_CELL_LSTM), folds the observation normalisation into the obs
columns of weight_ih and into bias_ih, refuses modules and arguments the kernel cannot run, and unroll() recomputes a
rollout's logits and log-probabilities with the kernel's input construction and reset rule over the state [h, c,
feedback]."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_head(H, width, act=nn.Tanh):
    if not width:
        return nn.Linear(H, 4)
    return nn.Sequential(nn.Linear(H, width), act(), nn.Linear(width, 4))


def head_linears(head):
    return [head] if isinstance(head, nn.Linear) else [m for m in head if isinstance(m, nn.Linear)]


def hand_packed(cell, head):
    """The packed buffer written out by hand from the header's list: weight_ih [4H][in], weight_hh [4H][H], bias_ih,
    bias_hh (zeros without bias), then each head layer's W and b."""
    H = cell.hidden_size
    z = np.zeros(4 * H)
    parts = [cell.weight_ih.detach().numpy().ravel(), cell.weight_hh.detach().numpy().ravel(),
             cell.bias_ih.detach().numpy() if cell.bias_ih is not None else z,
             cell.bias_hh.detach().numpy() if cell.bias_hh is not None else z]
    for m in head_linears(head):
        parts += [m.weight.detach().numpy().ravel(), m.bias.detach().numpy()]
    return np.concatenate([np.asarray(p, np.float64) for p in parts]).astype(np.float32)


@pytest.mark.parametrize("D,H,feedback,width,bias", [(9, 64, True, 0, True), (25, 17, False, 8, True),
                                                     (9, 1, True, 64, False), (4, 5, False, 0, False)])
def test_pack_order(D, H, feedback, width, bias):
    from metagym_b200 import LSTMPolicy, _lib
    torch.manual_seed(H)
    cell = nn.LSTMCell(D + 5 * feedback, H, bias=bias)
    head = make_head(H, width, nn.ReLU)
    pol = LSTMPolicy(cell, head, feedback=feedback, device="cpu")
    want = hand_packed(cell, head)
    assert pol.numel == want.size
    assert np.array_equal(pol.pack().numpy(), want)
    assert np.array_equal(pol.params.numpy(), want)
    if not bias:        # the bias block is exactly zero
        o = 4 * H * (D + 5 * feedback + H)
        assert not pol.params[o:o + 8 * H].any()
    assert pol.state_dim == 2 * H + 5 * feedback
    s = pol.struct()
    assert (s.hidden, s.feedback, s.reset, s.head_hidden, s.head_width, s.mode, s.cell) == (
        H, int(feedback), 0, int(width > 0), width, 0, _lib.RNN_CELL_LSTM)
    assert s.activation == (1 if width else 0)
    assert pol.struct(deterministic=True).mode == 1
    assert LSTMPolicy(cell, head, feedback=feedback, hidden_reset="task", device="cpu").struct().reset == 1
    st = pol.initial_state(7)
    assert st.shape == (7, 2 * H + 5 * feedback) and st.dtype == torch.float32 and not st.any()


def test_gru_struct_keeps_cell_zero():
    from metagym_b200 import GRUPolicy, _lib
    pol = GRUPolicy(nn.GRUCell(14, 8), make_head(8, 0), device="cpu")
    assert pol.struct().cell == _lib.RNN_CELL_GRU == 0


@pytest.mark.parametrize("feedback", [True, False])
def test_normalisation_fold(feedback):
    from metagym_b200 import LSTMPolicy
    torch.manual_seed(1)
    D, H = 9, 6
    cell, head = nn.LSTMCell(D + 5 * feedback, H), make_head(H, 3)
    mean, std = torch.randn(D, dtype=torch.float64), torch.rand(D, dtype=torch.float64) + 0.5
    pol = LSTMPolicy(cell, head, feedback=feedback, obs_mean=mean, obs_std=std, device="cpu")
    Wi = cell.weight_ih.detach().double().numpy().copy()
    bi = cell.bias_ih.detach().double().numpy() - Wi[:, :D] @ (mean / std).numpy()
    Wi[:, :D] /= std.numpy()
    want = hand_packed(cell, head).astype(np.float64)
    want[:Wi.size] = Wi.ravel()
    o = 4 * H * (D + 5 * feedback + H)
    want[o:o + 4 * H] = bi
    assert np.array_equal(pol.pack().numpy(), want.astype(np.float32))
    if feedback:        # the feedback columns are left as they are
        assert np.array_equal(pol.pack().numpy()[:Wi.size].reshape(4 * H, -1)[:, D:],
                              cell.weight_ih.detach().numpy()[:, D:])
    # only the std: bias_ih is unchanged
    p2 = LSTMPolicy(cell, head, feedback=feedback, obs_std=std, device="cpu").pack().numpy()
    assert np.array_equal(p2[o:o + 4 * H], cell.bias_ih.detach().numpy())
    # update() repacks into the same buffer
    buf = pol.params
    pol.update(nn.LSTMCell(D + 5 * feedback, H))
    assert pol.params is buf and not np.array_equal(pol.params.numpy(), want.astype(np.float32))


def test_refusals():
    from metagym_b200 import LSTMPolicy
    D, H = 9, 8
    cell, head = nn.LSTMCell(D + 5, H), make_head(H, 4)
    bad = [
        lambda: LSTMPolicy(nn.LSTM(D + 5, H), head, device="cpu"),
        lambda: LSTMPolicy(nn.GRUCell(D + 5, H), head, device="cpu"),
        lambda: LSTMPolicy(cell, head, hidden_reset="never", device="cpu"),
        lambda: LSTMPolicy(cell, head, feedback=2, device="cpu"),
        lambda: LSTMPolicy(nn.LSTMCell(D + 5, 65), make_head(65, 0), device="cpu"),
        lambda: LSTMPolicy(nn.LSTMCell(5, H), head, feedback=True, device="cpu"),
        lambda: LSTMPolicy(cell, make_head(H + 1, 0), device="cpu"),
        lambda: LSTMPolicy(cell, nn.Linear(H, 3), device="cpu"),
        lambda: LSTMPolicy(cell, make_head(H, 65), device="cpu"),
        lambda: LSTMPolicy(cell, nn.Sequential(nn.Linear(H, 4), nn.Tanh(), nn.Linear(4, 4), nn.Tanh(), nn.Linear(4, 4)),
                           device="cpu"),
        lambda: LSTMPolicy(cell, nn.Sequential(nn.Linear(H, 4), nn.Sigmoid(), nn.Linear(4, 4)), device="cpu"),
        lambda: LSTMPolicy(cell, nn.Sequential(nn.Linear(H, 4), nn.Tanh()), device="cpu"),
        lambda: LSTMPolicy(cell, head, obs_mean=torch.zeros(D + 5), device="cpu"),
        lambda: LSTMPolicy(cell, head, obs_std=torch.zeros(D), device="cpu"),
        lambda: LSTMPolicy(cell, head, obs_std=-torch.ones(D), device="cpu"),
        lambda: LSTMPolicy(cell, head, obs_std=torch.full((D,), float("inf")), device="cpu"),
        lambda: LSTMPolicy(cell, head, obs_mean=torch.full((D,), float("nan")), device="cpu"),
    ]
    for k, make in enumerate(bad):
        with pytest.raises(ValueError, match="LSTMPolicy"):
            make()
            print("not refused: case %d" % k)
    with pytest.raises(TypeError):          # the categorical head has no log_std, and LSTMPolicy takes none
        LSTMPolicy(cell, head, log_std=torch.zeros(4), device="cpu")
    pol = LSTMPolicy(cell, head, device="cpu")
    before = pol.params.clone()
    for upd in (lambda: pol.update(nn.LSTMCell(D + 5, H + 1)), lambda: pol.update(nn.LSTMCell(D + 4, H)),
                lambda: pol.update(nn.GRUCell(D + 5, H)),
                lambda: pol.update(head=make_head(H, 5)), lambda: pol.update(head=make_head(H, 4, nn.ReLU)),
                lambda: pol.update(head=make_head(H, 0)), lambda: pol.update(obs_std=torch.zeros(D)),
                lambda: pol.update(nn.LSTMCell(D + 5, H), obs_mean=torch.full((D,), float("nan")))):
        with pytest.raises(ValueError):
            upd()
    assert torch.equal(pol.params, before)


def test_struct_layout_and_constants_match_c():
    from metagym_b200 import _lib
    P = _lib.RnnPolicy
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "s.c"), os.path.join(d, "s")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "mgb200.h"\nint main(void){printf("%zu %zu %d '
                    '%d\\n",sizeof(mgb_rnn_policy),offsetof(mgb_rnn_policy,cell),MGB_RNN_CELL_GRU,MGB_RNN_CELL_LSTM);'
                    'return 0;}\n')
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    assert got == [40, 36, 0, 1]
    assert [ctypes.sizeof(P), P.cell.offset, _lib.RNN_CELL_GRU, _lib.RNN_CELL_LSTM] == got


def restated_unroll(cell, head, feedback, wipe_on_done, mean, std, out):
    """Independent float64 restatement in NumPy, step by step: x_t = [(obs - mean) / std, fb], the LSTM equations
    (gates i, f, g, o of W_ih x + b_ih + W_hh h + b_hh; c' = f c + i g; h' = o tanh(c')), the head, log_softmax; after
    step t the state row becomes zero where done and the reset rule fires, else (h_t, c_t, onehot(a_t), (float)r_t)."""
    f = lambda t: t.detach().double().numpy()                  # noqa: E731
    Wi, Wh, bi, bh = f(cell.weight_ih), f(cell.weight_hh), f(cell.bias_ih), f(cell.bias_hh)
    H = cell.hidden_size
    lins = head_linears(head)
    act_kind = None if isinstance(head, nn.Linear) else type(list(head)[1])
    T, N = out["act"].shape
    obs = np.concatenate([out["obs0"].numpy().reshape(1, N, -1), out["obs"].numpy().reshape(T, N, -1)[:-1]])
    obs = (obs - mean) / std
    st = out["state0"].numpy().astype(np.float64)
    hs, cs, fb = st[:, :H].copy(), st[:, H:2 * H].copy(), st[:, 2 * H:].copy()
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))                   # noqa: E731
    logits, logp = np.zeros((T, N, 4)), np.zeros((T, N))
    for t in range(T):
        for e in range(N):
            x = np.concatenate([obs[t, e], fb[e]]) if feedback else obs[t, e]
            v = Wi @ x + bi + Wh @ hs[e] + bh
            i, fg, g, o = sig(v[:H]), sig(v[H:2 * H]), np.tanh(v[2 * H:3 * H]), sig(v[3 * H:])
            c = fg * cs[e] + i * g
            h = o * np.tanh(c)
            y = h
            for k, m in enumerate(lins):
                y = f(m.weight) @ y + f(m.bias)
                if k < len(lins) - 1:
                    y = np.tanh(y) if act_kind is nn.Tanh else np.maximum(y, 0)
            a = int(out["act"][t, e])
            mx = y.max()
            logits[t, e] = y
            logp[t, e] = y[a] - (mx + np.log(np.exp(y - mx).sum()))
            if out["done"][t, e] and wipe_on_done:
                hs[e], cs[e], fb[e] = 0.0, 0.0, 0.0
            else:
                hs[e], cs[e] = h, c
                if feedback:
                    fb[e] = np.concatenate([np.eye(4)[a], [float(np.float32(out["rew"][t, e]))]])
    return logits, logp


def fake_rollout(T, N, D, S, resampled, seed):
    g = torch.Generator().manual_seed(seed)
    done = (torch.rand((T, N), generator=g) < 0.2).to(torch.uint8)
    done[T // 2, :] = 1                                     # every env resets mid-chunk
    return {"obs0": torch.randint(-1, 2, (N, D), generator=g).float(),
            "obs": torch.randint(-1, 2, (T, N, D), generator=g).float(),
            "act": torch.randint(0, 4, (T, N), generator=g).int(),
            "rew": torch.randn((T, N), generator=g, dtype=torch.float64) * 0.3,
            "done": done,
            "state0": torch.randn((N, S), generator=g),
            "resampled": resampled}


@pytest.mark.parametrize("feedback", [True, False], ids=["feedback", "no_feedback"])
@pytest.mark.parametrize("reset,resampled", [("episode", False), ("episode", True), ("task", False), ("task", True)])
@pytest.mark.parametrize("width,act", [(0, nn.Tanh), (6, nn.ReLU)])
def test_unroll_against_restatement(feedback, reset, resampled, width, act):
    from metagym_b200 import LSTMPolicy
    torch.manual_seed(7)
    D, H, T, N = 9, 5, 12, 6
    cell, head = nn.LSTMCell(D + 5 * feedback, H).double(), make_head(H, width, act).double()
    mean, std = np.linspace(-0.3, 0.3, D), np.linspace(0.5, 1.5, D)
    pol = LSTMPolicy(cell, head, feedback=feedback, hidden_reset=reset, obs_mean=mean, obs_std=std, device="cpu")
    out = fake_rollout(T, N, D, pol.state_dim, resampled, seed=3)
    logits, logp = pol.unroll(out)
    assert logits.shape == (T, N, 4) and logp.shape == (T, N) and logits.dtype == torch.float64
    wipe = reset == "episode" or resampled
    ref_logits, ref_logp = restated_unroll(cell, head, feedback, wipe, mean, std, out)
    assert np.abs(logits.detach().numpy() - ref_logits).max() < 1e-12
    assert np.abs(logp.detach().numpy() - ref_logp).max() < 1e-12
    # the reset rule matters here: the other rule gives other logits after the first done
    other, _ = restated_unroll(cell, head, feedback, not wipe, mean, std, out)
    assert np.abs(other - ref_logits).max() > 1e-6
    # the carried c matters: a state0 with another c gives other logits
    out2 = dict(out, state0=out["state0"].clone())
    out2["state0"][:, H:2 * H] += 1.0
    assert np.abs(pol.unroll(out2)[0].detach().numpy() - ref_logits).max() > 1e-6
    # gradients reach every cell and head parameter
    (logp.sum() + logits.pow(2).sum()).backward()
    for name, p in list(cell.named_parameters()) + list(head.named_parameters()):
        assert p.grad is not None and p.grad.abs().sum() > 0, name
