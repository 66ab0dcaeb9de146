"""CPU: the fused unroll's C ABI (mgb_rnn_seq_forward / mgb_rnn_seq_backward) against include/mgb200.h, and the
vectorised construction of the cell input X and of h_{t-1} (GRUPolicy / LSTMPolicy._cell_input, cell_seq.previous_h)
against the step loop they replace, in float64, with "episode" wipes and with "task" wipes from a trial handle's
new_tasks."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ["cell", "hidden", "in", "T", "n", "params_dev", "x_dev", "wipe_dev", "state0_dev", "h_dev", "gates_dev",
          "dh_dev", "dgi_dev", "dghn_dev", "dstate0_dev"]


def test_signatures_and_constant_match_the_header():
    from metagym_b200 import _lib
    src = open(os.path.join(ROOT, "include", "mgb200.h")).read()
    for name in ("mgb_rnn_seq_forward", "mgb_rnn_seq_backward"):
        assert re.search(r"\bint %s\(const mgb_rnn_seq \*seq, void \*stream\);" % name, src), name
        res, args = _lib.SIGNATURES[name]
        assert res is ctypes.c_int and args == [ctypes.POINTER(_lib.RnnSeq), ctypes.c_void_p]
    assert int(re.search(r"#define MGB_RNN_SEQ_CTA_ENVS (\d+)", src).group(1)) == _lib.RNN_SEQ_CTA_ENVS


def test_struct_layout_matches_the_header():
    from metagym_b200 import _lib
    body = "".join('printf("%%zu ", offsetof(mgb_rnn_seq, %s));' % f for f in FIELDS)
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "s.c")
        open(src, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "mgb200.h"\nint main(){%s'
                             'printf("%%zu\\n", sizeof(mgb_rnn_seq));return 0;}\n' % body)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    names = [f if f != "in" else "in_" for f in FIELDS]
    assert [f[0] for f in _lib.RnnSeq._fields_] == names
    assert got == [getattr(_lib.RnnSeq, f).offset for f in names] + [ctypes.sizeof(_lib.RnnSeq)]


def policy(kind, D, H, feedback, reset):
    from metagym_b200 import GRUPolicy, LSTMPolicy
    torch.manual_seed(0)
    cls, mod = (GRUPolicy, nn.GRUCell) if kind == "gru" else (LSTMPolicy, nn.LSTMCell)
    cell = mod(D + 5 * feedback, H).double()
    return cls(cell, nn.Linear(H, 4).double(), feedback=feedback, hidden_reset=reset, device="cpu")


def rollout_dict(pol, T, N, trial):
    g = torch.Generator().manual_seed(1)
    D = pol.obs_dim
    out = {"obs0": torch.randn((N, D), generator=g), "obs": torch.randn((T, N, D), generator=g),
           "act": torch.randint(0, 4, (T, N), generator=g, dtype=torch.int32),
           "rew": torch.randn((T, N), generator=g, dtype=torch.float64),
           "done": (torch.rand((T, N), generator=g) < 0.3).to(torch.uint8),
           "state0": torch.randn((N, pol.state_dim), generator=g, dtype=torch.float32)}
    if trial:
        out.update(resampled=True, episodes_per_task=2,
                   task_episodes0=torch.randint(0, 2, (N,), generator=g, dtype=torch.int32))
    return out


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("feedback", [True, False])
@pytest.mark.parametrize("reset,trial", [("episode", False), ("task", True), ("task", False)])
def test_vectorised_input_equals_the_step_loop(kind, feedback, reset, trial):
    from metagym_b200 import cell_seq
    from metagym_b200.metamaze import new_tasks
    T, N, H = 9, 37, 6
    pol = policy(kind, 7, H, feedback, reset)
    out = rollout_dict(pol, T, N, trial)
    obs, act, rew, wipe, state0 = pol._unroll_inputs(out)
    want = out["done"].bool() if reset == "episode" else new_tasks(out)
    assert torch.equal(wipe, want)
    if trial:
        assert bool(wipe.any()) and bool((out["done"].bool() & ~wipe).any())
    X = pol._cell_input(obs, act, rew, wipe, state0)
    nm = pol._memory * H
    fb = state0[:, nm:]
    for t in range(T):
        x = torch.cat([obs[t], fb], 1) if feedback else obs[t]
        assert torch.equal(X[t], x), t
        keep = ~wipe[t]
        new_fb = torch.cat([nn.functional.one_hot(act[t], 4).double(), rew[t][:, None]], 1)
        fb = torch.where(keep[:, None], new_fb, torch.zeros_like(new_fb))
    h = torch.randn((T, N, H), dtype=torch.float64)
    hp = cell_seq.previous_h(h, wipe, state0[:, :H])
    assert torch.equal(hp[0], state0[:, :H])
    for t in range(1, T):
        assert torch.equal(hp[t], torch.where(wipe[t - 1][:, None], torch.zeros_like(h[t - 1]), h[t - 1])), t


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_cpu_and_float64_cells_take_the_step_loop(kind):
    from metagym_b200 import cell_seq
    pol = policy(kind, 5, 4, True, "episode")
    assert not cell_seq.fits(pol._cell)
    out = rollout_dict(pol, 6, 11, False)
    a, b = pol.unroll(out), pol._unroll_reference(out)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_footprints_restated():
    from metagym_b200 import cell_seq
    # GRU / LSTM at in = 14, H = 64: DESIGN.md "Fused unroll"
    assert cell_seq.smem_bytes(3, 64, 14) == (134144, 114688)
    assert cell_seq.smem_bytes(4, 64, 14) == (187392, 131072)
    assert cell_seq.smem_bytes(3, 5, 14) == (4 * (3 * 8 * 19 + 48 + 24 * 128), 4 * (3 * 5 * 16 + 10 * 128))
