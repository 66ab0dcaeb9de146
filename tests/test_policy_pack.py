"""CPU: MLPPolicy packs a torch MLP into the layout the policy rollouts read (include/mgb200.h, mgb_policy), folds the
observation normalisation into the first layer, and refuses modules the kernels cannot run."""
import ctypes
import os
import subprocess
import tempfile

import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unpacked_forward(buf, obs_dim, widths, act, x):
    """Forward pass read straight from the packed layout: per layer W [out, in] row-major then b [out], first hidden
    layer to the 4-wide output layer, then log_std [4].  float64."""
    buf = buf.to(torch.float64)
    o, h = 0, x.to(torch.float64)
    dims = [obs_dim] + list(widths) + [4]
    for k in range(len(dims) - 1):
        i, j = dims[k], dims[k + 1]
        W = buf[o:o + i * j].reshape(j, i)
        o += i * j
        b = buf[o:o + j]
        o += j
        h = h @ W.T + b
        if k < len(dims) - 2:
            h = torch.tanh(h) if act == "tanh" else torch.relu(h)
    assert o + 4 == buf.numel()
    return h, buf[o:]


@pytest.mark.parametrize("widths,act", [([], "tanh"), ([64, 64], "tanh"), ([7], "relu"), ([64, 3, 17], "relu")])
def test_pack_reproduces_the_module(widths, act):
    from metagym_b200.policy import MLPPolicy
    torch.manual_seed(0)
    dims = [19] + widths + [4]
    layers = []
    for k in range(len(dims) - 1):
        layers.append(nn.Linear(dims[k], dims[k + 1]))
        if k < len(dims) - 2:
            layers.append(nn.Tanh() if act == "tanh" else nn.ReLU())
    m = nn.Sequential(*layers)
    ls = torch.tensor([-0.5, 0.0, 0.25, -1.0])
    p = MLPPolicy(m, log_std=ls, device="cpu")
    assert p.params.dtype == torch.float32 and p.params.numel() == sum(
        dims[k + 1] * (dims[k] + 1) for k in range(len(dims) - 1)) + 4
    # with no normalisation the layout is a single torch.cat of the module's flattened parameters and log_std
    assert torch.equal(p.params, torch.cat([t.detach().reshape(-1) for t in m.parameters()] + [ls]))
    x = torch.randn(33, 19)
    y, ls_packed = unpacked_forward(p.params, 19, widths, act, x)
    assert torch.allclose(y, m.double()(x.double()), rtol=0, atol=1e-12)
    m.float()
    assert torch.equal(ls_packed.float(), ls)
    assert p.struct().n_hidden == len(widths) and list(p.struct().width)[:len(widths)] == widths


def test_normalisation_is_folded_into_the_first_layer():
    from metagym_b200.policy import MLPPolicy
    torch.manual_seed(1)
    m = nn.Sequential(nn.Linear(9, 16), nn.Tanh(), nn.Linear(16, 4)).double()
    mean, std = torch.randn(9, dtype=torch.float64), torch.rand(9, dtype=torch.float64) + 0.5
    p = MLPPolicy(m.float(), obs_mean=mean, obs_std=std, device="cpu")
    x = torch.randn(50, 9, dtype=torch.float64) * 3
    y, _ = unpacked_forward(p.params, 9, [16], "tanh", x)
    ref = m.double()((x - mean) / std)
    # the folded weights are rounded once to float32: relative 2^-24 per weight, over 9 + 16 terms of size ~1
    assert torch.allclose(y, ref, rtol=0, atol=1e-5), (y - ref).abs().max()
    # update() keeps the buffer (a captured graph reads the same address) and the earlier normalisation
    addr = p.params.data_ptr()
    with torch.no_grad():
        m[0].weight.mul_(2.0)
    p.update(m.float())
    assert p.params.data_ptr() == addr
    y2, _ = unpacked_forward(p.params, 9, [16], "tanh", x)
    assert torch.allclose(y2, m.double()((x - mean) / std), rtol=0, atol=1e-5)


def test_refused_modules():
    from metagym_b200.policy import MLPPolicy
    bad = [
        nn.Linear(19, 4),                                                       # not a Sequential
        nn.Sequential(nn.Linear(19, 8), nn.Tanh()),                             # ends in an activation
        nn.Sequential(nn.Linear(19, 8), nn.Tanh(), nn.Linear(8, 3)),            # 3 outputs
        nn.Sequential(nn.Linear(19, 65), nn.Tanh(), nn.Linear(65, 4)),          # width 65
        nn.Sequential(nn.Linear(19, 8), nn.Tanh(), nn.Linear(8, 8), nn.ReLU(), nn.Linear(8, 4)),    # mixed activations
        nn.Sequential(nn.Linear(19, 8), nn.Sigmoid(), nn.Linear(8, 4)),         # unsupported activation
        nn.Sequential(*sum([[nn.Linear(8 if k else 19, 8), nn.Tanh()] for k in range(4)], []), nn.Linear(8, 4)),  # 4 hidden
        nn.Sequential(nn.Linear(19, 8), nn.Tanh(), nn.Linear(7, 4)),            # widths do not chain
    ]
    for m in bad:
        with pytest.raises(ValueError):
            MLPPolicy(m, device="cpu")
    p = MLPPolicy(nn.Sequential(nn.Linear(19, 8), nn.Tanh(), nn.Linear(8, 4)), device="cpu")
    with pytest.raises(ValueError):
        p.update(nn.Sequential(nn.Linear(19, 9), nn.Tanh(), nn.Linear(9, 4)))
    with pytest.raises(ValueError):
        p.update(log_std=torch.zeros(3))


def test_policy_struct_matches_header():
    from metagym_b200 import _lib
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "s.c")
        open(src, "w").write('#include <stdio.h>\n#include <stddef.h>\n#include "mgb200.h"\nint main(){printf("%zu %zu %zu '
                             '%zu\\n",sizeof(mgb_policy),offsetof(mgb_policy,width),offsetof(mgb_policy,activation),'
                             'offsetof(mgb_policy,mode));return 0;}\n')
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    P = _lib.Policy
    assert got == [ctypes.sizeof(P), P.width.offset, P.activation.offset, P.mode.offset]


def test_policy_draws_restated():
    """The Box-Muller restatement: u1 in (0, 1] keeps every normal finite, and the draws look standard normal."""
    import numpy as np
    from policy_draws import quad_policy_normals
    z = quad_policy_normals(0x123456789ABCDEF0, np.arange(4096) + (1 << 32) - 2048, 7)
    assert z.shape == (4096, 4) and np.isfinite(z).all()
    assert abs(z.mean()) < 0.05 and abs(z.std() - 1.0) < 0.05


def test_normalisation_must_be_finite_and_positive():
    """A zero, negative or non-finite std (or a non-finite mean) would fold into inf / NaN weights: refused, and the
    policy keeps its previous buffer."""
    from metagym_b200.policy import MLPPolicy
    m = nn.Sequential(nn.Linear(3, 4))
    for std in ([1.0, 0.0, 1.0], [1.0, -2.0, 1.0], [1.0, float("inf"), 1.0], [float("nan"), 1.0, 1.0]):
        with pytest.raises(ValueError):
            MLPPolicy(m, obs_std=torch.tensor(std), device="cpu")
    with pytest.raises(ValueError):
        MLPPolicy(m, obs_mean=torch.tensor([0.0, float("inf"), 0.0]), device="cpu")
    p = MLPPolicy(m, obs_std=torch.tensor([1.0, 2.0, 4.0]), device="cpu")
    before = p.params.clone()
    with pytest.raises(ValueError):
        p.update(obs_std=torch.tensor([1.0, 0.0, 1.0]))
    with pytest.raises(ValueError):
        p.update(nn.Sequential(nn.Linear(3, 4)), obs_mean=torch.tensor([float("nan")] * 3))
    assert torch.equal(p.params, before)
