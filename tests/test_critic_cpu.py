"""CPU: value heads (packing, refusals, population shapes), the mgb_critic ABI struct, and the float32 GAE restatement
against float64 textbook GAE."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

from critic_ref import gae_f32, gae_f64

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def seeded(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
    return module


def mlp(seed, widths=(64, 64), D=19):
    dims = [D] + list(widths) + [4]
    layers = []
    for k in range(len(dims) - 1):
        layers += [nn.Linear(dims[k], dims[k + 1]), nn.Tanh()]
    return seeded(nn.Sequential(*layers[:-1]), seed)


@pytest.mark.parametrize("widths", [(64, 64), (7,), ()])
def test_mlp_value_row_packs_at_row_4_before_log_std(widths):
    from metagym_b200.policy import MLPPolicy
    k = widths[-1] if widths else 19
    mean, std = np.linspace(-1, 1, 19), np.linspace(0.5, 2, 19)
    val = seeded(nn.Linear(k, 1), 7)
    plain = MLPPolicy(mlp(1, widths), log_std=[0.1, 0.2, 0.3, 0.4], obs_mean=mean, obs_std=std, device="cpu")
    critic = MLPPolicy(mlp(1, widths), log_std=[0.1, 0.2, 0.3, 0.4], obs_mean=mean, obs_std=std, device="cpu",
                       value=val)
    assert critic.has_value and not plain.has_value
    assert critic.numel == plain.numel + k + 1
    a, b = plain.pack(), critic.pack()
    head = plain.numel - 4 - 4 * (k + 1)               # where the output layer starts
    assert torch.equal(a[:head], b[:head])             # the hidden layers are untouched
    W, bias = b[head:head + 5 * k].reshape(5, k), b[head + 5 * k:head + 5 * k + 5]
    assert torch.equal(W[:4].reshape(-1), a[head:head + 4 * k]) and torch.equal(bias[:4], a[head + 4 * k:head + 4 * k + 4])
    Wv = val.weight.detach().double()
    bv = val.bias.detach().double()
    if not widths:        # the normalisation folds into the value row as into the others
        m64, s64 = torch.tensor(mean), torch.tensor(std)
        bv = bv - Wv @ (m64 / s64)
        Wv = Wv / s64
    assert torch.equal(W[4], Wv[0].float()) and torch.equal(bias[4:], bv.float())
    assert torch.equal(b[-4:], torch.tensor([0.1, 0.2, 0.3, 0.4]))        # log_std still follows


def test_mlp_without_value_packs_as_before():
    from metagym_b200.policy import MLPPolicy
    m = mlp(3)
    p = MLPPolicy(m, log_std=[0.0] * 4, device="cpu")
    lin = [x for x in m if isinstance(x, nn.Linear)]
    ref = torch.cat([torch.cat([l.weight.detach().reshape(-1), l.bias.detach()]) for l in lin] + [torch.zeros(4)])
    assert torch.equal(p.pack(), ref)


def test_mlp_evaluate_matches_the_module():
    from metagym_b200.policy import MLPPolicy
    m, v = mlp(4, (16,)), seeded(nn.Linear(16, 1), 5)
    p = MLPPolicy(m, device="cpu", value=v, obs_mean=[0.25] * 19, obs_std=[2.0] * 19)
    x = torch.randn(3, 5, 19)
    out, val = p.evaluate(x)
    z = m[1](m[0]((x - 0.25) / 2.0))
    assert out.shape == (3, 5, 4) and val.shape == (3, 5)
    assert torch.allclose(out, m[2](z)) and torch.allclose(val, v(z)[..., 0])


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("head_width", [0, 12])
def test_recurrent_value_row(kind, head_width):
    from metagym_b200.policy import GRUPolicy, LSTMPolicy
    H, D = 10, 9
    cls, cell = (GRUPolicy, nn.GRUCell) if kind == "gru" else (LSTMPolicy, nn.LSTMCell)
    head = nn.Linear(H, 4) if not head_width else nn.Sequential(nn.Linear(H, head_width), nn.ReLU(),
                                                                nn.Linear(head_width, 4))
    c, head = seeded(cell(D + 5, H), 1), seeded(head, 2)
    k = head_width or H
    val = seeded(nn.Linear(k, 1), 3)
    a = cls(c, head, device="cpu").pack()
    b = cls(c, head, device="cpu", value=val).pack()
    n_out = 4 * (k + 1)
    assert b.numel() == a.numel() + k + 1
    assert torch.equal(a[:-n_out], b[:-(n_out + k + 1)])
    W, bias = b[-5 * (k + 1):-5].reshape(5, k), b[-5:]
    assert torch.equal(W[:4].reshape(-1), a[-n_out:-4]) and torch.equal(bias[:4], a[-4:])
    assert torch.equal(W[4], val.weight.detach()[0]) and torch.equal(bias[4:], val.bias.detach())


def test_bad_value_heads_are_refused():
    from metagym_b200.policy import GRUPolicy, LSTMPolicy, MLPPolicy
    for bad in (nn.Linear(64, 2), nn.Linear(19, 1), nn.Sequential(nn.Linear(64, 1)), "value"):
        with pytest.raises(ValueError):
            MLPPolicy(mlp(0), device="cpu", value=bad)
    with pytest.raises(ValueError):
        MLPPolicy(mlp(0, ()), device="cpu", value=nn.Linear(64, 1))      # no hidden layer: k is obs_dim
    head = nn.Sequential(nn.Linear(8, 6), nn.Tanh(), nn.Linear(6, 4))
    with pytest.raises(ValueError):
        GRUPolicy(nn.GRUCell(14, 8), head, device="cpu", value=nn.Linear(8, 1))   # the head reads 6
    with pytest.raises(ValueError):
        LSTMPolicy(nn.LSTMCell(14, 8), nn.Linear(8, 4), device="cpu", value=nn.Linear(6, 1))
    plain = MLPPolicy(mlp(0), device="cpu")
    with pytest.raises(ValueError):
        plain.update(value=nn.Linear(64, 1))
    critic = MLPPolicy(mlp(0), device="cpu", value=nn.Linear(64, 1))
    with pytest.raises(ValueError):
        critic.update(value=nn.Linear(32, 1))
    v2 = seeded(nn.Linear(64, 1), 9)
    critic.update(value=v2)
    assert torch.equal(critic.params[-4 - 1:-4], v2.bias.detach())


def test_population_shape_includes_the_value_head():
    from metagym_b200.policy import GRUPolicy, MLPPolicy, PolicyPopulation
    with_v = [MLPPolicy(mlp(s), device="cpu", value=nn.Linear(64, 1)) for s in range(2)]
    without = MLPPolicy(mlp(5), device="cpu")
    pop = PolicyPopulation(with_v)
    assert pop.has_value and pop.numel == with_v[0].numel
    with pytest.raises(ValueError, match="value head"):
        PolicyPopulation(with_v[:1] + [without])
    assert not PolicyPopulation([without]).has_value
    t = PolicyPopulation.from_template(MLPPolicy(mlp(1), device="cpu", value=nn.Linear(64, 1)), 3)
    assert t.has_value and all(p.has_value for p in t.policies)
    assert torch.equal(t.params[2], t.params[0])
    g = [GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), device="cpu", value=nn.Linear(8, 1)) for _ in range(2)]
    assert PolicyPopulation(g).has_value
    with pytest.raises(ValueError):
        PolicyPopulation([g[0], GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), device="cpu")])


def test_gae_without_a_value_head_is_refused():
    from metagym_b200.policy import MLPPolicy, critic_args
    assert critic_args(MLPPolicy(mlp(0), device="cpu"), None) is None
    with pytest.raises(ValueError, match="value head"):
        critic_args(MLPPolicy(mlp(0), device="cpu"), (0.99, 0.95))
    assert critic_args(MLPPolicy(mlp(0), device="cpu", value=nn.Linear(64, 1)), (0.99, 0.95)) == (
        pytest.approx(0.99), pytest.approx(0.95))


def test_critic_struct_layout_matches_header():
    from metagym_b200 import _lib
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "c.c"), os.path.join(d, "c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "mgb200.h"\n'
                    'int main(void){printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(mgb_critic),'
                    'offsetof(mgb_critic,value_dev),offsetof(mgb_critic,value_last_dev),'
                    'offsetof(mgb_critic,final_value_dev),offsetof(mgb_critic,adv_dev),offsetof(mgb_critic,ret_dev),'
                    'offsetof(mgb_critic,gamma),offsetof(mgb_critic,lambda));return 0;}\n')
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    C = _lib.Critic
    assert got == [ctypes.sizeof(C), C.value_dev.offset, C.value_last_dev.offset, C.final_value_dev.offset,
                   C.adv_dev.offset, C.ret_dev.offset, C.gamma.offset, C.lam.offset]


def test_critic_entry_points_are_declared():
    from metagym_b200 import _lib
    for name in ("mgb_quad_rollout_critic", "mgb_maze_rollout_critic", "mgb_maze_rollout_rnn_critic"):
        res, args = _lib.SIGNATURES[name]
        assert args[-2] is not None and args[-2]._type_ is _lib.Critic


def random_chunk(rng, T, N, task_rule):
    rew = rng.normal(size=(T, N))
    done = rng.random((T, N)) < 0.15
    truncated = done & (rng.random((T, N)) < 0.5)
    # the task rule wipes only where the env drew a new maze: a subset of done
    cut = done & (rng.random((T, N)) < 0.4) if task_rule else done
    value = rng.normal(size=(T, N)).astype(np.float32)
    value_last = rng.normal(size=N).astype(np.float32)
    final_value = np.where(cut & truncated, rng.normal(size=(T, N)), np.nan).astype(np.float32)
    return rew, cut, truncated, value, value_last, final_value


@pytest.mark.parametrize("task_rule", [False, True])
@pytest.mark.parametrize("gamma,lam", [(0.99, 0.95), (1.0, 1.0), (0.0, 0.5), (0.9, 0.0)])
def test_gae_f32_restatement_against_float64(task_rule, gamma, lam):
    rng = np.random.default_rng(int(gamma * 100 + lam * 10 + task_rule))
    args = random_chunk(rng, 32, 257, task_rule)
    adv, ret = gae_f32(*args, gamma, lam)
    adv64, ret64 = gae_f64(*args, gamma, lam)
    assert adv.dtype == np.float32 and np.isfinite(adv).all()       # NaN final values are never read
    scale = 1.0 + np.abs(adv64)
    assert np.max(np.abs(adv - adv64) / scale) < 1e-5
    assert np.max(np.abs(ret - ret64) / (1.0 + np.abs(ret64))) < 1e-5


def test_gae_restatement_cuts_and_bootstraps():
    # one env, T = 3: a truncated cut at t = 1 bootstraps from final_value, nothing flows back across it
    rew = np.array([[1.0], [2.0], [4.0]])
    cut = np.array([[False], [True], [False]])
    trunc = np.array([[False], [True], [False]])
    value = np.array([[0.5], [0.25], [0.125]], np.float32)
    final_value = np.array([[np.nan], [8.0], [np.nan]], np.float32)
    adv, ret = gae_f32(rew, cut, trunc, value, np.array([16.0], np.float32), final_value, 0.5, 0.5)
    a2 = 4.0 + 0.5 * 16.0 - 0.125
    a1 = 2.0 + 0.5 * 8.0 - 0.25
    a0 = 1.0 + 0.5 * 0.25 - 0.5 + 0.25 * a1
    assert adv[:, 0].tolist() == [a0, a1, a2] and ret[:, 0].tolist() == [a0 + 0.5, a1 + 0.25, a2 + 0.125]
    trunc[1] = False        # ended, not truncated: no bootstrap
    adv, _ = gae_f32(rew, cut, trunc, value, np.array([16.0], np.float32), final_value, 0.5, 0.5)
    assert adv[1, 0] == 2.0 - 0.25
