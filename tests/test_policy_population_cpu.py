"""CPU: PolicyPopulation's packing, row views and refusals, and the population entry points of the C ABI."""
import ctypes
import os
import re

import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def mlp(seed, widths=(64, 64), D=19):
    g = torch.Generator().manual_seed(seed)
    dims = [D] + list(widths) + [4]
    layers = []
    for k in range(len(dims) - 1):
        layers += [nn.Linear(dims[k], dims[k + 1]), nn.Tanh()]
    m = nn.Sequential(*layers[:-1])
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
    return m


def test_rows_are_the_members_packs_and_views():
    from metagym_b200.policy import MLPPolicy, PolicyPopulation
    pols = [MLPPolicy(mlp(s), log_std=[0.1 * s] * 4, obs_mean=[0.5 * s] * 19, device="cpu") for s in range(3)]
    pop = PolicyPopulation(pols)
    assert pop.params.shape == (3, pols[0].numel) and pop.member_stride == pols[0].numel
    for m, p in enumerate(pols):
        assert torch.equal(pop.params[m], p.pack())
        assert p.params.data_ptr() == pop.params[m].data_ptr()
    pols[1].update(mlp(9))
    assert torch.equal(pop.params[1], pols[1].pack())
    assert pop.struct().params_dev == pop.params.data_ptr()


def test_rows_equal_parameters_to_vector():
    from metagym_b200.policy import GRUPolicy, LSTMPolicy, MLPPolicy, PolicyPopulation
    m = mlp(1)
    pop = PolicyPopulation.from_template(MLPPolicy(m, log_std=[0.1, 0.2, 0.3, 0.4], device="cpu"), 3)
    want = torch.cat([nn.utils.parameters_to_vector(m.parameters()), torch.tensor([0.1, 0.2, 0.3, 0.4])])
    for r in range(3):
        assert torch.equal(pop.params[r], want.float())
    for kind, cell in ((GRUPolicy, nn.GRUCell(14, 16)), (LSTMPolicy, nn.LSTMCell(14, 16))):
        head = nn.Sequential(nn.Linear(16, 8), nn.ReLU(), nn.Linear(8, 4))
        pop = PolicyPopulation.from_template(kind(cell, head, device="cpu"), 2)
        want = nn.utils.parameters_to_vector(list(cell.parameters()) + list(head.parameters()))
        assert torch.equal(pop.params[1], want)
        assert pop.initial_state(64).shape == (64, pop.state_dim)


def test_member_slice():
    from metagym_b200.policy import MLPPolicy, PolicyPopulation
    pop = PolicyPopulation.from_template(MLPPolicy(mlp(0), device="cpu"), 4)
    out = {"obs": torch.arange(2 * 128 * 3).reshape(2, 128, 3), "done": torch.zeros(2, 128), "obs0": torch.arange(128),
           "resampled": True}
    s = pop.member_slice(out, 2)
    assert torch.equal(s["obs"], out["obs"][:, 64:96]) and torch.equal(s["obs0"], out["obs0"][64:96])
    assert s["resampled"] is True and pop.envs_per_member(128) == 32
    assert torch.equal(pop.member_slice(torch.arange(128), 1), torch.arange(32, 64))


def test_population_refusals():
    from metagym_b200.policy import GRUPolicy, MLPPolicy, PolicyPopulation
    a = MLPPolicy(mlp(0), device="cpu")
    with pytest.raises(ValueError, match="at least one"):
        PolicyPopulation([])
    with pytest.raises(ValueError, match="one shape"):
        PolicyPopulation([a, MLPPolicy(mlp(1, (64, 32)), device="cpu")])
    with pytest.raises(ValueError, match="one shape"):
        PolicyPopulation([a, MLPPolicy(mlp(1), log_std=[0.0] * 4, device="cpu")])
    with pytest.raises(ValueError, match="every member"):
        PolicyPopulation([GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), device="cpu"), a])
    with pytest.raises(ValueError, match="once"):
        PolicyPopulation([a, a])
    with pytest.raises(ValueError, match="takes MLPPolicy"):
        PolicyPopulation([object()])
    g1 = GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), device="cpu")
    with pytest.raises(ValueError, match="one shape"):
        PolicyPopulation([g1, GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), hidden_reset="task", device="cpu")])
    pop = PolicyPopulation.from_template(a, 4)
    with pytest.raises(ValueError, match="multiple of it"):
        pop.envs_per_member(102)
    with pytest.raises(ValueError, match="envs per member"):
        pop.check_envs(64, 64)                      # E = 16
    with pytest.raises(ValueError, match="envs per member"):
        PolicyPopulation.from_template(a, 2).check_envs(192, 128)      # E = 96
    assert pop.check_envs(128, 128) == 32 and PolicyPopulation([a]).check_envs(7, 64) == 7
    with pytest.raises(ValueError, match="carries no state"):
        pop.initial_state(4)


def test_population_abi():
    from metagym_b200 import _lib
    src = open(os.path.join(ROOT, "include", "mgb200.h")).read()
    consts = dict(re.findall(r"#define (MGB_\w+) (\d+)", src))
    assert int(consts["MGB_POLICY_MEMBER_WARP"]) == _lib.POLICY_MEMBER_WARP == 32
    assert int(consts["MGB_QUAD_POLICY_CTA_ENVS"]) == _lib.QUAD_POLICY_CTA_ENVS == 64
    assert int(consts["MGB_MAZE2D_POLICY_CTA_ENVS"]) == _lib.MAZE2D_POLICY_CTA_ENVS == 128
    vp, i32, i64, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64
    pol, rnn, cfg = ctypes.POINTER(_lib.Policy), ctypes.POINTER(_lib.RnnPolicy), ctypes.POINTER(_lib.MazeSamplerCfg)
    S = _lib.SIGNATURES
    # each is the existing call with (members, member_stride) after the policy pointer
    for new, old, pt in (("mgb_quad_rollout_population", "mgb_quad_rollout_policy", pol),
                         ("mgb_maze_rollout_population", "mgb_maze_rollout_policy", pol),
                         ("mgb_maze_rollout_rnn_population", "mgb_maze_rollout_rnn", rnn)):
        args, base = S[new][1], S[old][1]
        assert args[:3] == [vp, i32, pt] and args[3:5] == [i32, i64] and args[5:] == base[3:], new
        assert S[new][0] is ctypes.c_int
        assert re.search(r"int %s\(mgb_\w+ \*h, int32_t T, const mgb_\w*policy \*pol, int32_t members,\s*"
                         r"int64_t member_stride," % new, src), new
    assert S["mgb_maze_rollout_population"][1][5:7] == [u64, cfg]
