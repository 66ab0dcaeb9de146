"""GPU: quadrotor rollouts driven by an on-device MLP policy (mgb_quad_rollout_policy, BatchedQuadrotor.rollout(policy=)).

Env side: bit for bit the open-loop rollout fed the actions the policy took.  Policy side: the actions and their
log-probabilities against a float64 torch forward pass of the same module on the observations the policy saw, with
the Gaussian draws restated from the Philox stream (tests/policy_draws.py).
"""
import ctypes
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from policy_draws import quad_policy_normals  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = 0x9E3779B97F4A7C15          # both 32-bit halves set
TASKS = ("velocity_control", "no_collision", "hovering_control")


def make_env(n, task, nt=40, base=0, auto_reset=True, final_obs=True, rng_seed=5):
    from metagym_b200 import BatchedQuadrotor
    kw = dict(seed=[0, 1, 2]) if task == "velocity_control" else {}
    return BatchedQuadrotor(task=task, dt=0.005, nt=nt, num_envs=n, device=0, squeeze=False, auto_reset=auto_reset,
                            final_obs=final_obs, rng_seed=rng_seed, env_index_base=base, **kw)


def make_module(D, widths=(64, 64), act=nn.Tanh, seed=0):
    g = torch.Generator().manual_seed(seed)
    dims = [D] + list(widths) + [4]
    layers = []
    for k in range(len(dims) - 1):
        lin = nn.Linear(dims[k], dims[k + 1])
        with torch.no_grad():
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) / math.sqrt(dims[k]))
            lin.bias.copy_(torch.randn(lin.bias.shape, generator=g) * 0.1)
        layers.append(lin)
        if k < len(dims) - 2:
            layers.append(act())
    with torch.no_grad():
        layers[-1].bias.add_(7.5)           # mid-range voltages, so that episodes last
    return nn.Sequential(*layers)


def make_policy(env, widths=(64, 64), act=nn.Tanh, seed=0, log_std=(-0.5, 0.0, 0.3, -1.0)):
    from metagym_b200.policy import MLPPolicy
    m = make_module(env.obs_dim, widths, act, seed)
    return m, MLPPolicy(m, log_std=torch.tensor(log_std), device=env.device)


def forward_bound(module, x):
    """float64 forward pass and a running bound on the float32 kernel's error.  Each output of a layer with `in` inputs
    is a chain of `in` fused multiply-adds from the bias: its rounding error is at most (in + 1) 2^-24 (|W| |x| + |b|)
    (standard bound for recursive summation, u = 2^-24).  An input error e propagates as |W| e (tanh and relu are
    1-Lipschitz), and tanhf adds at most 2 ulp of its result."""
    u = 2.0 ** -24
    h, err = x, torch.zeros_like(x)
    mods = list(module)
    for k in range(0, len(mods), 2):
        lin = mods[k]
        W, b = lin.weight.detach().double().cpu().to(x.device), lin.bias.detach().double().cpu().to(x.device)
        y = h @ W.T + b
        err = (lin.in_features + 1) * u * (h.abs() @ W.abs().T + b.abs()) + err @ W.abs().T
        if k + 1 < len(mods):
            if isinstance(mods[k + 1], nn.Tanh):
                y = torch.tanh(y)
                err = err + 2 * u * y.abs()
            else:
                y = torch.relu(y)
        h = y
    return h, err


def pre_action_obs(out):
    return torch.cat([out["obs0"][None], out["obs"][:-1]], 0)


def check_policy_side(env, module, log_std, out, seed, t0, deterministic=False):
    """act and logp of `out` against the float64 forward pass; returns the worst error relative to its bound."""
    T, N, _ = out["obs"].shape
    mean, bound = forward_bound(module, pre_action_obs(out).double())
    act = out["act"].double()
    genv = env.env_index_base + np.arange(N)
    worst = 0.0
    if deterministic:
        r = (act - mean).abs() / (bound + 2.0 ** -24 * mean.abs())
        return float(r.max())
    ls = torch.as_tensor(log_std, dtype=torch.float64, device=act.device)
    std = torch.exp(ls)
    for t in range(T):
        z = torch.as_tensor(quad_policy_normals(seed, genv, t0 + t), device=act.device)
        want = mean[t] + std * z
        # act = fmaf(expf(ls), z32, mean32): mean error (bound) + expf (1 ulp) and float Box-Muller (a few ulp of z,
        # through logf / sqrtf / sincospif) times std, + the final rounding
        tol = bound[t] + 8 * 2.0 ** -24 * std * (z.abs() + 1) + 2.0 ** -24 * want.abs()
        err = (act[t] - want).abs()
        worst = max(worst, float((err / tol).max()))
        if out.get("logp") is not None:
            lp = torch.distributions.Normal(mean[t], std).log_prob(act[t]).sum(-1)
            # d logp / d act = -(act - mean) / std^2 = -z / std; float32 sum of 4 terms of size z^2/2 + |ls|
            lp_tol = ((z.abs() / std) * tol).sum(-1) + 16 * 2.0 ** -24 * ((z * z / 2 + ls.abs()).sum(-1) + 4)
            lerr = (out["logp"][t].double() - lp).abs()
            worst = max(worst, float((lerr / lp_tol).max()))
    return worst


def assert_env_side_equal(a, b, want_final=True):
    for k in ("obs", "rew", "done"):
        assert torch.equal(a[k], b[k]), k
    if want_final:
        assert torch.equal(a["truncated"], b["truncated"])
        d = a["done"].bool()
        assert torch.equal(a["final_obs"][d], b["final_obs"][d])


@pytest.mark.parametrize("task", TASKS)
def test_env_side_bit_for_bit_and_policy_side(cuda_device, task):
    n, T = 1000, 48
    env = make_env(n, task, nt=30)
    env.reset()
    env.rollout(5)                                   # t_base != 0
    m, pol = make_policy(env)
    ls = (-0.5, 0.0, 0.3, -1.0)
    snap = env.snapshot()
    t0 = env._counters()
    out = env.rollout(T, policy=pol, act_seed=SEED)
    assert out["done"].any(), "no episode ended: auto-reset and final_obs are not exercised"
    env.restore(snap)
    ref = env.rollout(T, actions=out["act"])
    assert_env_side_equal(out, ref)
    worst = check_policy_side(env, m, ls, out, SEED, t0)
    assert worst <= 1.0, worst
    # mean mode
    env.restore(snap)
    det = env.rollout(T, policy=pol, deterministic=True)
    assert det["logp"] is None
    assert check_policy_side(env, m, ls, det, SEED, t0, deterministic=True) <= 1.0
    env.restore(snap)
    assert_env_side_equal(det, env.rollout(T, actions=det["act"]))
    env.close()


def test_relu_and_shapes(cuda_device):
    """ReLU, no hidden layer, three hidden layers of odd widths, and widths 1 and 64."""
    n, T = 300, 8
    env = make_env(n, "velocity_control")
    env.reset()
    for widths, act in (((), nn.ReLU), ((5, 64, 1), nn.ReLU), ((64, 3, 17), nn.Tanh)):
        m, pol = make_policy(env, widths, act, seed=len(widths))
        snap = env.snapshot()
        t0 = env._counters()
        out = env.rollout(T, policy=pol, act_seed=3)
        assert check_policy_side(env, m, (-0.5, 0.0, 0.3, -1.0), out, 3, t0) <= 1.0, widths
        env.restore(snap)
        assert_env_side_equal(out, env.rollout(T, actions=out["act"]))
    env.close()


def test_continuity(cuda_device):
    n, T = 257, 16
    env = make_env(n, "velocity_control", nt=20)
    obs = env.reset().clone()
    m, pol = make_policy(env)
    snap = env.snapshot()
    a = env.rollout(T, policy=pol, act_seed=SEED)
    assert torch.equal(a["obs0"], obs)                           # obs0 is what reset() returned
    b = env.rollout(T, policy=pol, act_seed=SEED)
    assert torch.equal(b["obs0"], a["obs"][-1])                  # ... and the last obs of the preceding rollout
    env.restore(snap)
    ab = env.rollout(2 * T, policy=pol, act_seed=SEED)           # two calls of T = one call of 2T
    for k in ("act", "logp", "obs", "rew", "done", "truncated"):
        assert torch.equal(ab[k], torch.cat([a[k], b[k]])), k
    env.restore(snap)                                            # a snapshot replays the rollout exactly
    again = env.rollout(T, policy=pol, act_seed=SEED)
    for k in ("act", "logp", "obs0", "obs", "rew", "done"):
        assert torch.equal(again[k], a[k]), k
    # after a step(): obs0 is the observation step() returned (auto-reset envs: the fresh episode's)
    o, _, _, _ = env.step(torch.full((n, 4), 7.0, device=env.device))
    o = o.clone()
    assert torch.equal(env.rollout(1, policy=pol)["obs0"], o)
    env.close()


@pytest.mark.parametrize("n,T", [(130, 1), (1000, 24)])
def test_sharding(cuda_device, n, T):
    """One handle of n envs = two handles of n/2 with env_index_base offsets, across genv = 2^32."""
    base = (1 << 32) - n // 2 - 3
    whole = make_env(n, "velocity_control", base=base)
    halves = [make_env(n // 2, "velocity_control", base=base + k * (n // 2)) for k in range(2)]
    m, pol = make_policy(whole)
    outs = []
    for env in [whole] + halves:
        env.reset()
        outs.append(env.rollout(T, policy=pol, act_seed=SEED))
    for k in ("act", "logp", "obs", "rew", "done", "truncated"):
        assert torch.equal(outs[0][k], torch.cat([outs[1][k], outs[2][k]], 1)), k
    assert torch.equal(outs[0]["obs0"], torch.cat([outs[1]["obs0"], outs[2]["obs0"]]))
    assert check_policy_side(whole, m, (-0.5, 0.0, 0.3, -1.0), outs[0], SEED, 0) <= 1.0
    for env in [whole] + halves:
        env.close()


def test_graph_sees_updated_weights(cuda_device):
    n, T = 512, 8
    env = make_env(n, "hovering_control")
    env.reset()
    m, pol = make_policy(env)
    D = env.obs_dim
    dev = env.device
    out = {"obs": torch.empty((T, n, D), device=dev), "rew": torch.empty((T, n), device=dev),
           "done": torch.empty((T, n), dtype=torch.uint8, device=dev), "act": torch.empty((T, n, 4), device=dev),
           "logp": torch.empty((T, n), device=dev), "obs0": torch.empty((n, D), device=dev),
           "final_obs": torch.empty((T, n, D), device=dev), "truncated": torch.empty((T, n), dtype=torch.uint8, device=dev)}
    env.rollout(T, policy=pol, act_seed=1, out=out)              # warm-up
    snap = env.snapshot()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.rollout(T, policy=pol, act_seed=1, out=out)
    m2 = make_module(D, seed=11)
    pol.update(m2, log_std=torch.tensor([0.1, -0.2, 0.0, -2.0]))
    env.restore(snap)
    g.replay()
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in out.items()}
    env.restore(snap)
    eager = env.rollout(T, policy=pol, act_seed=1)
    for k in ("act", "logp", "obs0", "obs", "rew", "done", "truncated"):
        assert torch.equal(got[k], eager[k]), k
    assert check_policy_side(env, m2, (0.1, -0.2, 0.0, -2.0), got, 1, snap["counters"][0].item()) <= 1.0
    env.close()


def _state(env):
    """(step counter, launch count, state records); the snapshot itself is one more launch"""
    return (env._counters(), env.launch_count, env.snapshot()["records"].cpu().clone())


def test_refusals_leave_the_handle_untouched(cuda_device):
    from metagym_b200 import _lib
    from metagym_b200.policy import MLPPolicy
    n, T = 128, 4
    env = make_env(n, "velocity_control")
    env.reset()
    m, pol = make_policy(env)
    D, dev = env.obs_dim, env.device
    f = lambda *s: torch.empty(s, device=dev)                         # noqa: E731
    logp, obs0 = f(T, n), f(n, D)
    lib = env._lib

    def call(p, T=T, logp_out=None, final=None):
        return lib.mgb_quad_rollout_policy(env._h, T, ctypes.byref(p) if p is not None else None, 0, None,
                                           _lib.ptr(logp_out), _lib.ptr(obs0), None, None, None, _lib.ptr(final), None,
                                           env._stream())

    before = _state(env)
    good = pol.struct()
    assert call(good, T=0) == MGB_ERR_ARG and call(good, T=-1) == MGB_ERR_ARG
    assert call(None) == MGB_ERR_ARG
    bad = []
    p = pol.struct(); p.params_dev = None; bad.append(p)
    p = pol.struct(); p.n_hidden = 4; bad.append(p)
    p = pol.struct(); p.n_hidden = -1; bad.append(p)
    p = pol.struct(); p.width[1] = 65; bad.append(p)
    p = pol.struct(); p.width[0] = 0; bad.append(p)
    p = pol.struct(); p.activation = 2; bad.append(p)
    p = pol.struct(); p.mode = 2; bad.append(p)
    for p in bad:
        assert call(p) == MGB_ERR_ARG
    assert call(pol.struct(deterministic=True), logp_out=logp) == MGB_ERR_ARG
    assert "MGB_POLICY_SAMPLE" in lib.mgb_last_error().decode()
    for arm in (lambda: env.set_mirrors([16]), lambda: env.set_multicast(16)):
        arm()
        assert call(good) == MGB_ERR_ARG
        env.set_mirrors([])
    torch.cuda.synchronize()
    after = _state(env)
    assert after[0] == before[0] and after[1] == before[1] + 1 and torch.equal(before[2], after[2])
    # final_obs needs auto_reset
    plain = make_env(n, "no_collision", auto_reset=False, final_obs=False)
    plain.reset()
    mp, pp = make_policy(plain)
    assert plain._lib.mgb_quad_rollout_policy(plain._h, T, ctypes.byref(pp.struct()), 0, None, None, None, None, None,
                                              None, _lib.ptr(f(T, n, D)), None, plain._stream()) == MGB_ERR_ARG
    # Python refusals
    with pytest.raises(ValueError):
        env.rollout(T, actions=torch.zeros((T, n, 4), device=dev), policy=pol)
    with pytest.raises(ValueError):
        env.rollout(T, policy=MLPPolicy(make_module(D + 1), log_std=torch.zeros(4), device=dev))
    with pytest.raises(ValueError):
        env.rollout(T, policy=MLPPolicy(make_module(D), device=dev))        # sampling without log_std
    assert env.rollout(T, policy=MLPPolicy(make_module(D), device=dev), deterministic=True)["logp"] is None
    last = _state(env)
    assert last[0] == after[0] + T and last[1] == after[1] + 2          # the snapshot and the last call ran
    env.close()
    plain.close()
