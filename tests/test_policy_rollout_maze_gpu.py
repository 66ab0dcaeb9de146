"""GPU: MetaMaze2D rollouts driven by an on-device MLP policy with a categorical head (mgb_maze_rollout_policy,
BatchedMetaMaze2D.rollout(policy=, resample=)).

Env side: bit for bit the open-loop rollout (mgb_maze_rollout, with a sampler cfg for `resample`) fed the
actions the policy took, path recording included.  Policy side: the actions against the inverse-CDF draw restated in
float64 from a torch forward pass of the same module on the windows the policy saw and the Philox uniforms of
tests/policy_draws.py; the log-probabilities against log_softmax.
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from policy_draws import maze_policy_uniforms  # noqa: E402
from test_maze_final_obs_gpu import MAX_STEPS, tasks, textures  # noqa: E402,F401  (fixtures)
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = 0x9E3779B97F4A7C15          # both 32-bit halves set
NEAR = 1e-5                        # a draw this close to a CDF boundary may fall on either side in float32


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def make_env(n, task_type="SURVIVAL", view_grid=1, base=0, record_path=False, final_obs=True, auto_reset=True):
    from metagym_b200 import BatchedMetaMaze2D
    return BatchedMetaMaze2D(max_steps=MAX_STEPS, task_type=task_type, view_grid=view_grid, num_envs=n, squeeze=False,
                             auto_reset=auto_reset, final_obs=final_obs, env_index_base=base, record_path=record_path)


def make_module(D, widths=(64, 64), act=nn.Tanh, seed=0, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    dims = [D] + list(widths) + [4]
    layers = []
    for k in range(len(dims) - 1):
        lin = nn.Linear(dims[k], dims[k + 1])
        with torch.no_grad():
            lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) * scale / dims[k] ** 0.5)
            lin.bias.copy_(torch.randn(lin.bias.shape, generator=g) * 0.1)
        layers.append(lin)
        if k < len(dims) - 2:
            layers.append(act())
    return nn.Sequential(*layers)


def make_policy(env, widths=(64, 64), act=nn.Tanh, seed=0):
    from metagym_b200.policy import MLPPolicy
    m = make_module(env._obs[0].numel(), widths, act, seed)
    return m, MLPPolicy(m, device=env.device)


def check_policy_side(env, module, out, seed, t0, deterministic=False):
    """-> (worst logp error relative to its bound, number of action mismatches, all of them near a CDF boundary)."""
    T, N = out["act"].shape
    pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, N, -1).double()
    logits, bound = forward_bound(module, pre)
    act = out["act"].long()
    b = bound.max(-1).values
    if deterministic:
        top2 = logits.topk(2, -1).values
        clear = (top2[..., 0] - top2[..., 1]) > 2 * b + 1e-6
        want = logits.argmax(-1)
        assert torch.equal(act[clear], want[clear])
        return 0.0, int((~clear).sum())
    genv = env.env_index_base + np.arange(N)
    worst, mism = 0.0, 0
    for t in range(T):
        u = torch.as_tensor(maze_policy_uniforms(seed, genv, t0 + t), device=act.device)
        cdf = torch.softmax(logits[t], -1).cumsum(-1)[:, :3]
        want = torch.where(u[:, None] < cdf, torch.arange(3, device=act.device), 3).min(-1).values
        bad = act[t] != want
        if bad.any():
            # the float32 softmax of logits within `bound` of the float64 ones moves c_k by far less than NEAR
            near = (u[:, None] - cdf).abs().min(-1).values < NEAR
            assert bool(near[bad].all()), "an action differs away from every CDF boundary"
            mism += int(bad.sum())
        if out.get("logp") is not None:
            lsm = torch.log_softmax(logits[t], -1)
            lp = lsm.gather(-1, act[t][:, None])[:, 0]
            # logp = (l_a - max) - logf(sum of 4 expf): twice the logit error, and a few ulp of each float32 term
            mx = logits[t].max(-1).values
            tol = 2 * b[t] + 2.0 ** -24 * (8 * (logits[t].gather(-1, act[t][:, None])[:, 0] - mx).abs() + 32)
            worst = max(worst, float(((out["logp"][t].double() - lp).abs() / tol).max()))
    return worst, mism


def assert_env_side_equal(a, b):
    for k in ("obs", "rew", "done", "truncated"):
        assert torch.equal(a[k], b[k]), k
    d = a["done"].bool()
    assert torch.equal(a["final_obs"][d], b["final_obs"][d])


@pytest.mark.parametrize("record_path", [False, True], ids=["plain", "path"])
@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
def test_env_side_and_policy_side(tasks, task_type, record_path):  # noqa: F811
    n, T = 1000, 40
    env, twin = (make_env(n, task_type, record_path=record_path) for _ in range(2))
    for e in (env, twin):
        e.set_task(tasks)
        e.reset()
        e.rollout(3)                                  # t_base != 0
    m, pol = make_policy(env)
    t0 = env._counters()
    out = env.rollout(T, policy=pol, act_seed=SEED)
    assert out["done"].any(), "no episode ended: auto-reset and final_obs are not exercised"
    ref = twin.rollout(T, actions=out["act"])
    assert_env_side_equal(out, ref)
    if record_path:
        for x, y in zip(env.trajectory(), twin.trajectory()):
            assert torch.equal(x, y)
    worst, mism = check_policy_side(env, m, out, SEED, t0)
    print("near-boundary action mismatches: %d of %d" % (mism, T * n))
    assert worst <= 1.0, worst
    # mean mode
    det = env.rollout(T, policy=pol, deterministic=True)
    assert det["logp"] is None
    _, ties = check_policy_side(env, m, det, SEED, 0, deterministic=True)
    print("near-tie argmaxes not checked: %d" % ties)
    assert_env_side_equal(det, twin.rollout(T, actions=det["act"]))


@pytest.mark.parametrize("record_path", [False, True], ids=["plain", "path"])
def test_resample_against_rollout_resample(record_path):
    n, T = 256, 48
    table, _ = slot_table(9, n)
    env, twin = (make_env(n, "SURVIVAL", record_path=record_path) for _ in range(2))
    for e in (env, twin):
        e.set_task(table, env2task=np.arange(n))
        e.reset()
    m, pol = make_policy(env, seed=3)
    rs = dict(seed=SEED, **CFG)
    out = env.rollout(T, policy=pol, act_seed=11, resample=rs)
    assert out["done"].sum() > 10
    ref = twin.rollout(T, actions=out["act"], resample=rs)
    assert_env_side_equal(out, ref)
    ag, life = env.agent_state()
    ag2, life2 = twin.agent_state()
    assert torch.equal(ag, ag2) and torch.equal(life, life2)
    if record_path:
        for x, y in zip(env.trajectory(), twin.trajectory()):
            assert torch.equal(x, y)
    worst, _ = check_policy_side(env, m, out, 11, 0)
    assert worst <= 1.0
    # the next call continues on the new mazes: obs0 is the last window of this one
    nxt = env.rollout(2, policy=pol, act_seed=11, resample=rs)
    assert torch.equal(nxt["obs0"], out["obs"][-1])


def test_continuity(tasks):  # noqa: F811
    n, T = 257, 16
    env = make_env(n, "SURVIVAL")
    env.set_task(tasks)
    obs = env.reset().clone()
    m, pol = make_policy(env, widths=(5, 64, 1), act=nn.ReLU)
    snap = env.snapshot()
    a = env.rollout(T, policy=pol, act_seed=SEED)
    assert torch.equal(a["obs0"], obs)
    b = env.rollout(T, policy=pol, act_seed=SEED)
    assert torch.equal(b["obs0"], a["obs"][-1])
    env.restore(snap)
    ab = env.rollout(2 * T, policy=pol, act_seed=SEED)
    for k in ("act", "logp", "obs", "rew", "done", "truncated"):
        assert torch.equal(ab[k], torch.cat([a[k], b[k]])), k
    env.restore(snap)
    again = env.rollout(T, policy=pol, act_seed=SEED)
    for k in ("act", "logp", "obs0", "obs", "rew", "done"):
        assert torch.equal(again[k], a[k]), k
    o, _, _, _ = env.step(torch.zeros(n, dtype=torch.int32, device=env.device))
    o = o.clone()
    assert torch.equal(env.rollout(1, policy=pol)["obs0"], o)


@pytest.mark.parametrize("n,T", [(130, 1), (1000, 24)])
def test_sharding(tasks, n, T):  # noqa: F811
    base = (1 << 32) - n // 2 - 3
    envs = [make_env(n, base=base)] + [make_env(n // 2, base=base + k * (n // 2)) for k in range(2)]
    e2t = [np.arange(n) % 4, np.arange(n // 2) % 4, (np.arange(n // 2) + n // 2) % 4]
    m, pol = make_policy(envs[0], seed=5)
    outs = []
    for env, et in zip(envs, e2t):
        env.set_task(tasks, env2task=et)
        env.reset()
        outs.append(env.rollout(T, policy=pol, act_seed=SEED))
    for k in ("act", "logp", "obs", "rew", "done", "truncated"):
        assert torch.equal(outs[0][k], torch.cat([outs[1][k], outs[2][k]], 1)), k
    assert torch.equal(outs[0]["obs0"], torch.cat([outs[1]["obs0"], outs[2]["obs0"]]))
    assert check_policy_side(envs[0], m, outs[0], SEED, 0)[0] <= 1.0


def test_graph_sees_updated_weights(tasks):  # noqa: F811
    n, T = 512, 8
    env = make_env(n, "ESCAPE")
    env.set_task(tasks)
    env.reset()
    m, pol = make_policy(env)
    out = env.rollout(T, policy=pol, act_seed=1)                 # warm-up; its buffers are reused below
    snap = env.snapshot()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.rollout(T, policy=pol, act_seed=1, out=out)
    m2 = make_module(env._obs[0].numel(), seed=11)
    pol.update(m2)
    env.restore(snap)
    g.replay()
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in out.items() if v is not None}
    env.restore(snap)
    eager = env.rollout(T, policy=pol, act_seed=1)
    for k in ("act", "logp", "obs0", "obs", "rew", "done", "truncated"):
        assert torch.equal(got[k], eager[k]), k
    assert check_policy_side(env, m2, got, 1, int(snap["counters"][0]))[0] <= 1.0


def test_policy_refusals_leave_the_handle_untouched(tasks, textures):  # noqa: F811
    from metagym_b200 import BatchedMetaMazeDiscrete3D, _lib
    from metagym_b200.policy import MLPPolicy
    n, T = 128, 4
    env = make_env(n)
    env.set_task(tasks)
    env.reset()
    m, pol = make_policy(env)
    dev = env.device
    logp = torch.empty((T, n), device=dev)
    lib = env._lib

    def call(h, p, T=T, logp_out=None, final=None, cfg=None):
        return lib.mgb_maze_rollout_policy(h, T, ctypes.byref(p) if p is not None else None, 0,
                                           ctypes.byref(cfg) if cfg is not None else None, 0, None, _lib.ptr(logp_out),
                                           None, None, None, None, _lib.ptr(final), None, env._stream())

    def state(e):
        c, lc = e._counters(), e.launch_count
        return c, lc, e.snapshot()["records"].cpu().clone()

    before = state(env)
    good = pol.struct()
    assert call(env._h, good, T=0) == MGB_ERR_ARG and call(env._h, None) == MGB_ERR_ARG
    bad = []
    p = pol.struct(); p.params_dev = None; bad.append(p)
    p = pol.struct(); p.n_hidden = 4; bad.append(p)
    p = pol.struct(); p.width[0] = 65; bad.append(p)
    p = pol.struct(); p.width[1] = 0; bad.append(p)
    p = pol.struct(); p.activation = 7; bad.append(p)
    p = pol.struct(); p.mode = 2; bad.append(p)
    for p in bad:
        assert call(env._h, p) == MGB_ERR_ARG
    assert call(env._h, pol.struct(deterministic=True), logp_out=logp) == MGB_ERR_ARG
    for arm in (lambda: env.set_mirrors([16]), lambda: env.set_multicast(16)):
        arm()
        assert call(env._h, good) == MGB_ERR_ARG
        env.set_mirrors([])
    torch.cuda.synchronize()
    after = state(env)
    assert after[0] == before[0] and after[1] == before[1] + 1 and torch.equal(after[2], before[2])
    # resample where mgb_maze_rollout refuses it: the same reason
    plain = make_env(n, auto_reset=False, final_obs=False)
    plain.set_task(tasks)
    plain.reset()
    cfg, _ = plain._sampler_cfg(seed=1, **CFG)
    assert call(plain._h, good, cfg=cfg) == MGB_ERR_ARG
    why = lib.mgb_last_error().decode().split(": ", 1)[1]
    assert lib.mgb_maze_rollout(plain._h, T, None, 0, None, None, None, None, None, None, ctypes.byref(cfg), 0,
                                plain._stream()) == MGB_ERR_ARG
    assert lib.mgb_last_error().decode().split(": ", 1)[1] == why
    # a 3-D handle
    d3 = BatchedMetaMazeDiscrete3D(resolution=(32, 32), textures=textures, max_steps=MAX_STEPS, num_envs=n,
                                   squeeze=False, auto_reset=True)
    d3.set_task(tasks)
    d3.reset()
    assert call(d3._h, good) == MGB_ERR_ARG
    # observation tiles + weights + activations beyond the opt-in shared memory: a 13 x 13 window with 64-wide layers
    wide = make_env(n, view_grid=6)
    wide.set_task(tasks)
    wide.reset()
    mw, pw = make_policy(wide)
    c0 = wide._counters()
    assert call(wide._h, pw.struct()) == MGB_ERR_ARG
    assert "shared memory" in lib.mgb_last_error().decode() and wide._counters() == c0
    with pytest.raises(_lib.MgbError):
        wide.rollout(T, policy=pw)
    # a 7 x 7 window with the same 64-wide layers fits
    mid = make_env(n, view_grid=3)
    mid.set_task(tasks)
    mid.reset()
    assert mid.rollout(T, policy=make_policy(mid)[1])["act"].shape == (T, n)
    mid.close()
    # Python refusals
    with pytest.raises(ValueError):
        env.rollout(T, actions=torch.zeros((T, n), dtype=torch.int32, device=dev), policy=pol)
    with pytest.raises(ValueError):
        env.rollout(T, policy=MLPPolicy(make_module(10), device=dev))
    for e in (env, plain, d3, wide):
        e.close()
