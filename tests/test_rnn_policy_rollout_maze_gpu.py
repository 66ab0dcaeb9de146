"""GPU: MetaMaze2D rollouts driven by an on-device GRU policy (mgb_maze_rollout_rnn,
BatchedMetaMaze2D.rollout(policy=GRUPolicy, state=)).

Env side: bit for bit the open-loop rollout fed the actions the policy took.  Policy side, teacher-forced: every h_t
the kernel reports lies within the float32 error bound of a float64 GRUCell on the inputs the header's rule gives
(x_t from the window and the feedback of step t - 1, c_t from state0, h_{t-1} and the reset rule); the actions and
log-probabilities are checked against the float64 head on h_t and the Philox uniforms of tests/policy_draws.py.  The
state written back is checked bit for bit.
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from policy_draws import maze_policy_uniforms  # noqa: E402
from test_maze_final_obs_gpu import MAX_STEPS, tasks  # noqa: E402,F401  (fixtures)
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402
from test_policy_rollout_maze_gpu import NEAR, SEED, assert_env_side_equal, make_env  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
U = 2.0 ** -24


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def make_policy(env, H=64, width=0, act=nn.Tanh, feedback=True, reset="episode", seed=0, bias=True):
    from metagym_b200.policy import GRUPolicy
    g = torch.Generator().manual_seed(seed)
    D = env._obs[0].numel()
    cell = nn.GRUCell(D + 5 * feedback, H, bias=bias)
    head = nn.Linear(H, 4) if not width else nn.Sequential(nn.Linear(H, width), act(), nn.Linear(width, 4))
    with torch.no_grad():
        for p in list(cell.parameters()) + list(head.parameters()):
            p.copy_(torch.randn(p.shape, generator=g) * (1.5 / max(p.shape[-1], 1) ** 0.5 if p.dim() == 2 else 0.3))
    return GRUPolicy(cell, head, feedback=feedback, hidden_reset=reset, device=env.device)


def random_state(pol, n, seed=1):
    g = torch.Generator().manual_seed(seed)
    s = torch.randn((n, pol.state_dim), generator=g) * 0.5
    return s.to(pol.device)


def unpack(pol):
    """float64 cell weights and an nn.Sequential head read from the packed float32 buffer (what the kernel reads)."""
    buf = pol.params.double()
    H, n_in = pol.hidden, pol.obs_dim + 5 * pol.feedback
    o = 0

    def take(k):
        nonlocal o
        o += k
        return buf[o - k:o]
    Wi, Wh = take(3 * H * n_in).reshape(3 * H, n_in), take(3 * H * H).reshape(3 * H, H)
    bi, bh = take(3 * H), take(3 * H)
    dims = [H] + ([pol.head_width] if pol.head_width else []) + [4]
    layers = []
    for k in range(len(dims) - 1):
        lin = nn.Linear(dims[k], dims[k + 1]).double().to(buf.device)
        with torch.no_grad():
            lin.weight.copy_(take(dims[k] * dims[k + 1]).reshape(dims[k + 1], dims[k]))
            lin.bias.copy_(take(dims[k + 1]))
        layers.append(lin)
        if k < len(dims) - 2:
            layers.append(nn.ReLU() if pol.activation == 1 else nn.Tanh())
    assert o == buf.numel()
    return Wi, Wh, bi, bh, nn.Sequential(*layers)


def gru_bound(Wi, Wh, bi, bh, x, c):
    """float64 h = GRUCell(x, c) and a bound on the float32 kernel's error, from the header's statement.  An fma chain of
    k terms from its bias errs by at most (k + 1) u (|b| + sum |w| |input|); the float32 add of the two chains adds
    u |v|; sigma(v) = 1 / (1 + expf(-v)) moves by at most |dv| / 4 and adds at most 8 u sigma (expf 2 ulp, one add, one
    division); fmaf(r, gh_n, gi_n) adds u |arg| and tanhf 2 ulp (4 u |n|); h = fmaf(z, c, (1 - z) n) adds a rounding
    to 1 - z, to the product and to the fma."""
    H = c.shape[-1]
    gi, gh = x @ Wi.T + bi, c @ Wh.T + bh
    ei = (x.shape[-1] + 1) * U * (x.abs() @ Wi.abs().T + bi.abs())
    eh = (H + 1) * U * (c.abs() @ Wh.abs().T + bh.abs())
    sl = lambda t, k: t[..., k * H:(k + 1) * H]               # noqa: E731
    gate, egate = [], []
    for k in range(2):
        v = sl(gi, k) + sl(gh, k)
        ev = sl(ei, k) + sl(eh, k) + U * (v.abs() + sl(ei, k) + sl(eh, k))
        s = torch.sigmoid(v)
        gate.append(s)
        egate.append(0.25 * ev + 8 * U * s)
    (r, z), (er, ez) = gate, egate
    arg = sl(gi, 2) + r * sl(gh, 2)
    earg = sl(ei, 2) + er * (sl(gh, 2).abs() + sl(eh, 2)) + r * sl(eh, 2) + U * (arg.abs() + 1e-300)
    n = torch.tanh(arg)
    en = earg + 4 * U * n.abs()
    h = (1 - z) * n + z * c
    e1z = ez + U * (1 - z)
    ep = e1z * (n.abs() + en) + (1 - z) * en + U * ((1 - z) * n).abs() * 2
    eh_ = ez * c.abs() + ep + U * h.abs() * 2
    return h, eh_ * 1.01 + 1e-30


def teacher_forced(pol, out, wipe_on_done):
    """(worst |hid - h_ref| / bound over every t, logits [T,N,4] float64 of the head on hid, their bound)."""
    Wi, Wh, bi, bh, head = unpack(pol)
    H, T, N = pol.hidden, out["act"].shape[0], out["act"].shape[1]
    hid = out["hid"].double()
    obs = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, N, -1).double()
    s0 = out["state0"].double()
    done = out["done"].bool()
    c = torch.empty((T, N, H), dtype=torch.float64, device=hid.device)
    fb = torch.empty((T, N, 5), dtype=torch.float64, device=hid.device)
    c[0], fb[0] = s0[:, :H], (s0[:, H:] if pol.feedback else 0)
    if T > 1:
        keep = ~(done[:-1] & wipe_on_done)[..., None]
        c[1:] = torch.where(keep, hid[:-1], 0.0)
        prev = torch.cat([torch.nn.functional.one_hot(out["act"][:-1].long(), 4).double(),
                          out["rew"][:-1].float().double()[..., None]], -1)
        fb[1:] = torch.where(keep, prev, 0.0)
    x = torch.cat([obs, fb], -1) if pol.feedback else obs
    h, eb = gru_bound(Wi, Wh, bi, bh, x, c)
    worst = float(((hid - h).abs() / eb).max())
    with torch.no_grad():
        logits, lb = forward_bound(head, hid)
    return worst, logits, lb


def check_actions(env, logits, bound, out, seed, t0, deterministic=False):
    """act and logp against the float64 head on hid (as test_policy_rollout_maze_gpu checks the MLP's); returns the
    worst logp error relative to its bound."""
    T, N = out["act"].shape
    act = out["act"].long()
    b = bound.max(-1).values
    if deterministic:
        top2 = logits.topk(2, -1).values
        clear = (top2[..., 0] - top2[..., 1]) > 2 * b + 1e-6
        assert torch.equal(act[clear], logits.argmax(-1)[clear])
        return 0.0
    genv = env.env_index_base + np.arange(N)
    worst = 0.0
    for t in range(T):
        u = torch.as_tensor(maze_policy_uniforms(seed, genv, t0 + t), device=act.device)
        cdf = torch.softmax(logits[t], -1).cumsum(-1)[:, :3]
        want = torch.where(u[:, None] < cdf, torch.arange(3, device=act.device), 3).min(-1).values
        bad = act[t] != want
        if bad.any():
            near = (u[:, None] - cdf).abs().min(-1).values < NEAR
            assert bool(near[bad].all()), "an action differs away from every CDF boundary"
        if out.get("logp") is not None:
            lp = torch.log_softmax(logits[t], -1).gather(-1, act[t][:, None])[:, 0]
            mx = logits[t].max(-1).values
            tol = 2 * b[t] + U * (8 * (logits[t].gather(-1, act[t][:, None])[:, 0] - mx).abs() + 32)
            worst = max(worst, float(((out["logp"][t].double() - lp).abs() / tol).max()))
    return worst


def expected_state(pol, out, wipe_on_done):
    """[hid[T-1] or 0, onehot(act[T-1]), (float)rew[T-1]] row for row, zero where done[T-1] and the rule fires."""
    h = out["hid"][-1]
    parts = [h]
    if pol.feedback:
        parts += [torch.nn.functional.one_hot(out["act"][-1].long(), 4).float(), out["rew"][-1].float()[:, None]]
    s = torch.cat(parts, 1)
    wipe = out["done"][-1].bool() & wipe_on_done
    return torch.where(wipe[:, None], torch.zeros_like(s), s)


def setup_pair(n, task_type, view_grid, resample, record_path, tasks):  # noqa: F811
    envs = []
    for _ in range(2):
        e = make_env(n, task_type, view_grid=view_grid, record_path=record_path)
        if resample:
            table, _ = slot_table(9, n)
            e.set_task(table, env2task=np.arange(n))
        else:
            e.set_task(tasks)
        e.reset()
        e.rollout(3)                                   # t_base != 0
        envs.append(e)
    return envs


# task type, view_grid, H, head width, head activation, feedback, reset rule, resample, record_path
CASES = [
    ("SURVIVAL", 1, 64, 0, nn.Tanh, True, "task", False, False),      # task mode keeps c across done
    ("SURVIVAL", 1, 64, 0, nn.Tanh, True, "task", True, True),        # ... and zeroes it on a new maze
    ("ESCAPE", 2, 17, 32, nn.ReLU, False, "episode", False, True),
    ("SURVIVAL", 2, 1, 5, nn.Tanh, True, "episode", True, False),
    ("ESCAPE", 1, 17, 0, nn.Tanh, False, "task", True, False),
    ("SURVIVAL", 1, 64, 64, nn.ReLU, True, "episode", False, False),
]


@pytest.mark.parametrize("case", CASES, ids=["%s-g%d-H%d-w%d-%s-%s-%s-%s-%s" % (c[0], c[1], c[2], c[3], c[4].__name__,
                                                                                 "fb" if c[5] else "nofb", c[6],
                                                                                 "rs" if c[7] else "nors",
                                                                                 "path" if c[8] else "nopath")
                                             for c in CASES])
def test_env_side_policy_side_and_state(tasks, case):  # noqa: F811
    task_type, vg, H, width, act, feedback, reset, resample, record_path = case
    n, T = 1000, 40
    env, twin = setup_pair(n, task_type, vg, resample, record_path, tasks)
    pol = make_policy(env, H, width, act, feedback, reset, seed=H + width)
    state = random_state(pol, n)
    before = state.clone()
    rs = dict(seed=SEED, **CFG) if resample else None
    t0 = env._counters()
    out = env.rollout(T, policy=pol, state=state, act_seed=SEED, resample=rs, want_hidden=True)
    assert out["resampled"] == resample
    assert out["done"].any(), "no episode ended: the reset rule is not exercised"
    ref = twin.rollout(T, actions=out["act"], resample=rs)
    assert_env_side_equal(out, ref)
    if record_path:
        for x, y in zip(env.trajectory(), twin.trajectory()):
            assert torch.equal(x, y)
    wipe = reset == "episode" or resample
    worst, logits, lb = teacher_forced(pol, out, wipe)
    assert worst <= 1.0, worst
    # the check sees the reset rule: the other rule breaks the bound
    assert teacher_forced(pol, out, not wipe)[0] > 1.0
    assert check_actions(env, logits, lb, out, SEED, t0) <= 1.0
    assert torch.equal(out["state0"], before)
    assert torch.equal(state, expected_state(pol, out, wipe))
    # deterministic mode continues from the state just written
    s1 = state.clone()
    det = env.rollout(T, policy=pol, state=state, deterministic=True, resample=rs, want_hidden=True)
    assert det["logp"] is None and torch.equal(det["state0"], s1)
    assert_env_side_equal(det, twin.rollout(T, actions=det["act"], resample=rs))
    worst, logits, lb = teacher_forced(pol, det, wipe)
    assert worst <= 1.0
    check_actions(env, logits, lb, det, 0, 0, deterministic=True)
    assert torch.equal(state, expected_state(pol, det, wipe))
    for e in (env, twin):
        e.close()


def test_unroll_matches_the_kernel(tasks):  # noqa: F811
    n, T = 256, 24
    env = make_env(n)
    env.set_task(tasks)
    env.reset()
    pol = make_policy(env, 17, 8, nn.Tanh, True, "episode", seed=4)
    state = random_state(pol, n)
    out = env.rollout(T, policy=pol, state=state, act_seed=3)
    _, logp = pol.unroll(out)
    assert logp.shape == (T, n)
    assert float((logp.detach() - out["logp"].cpu()).abs().max()) < 1e-4


@pytest.mark.parametrize("resample", [False, True], ids=["plain", "resample"])
def test_continuity(tasks, resample):  # noqa: F811
    n, T = 257, 24
    env = make_env(n, "SURVIVAL")
    if resample:
        env.set_task(slot_table(9, n)[0], env2task=np.arange(n))
    else:
        env.set_task(tasks)
    env.reset()
    pol = make_policy(env, 17, 5, nn.ReLU, True, "task", seed=2)
    rs = dict(seed=SEED, **CFG) if resample else None
    s0 = random_state(pol, n)
    snap = env.snapshot()
    st = s0.clone()
    a = env.rollout(T, policy=pol, state=st, act_seed=SEED, resample=rs, want_hidden=True)
    b = env.rollout(T, policy=pol, state=st, act_seed=SEED, resample=rs, want_hidden=True)
    assert torch.equal(b["obs0"], a["obs"][-1])
    env.restore(snap)
    st2 = s0.clone()
    ab = env.rollout(2 * T, policy=pol, state=st2, act_seed=SEED, resample=rs, want_hidden=True)
    for k in ("act", "logp", "obs", "rew", "done", "truncated", "hid"):
        assert torch.equal(ab[k], torch.cat([a[k], b[k]])), k
    d = ab["done"].bool()
    assert torch.equal(ab["final_obs"][d], torch.cat([a["final_obs"], b["final_obs"]])[d])
    assert torch.equal(st2, st) and torch.equal(ab["state0"], a["state0"]) and torch.equal(a["state0"], s0)


def test_sharding_with_resampling():
    n, T = 1000, 24
    base = (1 << 32) - n // 2 - 3
    half, _ = slot_table(9, n // 2)      # each shard's table starts with the food task: it sets the table's food cap
    table = half + half
    envs = [make_env(n, base=base)] + [make_env(n // 2, base=base + k * (n // 2)) for k in range(2)]
    for env, tab in zip(envs, [table, half, half]):
        env.set_task(tab, env2task=np.arange(env.num_envs))
        env.reset()
    pol = make_policy(envs[0], 64, 0, nn.Tanh, True, "task", seed=5)
    s0 = random_state(pol, n)
    states = [s0.clone(), s0[:n // 2].clone(), s0[n // 2:].clone()]
    rs = dict(seed=SEED, **CFG)
    outs = [env.rollout(T, policy=pol, state=s, act_seed=SEED, resample=rs, want_hidden=True)
            for env, s in zip(envs, states)]
    for k in ("act", "logp", "obs", "rew", "done", "truncated", "hid"):
        assert torch.equal(outs[0][k], torch.cat([outs[1][k], outs[2][k]], 1)), k
    for k in ("obs0", "state0"):
        assert torch.equal(outs[0][k], torch.cat([outs[1][k], outs[2][k]])), k
    assert torch.equal(states[0], torch.cat(states[1:]))
    assert outs[0]["done"].sum() > 10


def capture(env, T, pol, state, out, deterministic):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        env.rollout(T, policy=pol, state=state, act_seed=1, out=out, deterministic=deterministic)
    return g


def test_graph_replay_and_update(tasks):  # noqa: F811
    n, T = 512, 8
    env = make_env(n, "ESCAPE")
    env.set_task(tasks)
    env.reset()
    pol = make_policy(env, 17, 0, nn.Tanh, True, "episode")
    s0 = random_state(pol, n)
    state = s0.clone()
    det = env.rollout(T, policy=pol, state=state, deterministic=True, want_hidden=True)   # warm-up; buffers reused
    out = env.rollout(T, policy=pol, state=state, act_seed=1, want_hidden=True)
    snap = env.snapshot()
    s1 = state.clone()
    # A captured launch keeps the step counter it was captured at, so two replays draw the same uniforms; in mean mode
    # nothing is drawn, and two replays carry the env and the state exactly as two eager launches do.
    g = capture(env, T, pol, state, out, False)              # at the snapshot's counter (each capture advances it)
    g_det = capture(env, T, pol, state, det, True)
    state.copy_(s1)
    env.restore(snap)
    got = []
    for _ in range(2):
        g_det.replay()
        torch.cuda.synchronize()
        got.append({k: v.clone() for k, v in det.items() if isinstance(v, torch.Tensor)})
    got_state = state.clone()
    env.restore(snap)
    st = s1.clone()
    eager = [env.rollout(T, policy=pol, state=st, deterministic=True, want_hidden=True) for _ in range(2)]
    for gg, ee in zip(got, eager):
        for k in ("act", "obs0", "obs", "rew", "done", "truncated", "state0", "hid"):
            assert torch.equal(gg[k], ee[k]), k
    assert torch.equal(got_state, st)
    # sampling mode: a replay from the captured counter equals the eager launch from the same counter
    state.copy_(s1)
    env.restore(snap)
    g.replay()
    torch.cuda.synchronize()
    got = {k: v.clone() for k, v in out.items() if isinstance(v, torch.Tensor)}
    got_state = state.clone()
    env.restore(snap)
    st = s1.clone()
    eager = env.rollout(T, policy=pol, state=st, act_seed=1, want_hidden=True)
    for k in ("act", "logp", "obs0", "obs", "rew", "done", "truncated", "state0", "hid"):
        assert torch.equal(got[k], eager[k]), k
    assert torch.equal(got_state, st)
    # after update() the replay runs the new weights
    pol.update(make_policy(env, 17, 0, nn.Tanh, True, "episode", seed=11)._cell)
    env.restore(snap)
    state.copy_(s1)
    g.replay()
    torch.cuda.synchronize()
    new = {k: v.clone() for k, v in out.items() if isinstance(v, torch.Tensor)}
    env.restore(snap)
    st = s1.clone()
    eager = env.rollout(T, policy=pol, state=st, act_seed=1, want_hidden=True)
    for k in ("act", "logp", "obs", "state0", "hid"):
        assert torch.equal(new[k], eager[k]), k
    assert not torch.equal(new["hid"], got["hid"])
    assert torch.equal(state, st)
    assert teacher_forced(pol, new, True)[0] <= 1.0


def test_refusals_leave_everything_untouched(tasks):  # noqa: F811
    from metagym_b200 import BatchedQuadrotor, _lib
    from metagym_b200.policy import MLPPolicy
    from test_policy_rollout_maze_gpu import make_module
    n, T = 128, 4
    env = make_env(n)
    env.set_task(tasks)
    env.reset()
    pol = make_policy(env, 8, 4)
    dev = env.device
    lib = env._lib
    state = random_state(pol, n)
    outs = {"logp": torch.full((T, n), 7.0, device=dev), "act": torch.full((T, n), 7, dtype=torch.int32, device=dev),
            "hid": torch.full((T, n, 8), 7.0, device=dev), "state0": torch.full((n, pol.state_dim), 7.0, device=dev)}

    def call(e, p, T=T, st=state, logp=True, cfg=None):
        return lib.mgb_maze_rollout_rnn(e._h, T, ctypes.byref(p) if p is not None else None, 0,
                                        ctypes.byref(cfg) if cfg is not None else None, 0, _lib.ptr(st),
                                        _lib.ptr(outs["state0"]), _lib.ptr(outs["hid"]), _lib.ptr(outs["act"]),
                                        _lib.ptr(outs["logp"]) if logp else None, None, None, None, None, None, None,
                                        e._stream())

    def snapshot(e, st):
        return (e._counters(), e.launch_count, e.snapshot()["records"].cpu().clone(), st.clone(),
                {k: v.clone() for k, v in outs.items()})

    def untouched(a, b):      # b's snapshot() is the one launch between the two
        assert a[0] == b[0] and a[1] == b[1] + 1 and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
        for k in outs:
            assert torch.equal(a[4][k], b[4][k]), k

    before = snapshot(env, state)
    good = pol.struct()
    assert call(env, good, T=0) == MGB_ERR_ARG and call(env, None) == MGB_ERR_ARG
    bad = []
    for field, v in (("params_dev", None), ("hidden", 0), ("hidden", 65), ("feedback", 2), ("feedback", -1),
                     ("reset", 2), ("head_hidden", 2), ("head_width", 0), ("head_width", 65), ("activation", 7),
                     ("mode", 2)):
        p = pol.struct()
        setattr(p, field, v)
        bad.append(p)
    for p in bad:
        assert call(env, p) == MGB_ERR_ARG, [(f, getattr(p, f)) for f, _ in p._fields_]
    assert call(env, good, st=None) == MGB_ERR_ARG
    raw = torch.zeros(n * pol.state_dim + 1, device=dev)
    assert call(env, good, st=raw.view(torch.uint8)[1:]) == MGB_ERR_ARG and "aligned" in lib.mgb_last_error().decode()
    assert call(env, pol.struct(deterministic=True)) == MGB_ERR_ARG                     # logp in mean mode
    for arm in (lambda: env.set_mirrors([16]), lambda: env.set_multicast(16)):
        arm()
        assert call(env, good) == MGB_ERR_ARG
        env.set_mirrors([])
    torch.cuda.synchronize()
    after = snapshot(env, state)
    untouched(after, before)
    # auto_reset off
    plain = make_env(n, auto_reset=False, final_obs=False)
    plain.set_task(tasks)
    plain.reset()
    b = snapshot(plain, state)
    assert call(plain, good) == MGB_ERR_ARG and "auto_reset" in lib.mgb_last_error().decode()
    untouched(snapshot(plain, state), b)
    # resample where mgb_maze_rollout refuses it (the tasks table is shared, not one slot per env)
    cfg, _ = env._sampler_cfg(seed=1, **CFG)
    b = snapshot(env, state)
    assert call(env, good, cfg=cfg) == MGB_ERR_ARG
    untouched(snapshot(env, state), b)
    # shared memory beyond the opt-in limit: a 13 x 13 window with H = 64
    wide = make_env(n, view_grid=6)
    wide.set_task(tasks)
    wide.reset()
    pw = make_policy(wide, 64, 0)
    sw = random_state(pw, n)
    b = (wide._counters(), sw.clone())
    rc = lib.mgb_maze_rollout_rnn(wide._h, T, ctypes.byref(pw.struct()), 0, None, 0, _lib.ptr(sw), None, None, None,
                                  None, None, None, None, None, None, None, wide._stream())
    assert rc == MGB_ERR_ARG and "shared memory" in lib.mgb_last_error().decode()
    assert wide._counters() == b[0] and torch.equal(sw, b[1])
    with pytest.raises(_lib.MgbError):
        wide.rollout(T, policy=pw, state=sw)
    # Python refusals
    with pytest.raises(ValueError):
        env.rollout(T, policy=pol)                                        # no state
    with pytest.raises(ValueError):
        env.rollout(T, policy=MLPPolicy(make_module(9), device=dev), state=state)
    with pytest.raises(ValueError):
        env.rollout(T, state=state)
    for bad_state in (state[:-1], state.double(), state.cpu(), state[:, :-1], state.t().contiguous().t()):
        with pytest.raises(ValueError):
            env.rollout(T, policy=pol, state=bad_state)
    quad = BatchedQuadrotor(task="hovering_control", dt=0.005, nt=40, num_envs=8, device=0, squeeze=False)
    with pytest.raises(ValueError):
        quad.rollout(T, policy=pol)
    for e in (env, plain, wide, quad):
        e.close()
