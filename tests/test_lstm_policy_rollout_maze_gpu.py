"""GPU: MetaMaze2D rollouts driven by an on-device LSTM policy (mgb_maze_rollout_rnn with cell = MGB_RNN_CELL_LSTM,
BatchedMetaMaze2D.rollout(policy=LSTMPolicy, state=)).

Env side: bit for bit the open-loop rollout fed the actions the policy took.  Policy side, teacher-forced: every h_t
the kernel reports lies within the float32 error bound of a float64 LSTMCell on the inputs the header's rule gives
(x_t from the window and the feedback of step t - 1, h_{t-1} from state0, the kernel's h and the reset rule); the cell
state c is not reported per step, so the reference carries c in float64 with a bound that propagates through the steps,
and the final state's c is checked against it.  The actions and log-probabilities are checked against the float64 head
on h_t and the Philox uniforms of tests/policy_draws.py.  The rest of the state written back is checked bit for bit.
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

from test_maze_final_obs_gpu import MAX_STEPS, tasks  # noqa: E402,F401  (fixtures)
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402
from test_policy_rollout_maze_gpu import SEED, assert_env_side_equal, make_env  # noqa: E402
from test_rnn_policy_rollout_maze_gpu import capture, check_actions, random_state, setup_pair  # noqa: E402

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
U = 2.0 ** -24


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


def make_policy(env, H=64, width=0, act=nn.Tanh, feedback=True, reset="episode", seed=0, bias=True):
    from metagym_b200 import LSTMPolicy
    g = torch.Generator().manual_seed(seed)
    D = env._obs[0].numel()
    cell = nn.LSTMCell(D + 5 * feedback, H, bias=bias)
    head = nn.Linear(H, 4) if not width else nn.Sequential(nn.Linear(H, width), act(), nn.Linear(width, 4))
    with torch.no_grad():
        for p in list(cell.parameters()) + list(head.parameters()):
            p.copy_(torch.randn(p.shape, generator=g) * (1.5 / max(p.shape[-1], 1) ** 0.5 if p.dim() == 2 else 0.3))
    return LSTMPolicy(cell, head, feedback=feedback, hidden_reset=reset, device=env.device)


def unpack(pol):
    """float64 cell weights and an nn.Sequential head read from the packed float32 buffer (what the kernel reads)."""
    buf = pol.params.double()
    H, n_in = pol.hidden, pol.obs_dim + 5 * pol.feedback
    o = 0

    def take(k):
        nonlocal o
        o += k
        return buf[o - k:o]
    Wi, Wh = take(4 * H * n_in).reshape(4 * H, n_in), take(4 * H * H).reshape(4 * H, H)
    bi, bh = take(4 * H), take(4 * H)
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


def lstm_bound(Wi, Wh, bi, bh, x, hp, c, ec):
    """float64 (h', c') = LSTMCell(x, (hp, c)) and bounds on the float32 kernel's h' and c', from the header's statement,
    where the kernel's c differs from c by at most ec.  An fma chain of k terms from its bias errs by at most (k + 1) u
    (|b| + sum |w| |input|); the float32 add of the two chains adds u |v|; sigma(v) = 1 / (1 + expf(-v)) moves by at most
    |dv| / 4 and adds at most 8 u sigma (expf 2 ulp, one add, one division); tanhf is 1-Lipschitz and adds 2 ulp (4 u
    of its result); c' = fmaf(f, c, i g) rounds i g and the fma; h' = o tanhf(c') rounds the product."""
    H = hp.shape[-1]
    gi, gh = x @ Wi.T + bi, hp @ Wh.T + bh
    ei = (x.shape[-1] + 1) * U * (x.abs() @ Wi.abs().T + bi.abs())
    eh = (H + 1) * U * (hp.abs() @ Wh.abs().T + bh.abs())
    v = gi + gh
    ev = ei + eh + U * (v.abs() + ei + eh)
    sl = lambda t, k: t[..., k * H:(k + 1) * H]               # noqa: E731
    sig = [torch.sigmoid(sl(v, k)) for k in (0, 1, 3)]
    (i, f, o), (e_i, e_f, e_o) = sig, [0.25 * sl(ev, k) + 8 * U * s for k, s in zip((0, 1, 3), sig)]
    g = torch.tanh(sl(v, 2))
    e_g = sl(ev, 2) + 4 * U * g.abs()
    p = i * g
    e_p = e_i * (g.abs() + e_g) + i * e_g + U * (p.abs() + e_i * (g.abs() + e_g) + i * e_g)
    c2 = f * c + p
    e_c2 = e_f * (c.abs() + ec) + f * ec + e_p
    e_c2 = e_c2 + U * (c2.abs() + e_c2)
    th = torch.tanh(c2)
    e_th = e_c2 + 4 * U * th.abs()
    h2 = o * th
    e_h2 = e_o * (th.abs() + e_th) + o * e_th
    e_h2 = e_h2 + U * (h2.abs() + e_h2)
    return h2, e_h2 * 1.01 + 1e-30, c2, e_c2 * 1.01 + 1e-30


def teacher_forced(pol, out, wipe_on_done):
    """(worst |hid - h_ref| / bound over every t, logits [T,N,4] float64 of the head on hid, their bound, the float64
    reference c after step T - 1 with its zeroing applied, its bound)."""
    Wi, Wh, bi, bh, head = unpack(pol)
    H, T = pol.hidden, out["act"].shape[0]
    hid = out["hid"].double()
    obs = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, hid.shape[1], -1).double()
    s0 = out["state0"].double()
    done = out["done"].bool()
    hp, c, fb = s0[:, :H], s0[:, H:2 * H], s0[:, 2 * H:]
    ec = torch.zeros_like(c)
    worst = 0.0
    for t in range(T):
        x = torch.cat([obs[t], fb], -1) if pol.feedback else obs[t]
        h, eb, c, ec = lstm_bound(Wi, Wh, bi, bh, x, hp, c, ec)
        worst = max(worst, float(((hid[t] - h).abs() / eb).max()))
        keep = ~(done[t] & wipe_on_done)[:, None]
        hp = torch.where(keep, hid[t], 0.0)
        c, ec = torch.where(keep, c, 0.0), torch.where(keep, ec, 0.0)
        if pol.feedback:
            prev = torch.cat([torch.nn.functional.one_hot(out["act"][t].long(), 4).double(),
                              out["rew"][t].float().double()[:, None]], -1)
            fb = torch.where(keep, prev, 0.0)
    with torch.no_grad():
        logits, lb = forward_bound(head, hid)
    return worst, logits, lb, c, ec


def check_state(pol, out, state, wipe_on_done, c_ref, ec):
    """h and the feedback of the state written back, bit for bit: [hid[T-1], onehot(act[T-1]), (float)rew[T-1]], zero
    where done[T-1] and the rule fires; c within the propagated bound of the float64 reference (exactly 0 where wiped)."""
    H = pol.hidden
    wipe = (out["done"][-1].bool() & wipe_on_done)[:, None]
    assert torch.equal(state[:, :H], torch.where(wipe, 0.0, out["hid"][-1]))
    if pol.feedback:
        fb = torch.cat([torch.nn.functional.one_hot(out["act"][-1].long(), 4).float(), out["rew"][-1].float()[:, None]], 1)
        assert torch.equal(state[:, 2 * H:], torch.where(wipe, 0.0, fb))
    c = state[:, H:2 * H]
    assert not c[wipe.expand_as(c)].any()
    assert float(((c.double() - c_ref).abs() / (ec + 1e-300)).max()) <= 1.0       # ec is 0 where wiped


# task type, view_grid, H, head width, head activation, feedback, reset rule, resample, record_path
CASES = [
    ("SURVIVAL", 1, 64, 0, nn.Tanh, True, "task", False, False),      # task mode keeps h and c across done
    ("SURVIVAL", 1, 64, 0, nn.Tanh, True, "task", True, True),        # ... and zeroes them on a new maze
    ("ESCAPE", 2, 17, 32, nn.ReLU, False, "episode", False, True),    # head wider than H: the h columns widen
    ("SURVIVAL", 2, 1, 5, nn.Tanh, True, "episode", True, False),
    ("ESCAPE", 1, 17, 0, nn.Tanh, False, "task", True, False),
    ("SURVIVAL", 1, 64, 64, nn.ReLU, True, "episode", True, False),   # the largest head at view_grid 1, resampling
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
    worst, logits, lb, c_ref, ec = teacher_forced(pol, out, wipe)
    assert worst <= 1.0, worst
    # the check sees the reset rule: the other rule breaks the bound
    assert teacher_forced(pol, out, not wipe)[0] > 1.0
    assert check_actions(env, logits, lb, out, SEED, t0) <= 1.0
    assert torch.equal(out["state0"], before)
    check_state(pol, out, state, wipe, c_ref, ec)
    # deterministic mode continues from the state just written
    s1 = state.clone()
    det = env.rollout(T, policy=pol, state=state, deterministic=True, resample=rs, want_hidden=True)
    assert det["logp"] is None and torch.equal(det["state0"], s1)
    assert_env_side_equal(det, twin.rollout(T, actions=det["act"], resample=rs))
    worst, logits, lb, c_ref, ec = teacher_forced(pol, det, wipe)
    assert worst <= 1.0
    check_actions(env, logits, lb, det, 0, 0, deterministic=True)
    check_state(pol, det, state, wipe, c_ref, ec)
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
    # the state, c included, is carried across the launch boundary bit for bit
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


def test_graph_replay_and_update(tasks):  # noqa: F811
    n, T = 512, 8
    env = make_env(n, "ESCAPE")
    env.set_task(tasks)
    env.reset()
    pol = make_policy(env, 17, 0, nn.Tanh, True, "episode")
    s0 = random_state(pol, n)
    state = s0.clone()
    env.rollout(T, policy=pol, state=state, deterministic=True, want_hidden=True)     # warm-up
    out = env.rollout(T, policy=pol, state=state, act_seed=1, want_hidden=True)     # buffers the graph reuses
    snap = env.snapshot()
    s1 = state.clone()
    g = capture(env, T, pol, state, out, False)              # at the snapshot's counter (each capture advances it)

    def replay():
        state.copy_(s1)
        env.restore(snap)
        g.replay()
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in out.items() if isinstance(v, torch.Tensor)}, state.clone()

    def eager():
        env.restore(snap)
        st = s1.clone()
        return env.rollout(T, policy=pol, state=st, act_seed=1, want_hidden=True), st

    got, got_state = replay()
    want, want_state = eager()
    for k in ("act", "logp", "obs0", "obs", "rew", "done", "truncated", "state0", "hid"):
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(got_state, want_state)
    # after update() the replay runs the new weights
    pol.update(make_policy(env, 17, 0, nn.Tanh, True, "episode", seed=11)._cell)
    new, new_state = replay()
    want, want_state = eager()
    for k in ("act", "logp", "obs", "state0", "hid"):
        assert torch.equal(new[k], want[k]), k
    assert not torch.equal(new["hid"], got["hid"])
    assert torch.equal(new_state, want_state)
    assert teacher_forced(pol, new, True)[0] <= 1.0


# Static shared memory of the kPolLstm kernels as cudaFuncGetAttributes reports it, which the host adds to the dynamic
# bytes before comparing with the opt-in limit: none, since the tiles, weights and columns are all dynamic.  (The 1 KB
# that cuobjdump -res-usage lists for every kernel of the library is the per-block reserved shared memory, which the
# opt-in limit, 227 KB on the H100, already excludes.)  The refusal test reads the host's total back from its message.
STATIC_SMEM = 0


def smem_bytes(view_grid, H, width, feedback, rs, n=15, threads=128):
    """The LSTM rollout's shared memory per CTA, restated from DESIGN.md "Recurrent policies": two observation tiles
    (+ one sampler workspace per warp with resampling, which grows with the maze size n), then the staged cell (4 gates
    of weight_ih and weight_hh and 8 biases per unit, H padded to 8) and head (MgbMlp layout), then the columns x [in],
    c [H], h [Hr], h [Hr], Hr = max(H, head width); plus STATIC_SMEM."""
    D = (2 * view_grid + 1) ** 2
    base = 2 * threads * D * 4
    if rs:
        base += threads // 32 * ((7 * n * n + ((n - 1) // 2) ** 2 + 15) // 16 * 16)
    base = (base + 15) // 16 * 16
    Hp, n_in = (H + 7) // 8 * 8, D + 5 * feedback
    s = 4 * Hp * n_in + 4 * Hp * H + 8 * Hp
    head, ins = 0, [H] + ([width] if width else [])
    for k, i in enumerate(ins):
        last = k == len(ins) - 1
        out = 4 if last else width
        gw = 4 if last else 8
        rows = (out + gw - 1) // gw * gw
        head = (head + rows * i + rows + 7) // 8 * 8
    Hr = max(H, width)
    return base + (s + head + (n_in + H + 2 * Hr) * threads) * 4 + STATIC_SMEM


def test_refusals_leave_everything_untouched(tasks):  # noqa: F811
    from metagym_b200 import BatchedQuadrotor, _lib
    from metagym_b200.policy import GRUPolicy
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
                     ("mode", 2), ("cell", 2), ("cell", -1)):
        p = pol.struct()
        setattr(p, field, v)
        bad.append(p)
    for p in bad:
        assert call(env, p) == MGB_ERR_ARG, [(f, getattr(p, f)) for f, _ in p._fields_]
        if p.cell not in (0, 1):
            assert "unknown cell" in lib.mgb_last_error().decode()
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
    # shared memory: refused exactly where the footprint exceeds the opt-in limit, with nothing touched.  Each shape is
    # the largest H that fits at its view_grid, head and resampling (9 x 9 mazes), checked against H + 1.  The nearer
    # side of each pair is 160 to 1760 bytes from the limit, and the refusal's own byte count must match exactly
    optin = torch.cuda.get_device_properties(dev).shared_memory_per_block_optin
    largest = [(2, 61, 0, False), (3, 48, 0, False), (4, 29, 0, False), (3, 36, 64, False), (2, 60, 0, True),
               (3, 35, 64, True), (1, 64, 64, True)]
    for vg, H, w, rsm in largest:
        assert smem_bytes(vg, H, w, True, rsm, n=9) <= optin, (vg, H, w, rsm)
        if H < 64:
            assert smem_bytes(vg, H + 1, w, True, rsm, n=9) > optin, (vg, H, w, rsm)
    shapes = [(vg, H + k, w, rsm) for vg, H, w, rsm in largest for k in (0, 1) if H + k <= 64] + [(6, 64, 0, False)]
    for vg, H, w, rsm in shapes:
        want = smem_bytes(vg, H, w, True, rsm, n=9)
        e = make_env(n, view_grid=vg)
        if rsm:
            e.set_task(slot_table(9, n)[0], env2task=np.arange(n))
        else:
            e.set_task(tasks)
        e.reset()
        pw = make_policy(e, H, w)
        sw = random_state(pw, n)
        b = (e._counters(), e.launch_count, sw.clone())
        c = e._sampler_cfg(seed=1, **CFG)[0] if rsm else None
        rc = lib.mgb_maze_rollout_rnn(e._h, T, ctypes.byref(pw.struct()), 0, ctypes.byref(c) if rsm else None, 0,
                                      _lib.ptr(sw), None, None, None, None, None, None, None, None, None, None,
                                      e._stream())
        torch.cuda.synchronize()
        if want <= optin:
            assert rc == 0, (vg, H, w, rsm, lib.mgb_last_error().decode())
        else:
            msg = lib.mgb_last_error().decode()
            assert rc == MGB_ERR_ARG and "needs %d bytes of shared memory" % want in msg, (vg, H, w, rsm, want, msg)
            assert e._counters() == b[0] and e.launch_count == b[1] and torch.equal(sw, b[2])
            with pytest.raises(_lib.MgbError):
                e.rollout(T, policy=pw, state=sw, resample=dict(seed=1, **CFG) if rsm else None)
        e.close()
    # Python refusals
    with pytest.raises(ValueError):
        env.rollout(T, policy=pol)                                        # no state
    gru = GRUPolicy(nn.GRUCell(14, 8), nn.Linear(8, 4), device=dev)
    with pytest.raises(ValueError):
        env.rollout(T, policy=gru, state=state)                           # an LSTM state is not a GRU state
    for bad_state in (state[:-1], state.double(), state.cpu(), state[:, :-1], state.t().contiguous().t()):
        with pytest.raises(ValueError):
            env.rollout(T, policy=pol, state=bad_state)
    quad = BatchedQuadrotor(task="hovering_control", dt=0.005, nt=40, num_envs=8, device=0, squeeze=False)
    with pytest.raises(ValueError):
        quad.rollout(T, policy=pol)
    for e in (env, plain, quad):
        e.close()
