"""GPU: every compiled policy-rollout instantiation, checked numerically at the shapes and edges where the policy paths
could go wrong without the per-kind tests noticing.

The library compiles maze2d_rollout_kernel<0, FIN, REC, RS, POL> for the three policy kinds (POL: MLP, GRU, LSTM) over
terminal outputs (FIN), path recording (REC) and in-launch resampling (RS), 24 instantiations, and
quad_rollout_kernel<SIMPLE, 0, FIN, true> over the two physics paths and FIN, 4 more.  Each one is launched here at least
once and checked as the per-kind tests check theirs: the env side bit for bit against the open-loop rollout fed the
actions the policy took, the policy side against the float64 references of test_policy_rollout_gpu,
test_policy_rollout_maze_gpu, test_rnn_policy_rollout_maze_gpu and test_lstm_policy_rollout_maze_gpu (imported, bounds
unchanged), and the carried state written back.  On top of that:

- wide windows (view_grid 3 and 4: 49 and 81 policy inputs, or 54 and 86 with feedback) at the largest footprint that
  fits the opt-in shared memory;
- the MLP and GRU footprints restated in Python, refused exactly one step above the largest shape that fits, with the
  byte count in the message and nothing touched;
- the "every output may be NULL" contract of all three entry points: dropping any output leaves every other output, the
  env state and the carried state bit-identical;
- batch tails whose bulk-store destinations are not 16-byte aligned, and a quadrotor CTA with a single env.
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import test_lstm_policy_rollout_maze_gpu as lstm_t  # noqa: E402
import test_policy_rollout_gpu as quad_t  # noqa: E402
import test_policy_rollout_maze_gpu as mlp_t  # noqa: E402
import test_rnn_policy_rollout_maze_gpu as gru_t  # noqa: E402
from test_maze2d_resample_rollout_gpu import CFG, slot_table  # noqa: E402
from test_maze_final_obs_gpu import tasks  # noqa: E402,F401  (fixture)

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = 0x9E3779B97F4A7C15          # both 32-bit halves set
LOG_STD = (-0.5, 0.0, 0.3, -1.0)
THREADS = 128                      # envs per maze rollout CTA (k2dThreads)


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


# ---------------------------------------------------------------------------------------------------------------
# MetaMaze2D: one runner and one checker for the three policy kinds
# ---------------------------------------------------------------------------------------------------------------

class Shape:
    """A maze policy: MLP `widths`, or a cell of H units with a head of `width` (0: Linear(H, 4))."""

    def __init__(self, kind, widths=(), H=0, width=0, act=nn.Tanh, feedback=True, reset="episode", task_type="SURVIVAL",
                 view_grid=1):
        self.kind, self.widths, self.H, self.width, self.act = kind, tuple(widths), H, width, act
        self.feedback, self.reset, self.task_type, self.view_grid = feedback, reset, task_type, view_grid

    def __repr__(self):
        net = "w%s" % "-".join(map(str, self.widths)) if self.kind == "mlp" else \
            "H%d-w%d-%s-%s" % (self.H, self.width, "fb" if self.feedback else "nofb", self.reset)
        return "%s-%s-%s-%s-g%d" % (self.kind, net, self.act.__name__, self.task_type, self.view_grid)

    def policy(self, env, seed=0):
        """(module or None, policy)"""
        if self.kind == "mlp":
            return mlp_t.make_policy(env, self.widths, self.act, seed)
        make = gru_t.make_policy if self.kind == "gru" else lstm_t.make_policy
        return None, make(env, self.H, self.width, self.act, self.feedback, self.reset, seed=seed)


def maze_pair(n, shape, rs, rec, fin, tasks, maze_n=9):  # noqa: F811
    """Two identical MetaMaze2D handles a few steps in (t_base != 0): one for the policy, one for the open-loop twin.
    With resampling, one table slot per env of maze_n x maze_n mazes."""
    envs = []
    for _ in range(2):
        e = mlp_t.make_env(n, shape.task_type, view_grid=shape.view_grid, record_path=rec, final_obs=fin)
        if rs:
            e.set_task(slot_table(maze_n, n)[0], env2task=np.arange(n))
        else:
            e.set_task(tasks)
        e.reset()
        e.rollout(3)
        envs.append(e)
    return envs


def maze_rollout(shape, env, pol, T, state, rs, out=None, seed=SEED):
    rs = dict(seed=SEED, **CFG) if rs else None
    if shape.kind == "mlp":
        return env.rollout(T, policy=pol, act_seed=seed, resample=rs, out=out)
    return env.rollout(T, policy=pol, state=state, act_seed=seed, resample=rs, want_hidden=True, out=out)


def assert_maze_env_side(out, ref):
    """obs, rew, done bit for bit, and the terminal outputs the policy rollout produced."""
    if out.get("final_obs") is not None and out.get("truncated") is not None:
        mlp_t.assert_env_side_equal(out, ref)
        return
    for k in ("obs", "rew", "done"):
        assert torch.equal(out[k], ref[k]), k
    if out.get("truncated") is not None:
        assert torch.equal(out["truncated"], ref["truncated"])


def check_maze(shape, env, twin, T, rs, rec, out=None):
    """Run `shape` on env from a random carried state, then check the env side against the twin, the policy side against
    the float64 reference and the state written back.  Returns the rollout's outputs."""
    n = env.num_envs
    model, pol = shape.policy(env, seed=shape.H + len(shape.widths) + shape.width)
    state = before = None
    if shape.kind != "mlp":
        state = gru_t.random_state(pol, n)
        before = state.clone()
    t0 = env._counters()
    out = maze_rollout(shape, env, pol, T, state, rs, out)
    assert out["done"].any(), "no episode ended: auto-reset (and the reset rule) is not exercised"
    ref = twin.rollout(T, actions=out["act"], resample=dict(seed=SEED, **CFG) if rs else None)
    assert_maze_env_side(out, ref)
    if rec:
        for x, y in zip(env.trajectory(), twin.trajectory()):
            assert torch.equal(x, y)
    if rs:
        for x, y in zip(env.agent_state(), twin.agent_state()):
            assert torch.equal(x, y)
    if shape.kind == "mlp":
        worst, _ = mlp_t.check_policy_side(env, model, out, SEED, t0)
        assert worst <= 1.0, worst
        return out
    wipe = shape.reset == "episode" or bool(rs)
    assert torch.equal(out["state0"], before)
    if shape.kind == "gru":
        worst, logits, lb = gru_t.teacher_forced(pol, out, wipe)
        assert worst <= 1.0, worst
        assert gru_t.check_actions(env, logits, lb, out, SEED, t0) <= 1.0
        assert torch.equal(state, gru_t.expected_state(pol, out, wipe))
    else:
        worst, logits, lb, c_ref, ec = lstm_t.teacher_forced(pol, out, wipe)
        assert worst <= 1.0, worst
        assert gru_t.check_actions(env, logits, lb, out, SEED, t0) <= 1.0
        lstm_t.check_state(pol, out, state, wipe, c_ref, ec)
    return out


# ---------------------------------------------------------------------------------------------------------------
# 1. The maze instantiation matrix: kind x FIN x REC x RS, one case per compiled kernel
# ---------------------------------------------------------------------------------------------------------------

# eight shapes per kind, one per (FIN, REC, RS) in product order: H in {1, 8, 17, 64}, widths that are not multiples of
# 8, both activations, both task types, feedback on and off, both reset rules, view_grid 1 and 2
MATRIX_SHAPES = {
    "mlp": [Shape("mlp", (17,), act=nn.ReLU), Shape("mlp", (64, 64), task_type="ESCAPE"),
            Shape("mlp", (1, 8), view_grid=2), Shape("mlp", (), act=nn.ReLU, task_type="ESCAPE"),
            Shape("mlp", (5, 64, 1), act=nn.ReLU, view_grid=2), Shape("mlp", (8,)),
            Shape("mlp", (33, 17), task_type="ESCAPE", view_grid=2), Shape("mlp", (64,), act=nn.ReLU)],
    "gru": [Shape("gru", H=1, width=5, reset="task"), Shape("gru", H=8, width=0, feedback=False, task_type="ESCAPE"),
            Shape("gru", H=17, width=13, act=nn.ReLU, view_grid=2), Shape("gru", H=64, width=0, reset="task"),
            Shape("gru", H=64, width=64, act=nn.ReLU, task_type="ESCAPE"), Shape("gru", H=17, width=0, reset="task"),
            Shape("gru", H=8, width=33, feedback=False, view_grid=2), Shape("gru", H=1, width=0, task_type="ESCAPE")],
    "lstm": [Shape("lstm", H=17, width=0, reset="task", task_type="ESCAPE"), Shape("lstm", H=1, width=3),
             Shape("lstm", H=8, width=64, act=nn.ReLU, feedback=False, view_grid=2),
             Shape("lstm", H=64, width=0, reset="task"), Shape("lstm", H=17, width=33, task_type="ESCAPE"),
             Shape("lstm", H=64, width=64, act=nn.ReLU), Shape("lstm", H=1, width=0, reset="task", view_grid=2),
             Shape("lstm", H=8, width=5, feedback=False, task_type="ESCAPE")],
}
MATRIX = [(kind, fin, rec, rs, MATRIX_SHAPES[kind][4 * fin + 2 * rec + rs])
          for kind in ("mlp", "gru", "lstm") for fin in (0, 1) for rec in (0, 1) for rs in (0, 1)]


@pytest.mark.parametrize("kind,fin,rec,rs,shape", MATRIX,
                         ids=["%s-fin%d-rec%d-rs%d-%r" % (k, f, r, s, sh) for k, f, r, s, sh in MATRIX])
def test_maze_instantiation_matrix(tasks, kind, fin, rec, rs, shape):  # noqa: F811
    """FIN off: final_obs=False, so the rollout produces neither terminal rows nor truncation flags."""
    n, T = 300, 24
    env, twin = maze_pair(n, shape, rs, rec, bool(fin), tasks)
    out = check_maze(shape, env, twin, T, rs, rec)
    assert ("final_obs" in out) == bool(fin) and ("truncated" in out) == bool(fin)
    for e in (env, twin):
        e.close()


def maze_outputs(env, kind, pol, T, keys, fill=True):
    """A caller-owned `out` dict holding exactly `keys`, every buffer filled with a sentinel (or left empty)."""
    N, dev = env.num_envs, env.device
    shape = tuple(env._obs.shape[1:])
    spec = {"obs": ((T, N) + shape, torch.float32), "rew": ((T, N), torch.float64), "done": ((T, N), torch.uint8),
            "act": ((T, N), torch.int32), "logp": ((T, N), torch.float32), "obs0": ((N,) + shape, torch.float32),
            "final_obs": ((T, N) + shape, torch.float32), "truncated": ((T, N), torch.uint8)}
    if kind != "mlp":
        spec["state0"] = ((N, pol.state_dim), torch.float32)
        spec["hid"] = ((T, N, pol.hidden), torch.float32)
    return {k: sentinel(*spec[k], dev, fill) for k in keys}


def sentinel(shape, dtype, dev, fill=True):
    t = torch.empty(shape, dtype=dtype, device=dev)
    if fill:
        t.fill_(-12345.0 if dtype.is_floating_point else (0xAB if dtype == torch.uint8 else -7))
    return t


@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm"])
def test_maze_truncated_without_final_obs(tasks, kind):  # noqa: F811
    """FIN on through `truncated` alone: an `out` without final_obs.  The flags match the twin's, and nothing else moves."""
    n, T = 300, 24
    shape = {"mlp": Shape("mlp", (17, 5)), "gru": Shape("gru", H=17, width=5),
             "lstm": Shape("lstm", H=8, width=0, reset="task")}[kind]
    env, twin = maze_pair(n, shape, False, False, True, tasks)
    _, pol = shape.policy(env, seed=shape.H + len(shape.widths) + shape.width)
    keys = ["obs", "rew", "done", "act", "logp", "obs0", "truncated"] + ([] if kind == "mlp" else ["state0", "hid"])
    out = check_maze(shape, env, twin, T, False, False, out=maze_outputs(env, kind, pol, T, keys))
    assert "final_obs" not in out and out["truncated"].any()
    for e in (env, twin):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 2. The quadrotor instantiation matrix and the configurations the policy tests skip
# ---------------------------------------------------------------------------------------------------------------

def make_quad(n, task, **kw):
    from metagym_b200 import BatchedQuadrotor
    if task == "velocity_control":
        kw.setdefault("seed", [0, 1, 2])
    kw.setdefault("nt", 20)
    return BatchedQuadrotor(task=task, dt=0.005, num_envs=n, device=0, squeeze=False, rng_seed=5, **kw)


def check_quad(env, T=32, widths=(64, 64), act=nn.Tanh, seed=0):
    """Policy rollout from a snapshot, then the open-loop rollout from the same snapshot fed its actions; the policy side
    against the float64 forward pass.  Returns the policy rollout's outputs."""
    env.reset()
    env.rollout(5)                                   # t_base != 0
    m, pol = quad_t.make_policy(env, widths, act, seed, LOG_STD)
    snap = env.snapshot()
    t0 = env._counters()
    out = env.rollout(T, policy=pol, act_seed=SEED)
    assert out["done"].any(), "no episode ended"
    records = env.snapshot()["records"].clone()
    env.restore(snap)
    ref = env.rollout(T, actions=out["act"])
    quad_t.assert_env_side_equal(out, ref, want_final=env._want_final)
    assert torch.equal(env.snapshot()["records"], records)
    assert quad_t.check_policy_side(env, m, LOG_STD, out, SEED, t0) <= 1.0
    return out


def general():
    from oracle import quad_oracle as qo
    return qo.general_params()


@pytest.mark.parametrize("fin", [False, True], ids=["fin0", "fin1"])
@pytest.mark.parametrize("simple", [True, False], ids=["default", "general"])
def test_quad_instantiation_matrix(simple, fin):
    """quad_rollout_kernel<SIMPLE, 0, FIN, true>: the default physics (SIMPLE) and qo.general_params(), FIN off
    (final_obs=False) and on."""
    task = "velocity_control" if fin else "hovering_control"
    env = make_quad(300, task, final_obs=fin, auto_reset=True, simulator_conf=None if simple else general())
    assert env.step_kernel_name().endswith("<true>" if simple else "<false>")      # the SIMPLE the handle runs
    out = check_quad(env, widths=(64, 17) if simple else (64, 64), act=nn.ReLU if fin else nn.Tanh)
    assert ("final_obs" in out) == fin
    env.close()


@pytest.mark.parametrize("simple", [True, False], ids=["default", "general"])
def test_quad_rk4(simple):
    env = make_quad(200, "hovering_control", final_obs=True, auto_reset=True, integrator="rk4", rk4_steps=2,
                    simulator_conf=None if simple else general())
    check_quad(env, widths=(33,))
    env.close()


@pytest.mark.parametrize("task", ["hovering_control", "no_collision"])
def test_quad_obstacle_map(quad_golden, tmp_path, task):
    path = tmp_path / "map.txt"
    path.write_text("".join(" ".join(str(int(v)).zfill(2) for v in row) + "\n" for row in quad_golden["map_obst"]))
    env = make_quad(200, task, final_obs=True, auto_reset=True, map_file=str(path))
    check_quad(env, widths=(64, 5, 64))
    env.close()


@pytest.mark.parametrize("task", ["velocity_control", "hovering_control"])
def test_quad_without_auto_reset(task):
    """auto_reset=False: finished envs keep stepping; the episodes (nt = 12) end inside the launch."""
    env = make_quad(200, task, nt=12, auto_reset=False)
    out = check_quad(env, T=24)
    assert bool(out["done"].any(0).all()), "an episode did not end inside the launch"
    env.close()


# ---------------------------------------------------------------------------------------------------------------
# 3. Wide windows and the largest footprints, checked numerically
# ---------------------------------------------------------------------------------------------------------------

OPTIN_H100 = 232448      # cudaDevAttrMaxSharedMemoryPerBlockOptin of the H100


def tiles_bytes(view_grid, rs, maze_n, threads=THREADS):
    """maze2d_tiles_bytes: two observation tiles, plus one sampler workspace per warp when resampling (7 n^2 + ((n -
    1) / 2)^2 bytes rounded up to 16), rounded up to 16 bytes."""
    D = (2 * view_grid + 1) ** 2
    b = 2 * threads * D * 4
    if rs:
        b += threads // 32 * ((7 * maze_n * maze_n + ((maze_n - 1) // 2) ** 2 + 15) // 16 * 16)
    return (b + 15) // 16 * 16


def mlp_staged(n_in, widths):
    """mgb_mlp_plan's staged floats without log_std: per layer, its rows (the outputs rounded up to the group, 8 for a
    hidden layer and 4 for the output layer) times its inputs, then one bias per row, padded to 8 floats."""
    s, ins, outs = 0, [n_in] + list(widths), list(widths) + [4]
    for k, (i, o) in enumerate(zip(ins, outs)):
        g = 4 if k == len(outs) - 1 else 8
        rows = (o + g - 1) // g * g
        s = (s + rows * i + rows + 7) // 8 * 8
    return s


def smem_bytes(kind, view_grid, H=0, widths=(), feedback=True, rs=False, maze_n=15, threads=THREADS):
    """Dynamic shared memory of a policy rollout CTA (the kernels have no static shared memory): the tiles, then
    - MLP (mgb_mlp_smem_bytes): the staged layers and two activation buffers of max(D, hidden widths) rows;
    - GRU / LSTM (mgb_rnn_smem_bytes): NG gates of weight_ih and weight_hh and 2 NG biases per unit, H padded to 8, the
      head (widths: () or (w,)) as an MLP on H inputs, and the columns x [in], c [C], h0 [Hr], h1 [Hr], w [Hw] with
      GRU: C = 0, Hr = H, Hw = w; LSTM: C = H, Hr = max(H, w), Hw = 0."""
    D = (2 * view_grid + 1) ** 2
    base = tiles_bytes(view_grid, rs, maze_n, threads)
    if kind == "mlp":
        return base + (mlp_staged(D, widths) + 2 * max([D] + list(widths)) * threads) * 4
    NG = 3 if kind == "gru" else 4
    Hp, n_in, w = (H + 7) // 8 * 8, D + 5 * feedback, (widths[0] if widths else 0)
    staged = NG * Hp * n_in + NG * Hp * H + 2 * NG * Hp + mlp_staged(H, widths)
    C, Hr, Hw = (0, H, w) if NG == 3 else (H, max(H, w), 0)
    return base + (staged + (n_in + C + 2 * Hr + Hw) * threads) * 4


def largest_h(kind, view_grid, width, rs, maze_n=9, optin=OPTIN_H100):
    fits = [H for H in range(1, 65)
            if smem_bytes(kind, view_grid, H, (width,) if width else (), True, rs, maze_n) <= optin]
    return max(fits) if fits else None


def test_restated_footprints_agree():
    """The restatement here is the LSTM test's for the LSTM, and gives DESIGN.md's "largest H that fits" tables (15 x 15
    mazes with resampling)."""
    for vg in range(1, 7):
        for H in (1, 8, 17, 29, 64):
            for w in (0, 5, 64):
                for rs in (False, True):
                    assert smem_bytes("lstm", vg, H, (w,) if w else (), True, rs, 15) == \
                        lstm_t.smem_bytes(vg, H, w, True, rs, n=15)
    table = {"lstm": [[64, 61, 48, 29, 8, None], [64, 59, 45, 26, 8, None], [64, 56, 36, 15, None, None],
                      [64, 53, 32, 9, None, None]],
             "gru": [[64, 64, 61, 40, 15, None], [64, 64, 58, 37, 10, None], [64, 64, 47, 24, None, None],
                     [64, 61, 44, 24, None, None]]}
    for kind, rows in table.items():
        for (w, rs), row in zip(((0, False), (0, True), (64, False), (64, True)), rows):
            assert [largest_h(kind, vg, w, rs, 15) for vg in range(1, 7)] == row, (kind, w, rs)


WIDE = ([(Shape("mlp", (64, 64), view_grid=3), False), (Shape("mlp", (64, 64), view_grid=4, task_type="ESCAPE"), True),
         (Shape("mlp", (), view_grid=4), False)]
        + [(Shape(kind, H=largest_h(kind, vg, w, rs), width=w, reset="task" if rs else "episode", view_grid=vg), rs)
           for kind in ("gru", "lstm") for vg in (3, 4) for w in (0, 64) for rs in (False, True)])


@pytest.mark.parametrize("shape,rs", WIDE, ids=["%r-rs%d" % w for w in WIDE])
def test_wide_windows_at_the_largest_footprint(tasks, shape, rs):  # noqa: F811
    """view_grid 3 and 4 with every output on; a cell at the largest H that fits its window, head and resampling (9 x 9
    mazes, DESIGN.md "largest H that fits")."""
    n, T = 300, 24
    env, twin = maze_pair(n, shape, rs, True, True, tasks)
    optin = torch.cuda.get_device_properties(env.device).shared_memory_per_block_optin
    head = shape.widths if shape.kind == "mlp" else ((shape.width,) if shape.width else ())
    assert smem_bytes(shape.kind, shape.view_grid, shape.H, head, True, rs, 9) <= optin
    if shape.kind != "mlp" and shape.H < 64:
        assert smem_bytes(shape.kind, shape.view_grid, shape.H + 1, head, True, rs, 9) > optin
    check_maze(shape, env, twin, T, rs, True)
    for e in (env, twin):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 4. MLP and GRU footprint boundaries
# ---------------------------------------------------------------------------------------------------------------

def footprint_env(n, view_grid, rs, maze_n, tasks):  # noqa: F811
    e = mlp_t.make_env(n, view_grid=view_grid)
    if rs:
        e.set_task(slot_table(maze_n, n)[0], env2task=np.arange(n))
    else:
        e.set_task(tasks)
    e.reset()
    return e


def assert_boundary(lib, e, call, want, optin, state=None):
    """rc 0 when `want` fits; otherwise the refusal names exactly `want` bytes, and the counters, the launch count, the
    env state and the carried state are untouched."""
    records = e.snapshot()["records"].clone()
    before = (e._counters(), e.launch_count, None if state is None else state.clone())
    rc = call()
    torch.cuda.synchronize()
    if want <= optin:
        assert rc == 0, lib.mgb_last_error().decode()
        return
    msg = lib.mgb_last_error().decode()
    assert rc == MGB_ERR_ARG and "needs %d bytes of shared memory" % want in msg, (want, msg)
    assert e._counters() == before[0] and e.launch_count == before[1]
    assert torch.equal(e.snapshot()["records"], records)
    if state is not None:
        assert torch.equal(state, before[2])


def test_mlp_footprint_boundary(tasks):  # noqa: F811
    """The largest MLP that fits runs and the next one up is refused: in view_grid (4 fits with three 64-wide layers,
    5 does not even without hidden layers, the activation buffers hold the window), and in the last hidden layer's
    width with resampling (21 x 21 mazes), and with a 31 x 31 maze's sampler workspaces, where (64, 64) fits with 32
    bytes to spare and one more layer does not."""
    from metagym_b200 import _lib
    n, T = 128, 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert optin == OPTIN_H100
    fits = [w for w in range(1, 65) if smem_bytes("mlp", 4, widths=(64, 64, w), rs=True, maze_n=21) <= optin]
    w21 = max(fits)
    assert 1 < w21 < 64
    assert optin - smem_bytes("mlp", 4, widths=(64, 64), rs=True, maze_n=31) == 32
    shapes = [(4, (64, 64, 64), False, 15), (5, (), False, 15), (4, (64, 64, w21), True, 21),
              (4, (64, 64, w21 + 1), True, 21), (4, (64, 64), True, 31), (4, (64, 64, 1), True, 31)]
    results = []
    for vg, widths, rs, maze_n in shapes:
        e = footprint_env(n, vg, rs, maze_n, tasks)
        lib = e._lib
        _, pol = mlp_t.make_policy(e, widths)
        cfg = e._sampler_cfg(seed=1, **CFG)[0] if rs else None
        want = smem_bytes("mlp", vg, widths=widths, rs=rs, maze_n=maze_n)

        def call():
            return lib.mgb_maze_rollout_policy(e._h, T, ctypes.byref(pol.struct()), 0,
                                               ctypes.byref(cfg) if rs else None, 0, None, None, None, None, None,
                                               None, None, None, e._stream())
        assert_boundary(lib, e, call, want, optin)
        results.append(want <= optin)
        if want > optin:
            with pytest.raises(_lib.MgbError):
                e.rollout(T, policy=pol, resample=dict(seed=1, **CFG) if rs else None)
        e.close()
    assert results == [True, False, True, False, True, False]


# view_grid, largest H, head width, resampling (9 x 9 mazes)
GRU_LARGEST = [(3, 61, 0, False), (4, 40, 0, False), (5, 15, 0, False), (3, 47, 64, False), (4, 24, 64, False),
               (3, 60, 0, True), (2, 63, 64, True), (5, 13, 0, True)]


def test_gru_footprint_boundary(tasks):  # noqa: F811
    """Each shape is the largest GRU that fits its view_grid, head and resampling; H + 1 is refused with the exact
    byte count and nothing touched."""
    from metagym_b200 import _lib
    n, T = 128, 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    for vg, H, w, rs in GRU_LARGEST:
        assert largest_h("gru", vg, w, rs, 9, optin) == H, (vg, H, w, rs)
    for vg, H, w, rs in [(vg, H + k, w, rs) for vg, H, w, rs in GRU_LARGEST for k in (0, 1)]:
        e = footprint_env(n, vg, rs, 9, tasks)
        lib = e._lib
        pol = gru_t.make_policy(e, H, w)
        st = gru_t.random_state(pol, n)
        cfg = e._sampler_cfg(seed=1, **CFG)[0] if rs else None
        want = smem_bytes("gru", vg, H, (w,) if w else (), True, rs, 9)

        def call():
            return lib.mgb_maze_rollout_rnn(e._h, T, ctypes.byref(pol.struct()), 0, ctypes.byref(cfg) if rs else None,
                                            0, _lib.ptr(st), None, None, None, None, None, None, None, None, None,
                                            None, e._stream())
        assert_boundary(lib, e, call, want, optin, st)
        if want > optin:
            with pytest.raises(_lib.MgbError):
                e.rollout(T, policy=pol, state=st, resample=dict(seed=1, **CFG) if rs else None)
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 5. The null-output contract of mgb_maze_rollout_policy, mgb_maze_rollout_rnn and mgb_quad_rollout_policy
# ---------------------------------------------------------------------------------------------------------------

OPTIONAL = ("act", "logp", "obs0", "obs", "rew", "done", "final_obs", "truncated")     # + state0, hid for the cells


def assert_drops_change_nothing(env, keys, run, alloc, state0=None):
    """Run from a snapshot (and a clone of state0) with every output, then without each output in turn and without all
    of them: the outputs that remain, the snapshot records and the carried state are bit-identical every time."""
    snap = env.snapshot()

    def once(ks):
        env.restore(snap)
        st = None if state0 is None else state0.clone()
        out = alloc(ks)
        run(out, st)
        return out, env.snapshot()["records"].clone(), st

    full, rec, st_full = once(keys)
    assert full["done"].any()
    for drop in [(k,) for k in keys] + [tuple(keys)]:
        out, r, st = once([k for k in keys if k not in drop])
        for k in keys:
            if k not in drop:
                assert torch.equal(out[k], full[k]), (drop, k)
        assert torch.equal(r, rec), drop
        if state0 is not None:
            assert torch.equal(st, st_full), drop


NULL_MAZE = [(Shape("mlp", (17, 64)), False), (Shape("mlp", (5,), act=nn.ReLU, view_grid=2), True),
             (Shape("gru", H=17, width=5), False), (Shape("gru", H=8, width=0, reset="task"), True),
             (Shape("lstm", H=17, width=0), False), (Shape("lstm", H=8, width=33, reset="task", view_grid=2), True)]


@pytest.mark.parametrize("shape,rs", NULL_MAZE, ids=["%r-rs%d" % (s, r) for s, r in NULL_MAZE])
def test_maze_null_outputs(tasks, shape, rs):  # noqa: F811
    n, T = 200, 24
    env, twin = maze_pair(n, shape, rs, True, True, tasks)
    twin.close()
    _, pol = shape.policy(env, seed=3)
    keys = OPTIONAL + (() if shape.kind == "mlp" else ("state0", "hid"))
    state0 = None if shape.kind == "mlp" else gru_t.random_state(pol, n)
    assert_drops_change_nothing(env, keys, lambda out, st: maze_rollout(shape, env, pol, T, st, rs, out),
                                lambda ks: maze_outputs(env, shape.kind, pol, T, ks), state0)
    env.close()


def test_maze_snapshot_records_do_not_depend_on_the_buffer(tasks):  # noqa: F811
    """With path recording the entries (2 (max_steps + 1) bytes) are padded to 16 bytes in each record; a snapshot
    writes the padding too, so that the same state gives the same records whatever the buffer held."""
    env = mlp_t.make_env(100, record_path=True)
    env.set_task(tasks)
    env.reset()
    env.rollout(5)
    snaps = [env.snapshot() for _ in range(2)]
    for s, v in zip(snaps, (0x00, 0xFF)):
        s["records"].fill_(v)
        env.snapshot(out=s)
    assert torch.equal(snaps[0]["records"], snaps[1]["records"])
    env.close()


def quad_outputs(env, T, keys):
    N, D, dev = env.num_envs, env.obs_dim, env.device
    spec = {"obs": (T, N, D), "rew": (T, N), "act": (T, N, 4), "logp": (T, N), "obs0": (N, D), "final_obs": (T, N, D)}
    return {k: sentinel(spec[k], torch.float32, dev) if k in spec else sentinel((T, N), torch.uint8, dev)
            for k in keys}


@pytest.mark.parametrize("task", ["velocity_control", "hovering_control"])
def test_quad_null_outputs(task):
    n, T = 200, 32
    env = make_quad(n, task, final_obs=True, auto_reset=True)
    env.reset()
    env.rollout(5)
    _, pol = quad_t.make_policy(env, (64, 17), nn.Tanh, 0, LOG_STD)
    assert_drops_change_nothing(env, OPTIONAL, lambda out, st: env.rollout(T, policy=pol, act_seed=SEED, out=out),
                                lambda ks: quad_outputs(env, T, ks))
    env.close()


# ---------------------------------------------------------------------------------------------------------------
# 6. Batch tails: misaligned bulk-store destinations, partial warps and CTAs
# ---------------------------------------------------------------------------------------------------------------

TAIL_SHAPES = {"mlp": Shape("mlp", (17, 64)), "gru": Shape("gru", H=17, width=5, reset="task"),
               "lstm": Shape("lstm", H=8, width=0)}
TAILS = [(kind, n, rs) for kind in ("mlp", "gru", "lstm") for n in (1, 31, 129, 161) for rs in (False, True)]


@pytest.mark.parametrize("kind,n,rs", TAILS, ids=["%s-n%d-rs%d" % t for t in TAILS])
def test_maze_batch_tails(tasks, kind, n, rs):  # noqa: F811
    """view_grid 1: D = 9 floats per env, so a step's obs block starts at t n D 4 bytes, 16-byte aligned only for even t
    when n is odd, and the last CTA's (or, with resampling, the last warp's) rows are not a multiple of 16 bytes: the
    per-element stores run."""
    shape = TAIL_SHAPES[kind]
    T = 24
    env, twin = maze_pair(n, shape, rs, False, True, tasks)
    check_maze(shape, env, twin, T, rs, False)
    for e in (env, twin):
        e.close()


@pytest.mark.parametrize("n", [1, 65])
def test_quad_batch_tails(n):
    """64 envs per CTA: a single env, and a last CTA holding one env."""
    env = make_quad(n, "velocity_control", final_obs=True, auto_reset=True)
    check_quad(env, T=48)
    env.close()
