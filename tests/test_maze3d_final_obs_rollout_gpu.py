"""GPU tests of terminal observations and truncation flags from the fused MetaMaze 3-D rollouts (mgb_maze_rollout):
maze3d_rollout_kernel<true> (discrete, pose cache) and maze3d_kernel<false, true, true> (continuous, direct
renderer).  Against step() twins with final_obs=True bit for bit, against
handles that run the plain rollout (whose outputs must not move), and against the CPU oracle."""
import itertools

import numpy as np
import pytest

from maze_continuous_draws import maze_continuous_rollout_actions
from util import task_from_arrays

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
MAX_STEPS = 17      # with step_reward = -1/16 and no food eaten, life 1.0 runs out exactly on the last allowed step
SENTINEL = {"uint8": 77, "int32": -7, "float32": -7.0}


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


@pytest.fixture(scope="module")
def tasks(maze_golden):
    """Five 15x15 tasks whose episodes end in every way.  SURVIVAL, step_reward -1/16: tasks 0, 3 and 4 start with life
    1.0, so an env that eats nothing dies on step 17, the last allowed one (death and time-out coincide); task 1 starts
    with 2.0 and times out alive; task 2 loses 0.5 per step from 0.5 and dies on step 2 with life -0.5, whose life-bar end
    index is negative and wraps like a Python slice (maze_discrete_3d.py:118-126).  ESCAPE: the goal of tasks 0 and 2 is
    an open cell next to the start, tasks 1 and 3 keep their far goal and time out, and task 4 is walled in on its start
    cell, which is its goal: its envs finish on every step, so every one of their rollout items is doubled."""
    g = maze_golden
    out = []
    for k in range(5):
        j = k % 4
        t = task_from_arrays(g["tasks15.walls"][j], g["tasks15.texts"][j], g["tasks15.food"][j],
                             g["tasks15.interval"][j] // 10, g["tasks15.scalars"][j])
        t = t._replace(step_reward=(-0.0625, -0.0625, -0.5, -0.0625, -0.0625)[k],
                       initial_life=(1.0, 2.0, 0.5, 1.0, 1.0)[k], max_life=2.0)
        w = np.array(t.cell_walls)
        sx, sy = t.start
        near = [(sx + dx, sy + dy) for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1))]
        if k in (0, 2):
            t = t._replace(goal=[c for c in near if w[c] == 0][0])
        if k == 4:
            for c in near:
                w[c] = 1
            t = t._replace(cell_walls=w, goal=tuple(t.start))
        out.append(t)
    return out


def make_env(kind, task_type, n, res, dtype, textures, monkeypatch, pipe=None, **kw):
    from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    if pipe is not None:
        monkeypatch.setenv("MGB_MAZE_RENDER_PIPE", pipe)       # read when the handle is created
    cls = BatchedMetaMazeContinuous3D if kind == "C3D" else BatchedMetaMazeDiscrete3D
    kw = dict(dict(max_steps=MAX_STEPS, task_type=task_type, num_envs=n, squeeze=False, auto_reset=True), **kw)
    return cls(resolution=res, obs_dtype=dtype, textures=textures, **kw)


def ready(env, tasks):
    env.set_task(tasks)
    env.reset()
    return env


def random_actions(torch, kind, rng, T, n):
    if kind == "C3D":
        return torch.as_tensor(rng.uniform(-1.3, 1.3, (T, n, 2)).astype(np.float32)).cuda()   # clipped by the kernel
    return torch.as_tensor(rng.randint(0, 4, (T, n)).astype(np.int32)).cuda()


def full_out(torch, env, T, drawn=False):
    """A caller's out dict with final_obs pre-filled with a sentinel (rows with done = 0 must keep it)."""
    n, shape, dt = env.num_envs, tuple(env._obs.shape[1:]), env._obs.dtype
    act_shape = (T, n, 2) if env.KIND == 2 else (T, n)
    return {"obs": torch.empty((T, n) + shape, dtype=dt, device="cuda"),
            "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
            "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"),
            "act": torch.empty(act_shape, dtype=torch.float32 if env.KIND == 2 else torch.int32, device="cuda")
            if drawn else None,
            "final_obs": torch.full((T, n) + shape, SENTINEL[env.obs_dtype], dtype=dt, device="cuda"),
            "truncated": torch.full((T, n), 9, dtype=torch.uint8, device="cuda")}


def state(env):
    out = list(env.agent_state())
    if env.KIND == 2:
        out += list(env.pose())
    return out


def assert_same_state(torch, a, b):
    for x, y in zip(state(a), state(b)):
        assert torch.equal(x, y)


def oracle_frame(dtype, o):
    """The oracle's observation in the obs dtype (uint8 = min(value, 255))."""
    v = o._observe()
    if dtype == "uint8":
        return np.minimum(v, 255).astype(np.uint8)
    return v.astype(np.float32) if dtype == "float32" else v


# ---------------------------------------------------------------------------------------------------------------------
# 1. rollout = single steps, and = the plain rollout
# ---------------------------------------------------------------------------------------------------------------------
# discrete: a CTA owns several envs above 5 x the SM count (660 on an H100); continuous: above the SM count
DISC_SHAPES = [((32, 32), 24), ((40, 24), 700)]
CONT_SHAPES = [((32, 32), 150), ((40, 24), 24), ((40, 24), 150), ((32, 32), 24)]
CASES = [("D3D", dt, tt, None) + DISC_SHAPES[(k + k // 2) % 2]
         for k, (dt, tt) in enumerate(itertools.product(["uint8", "int32", "float32"], ["SURVIVAL", "ESCAPE"]))]
CASES += [("C3D", dt, tt, pipe) + CONT_SHAPES[(k // 2) % 4]
          for k, (dt, tt, pipe) in enumerate(itertools.product(["uint8", "int32", "float32"], ["SURVIVAL", "ESCAPE"],
                                                               ["1", "0"]))]
# a screen whose two record sets do not fit in shared memory with their crossing lists: the lists go to global scratch
CASES += [("C3D", "uint8", "SURVIVAL", "1", (256, 256), 20)]


@pytest.mark.parametrize("kind,dtype,task_type,pipe,res,n", CASES)
def test_rollout_equals_single_steps(torch_mod, textures, tasks, monkeypatch, kind, dtype, task_type, pipe, res, n):
    """rollout(T, actions, final_obs=True, out=...) against T step() calls of a final_obs=True twin: obs, rew, done and
    truncated of every step, final_obs where done, the sentinel where done is 0, the state (and pose) at the end.  A
    third handle's plain rollout gives the same obs, rew, done and state."""
    torch = torch_mod
    roll, twin, plain = (ready(make_env(kind, task_type, n, res, dtype, textures, monkeypatch, pipe, final_obs=f), tasks)
                         for f in (False, True, False))
    T = 40
    acts = random_actions(torch, kind, np.random.RandomState(n + res[0]), T, n)
    out = full_out(torch, roll, T)
    assert roll.rollout(T, actions=acts, out=out, final_obs=True) is out
    ref = plain.rollout(T, actions=acts)
    assert "final_obs" not in ref and "truncated" not in ref
    for k in ("obs", "rew", "done"):
        assert torch.equal(ref[k], out[k]), k
    kinds = np.zeros(3, np.int64)      # terminal, truncated, terminal on the last allowed step
    for t in range(T):
        steps_before = twin.agent_state()[0][:, 3].cpu().numpy()
        o, r, d, _ = twin.step(acts[t])
        assert torch.equal(out["obs"][t], o), (t, int((out["obs"][t] != o).sum()))
        assert torch.equal(out["rew"][t], r) and torch.equal(out["done"][t].bool(), d), t
        assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
        assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
        assert (out["final_obs"][t][~d] == SENTINEL[dtype]).all(), t
        term = (d & ~twin.truncated).cpu().numpy()
        kinds += [term.sum(), twin.truncated.sum().item(), (term & (steps_before + 1 == MAX_STEPS)).sum()]
    assert_same_state(torch, roll, twin)
    assert_same_state(torch, roll, plain)
    assert kinds[0] > 0 and kinds[1] > 0, kinds
    if task_type == "SURVIVAL":
        assert kinds[2] > 0, kinds     # a death on the last allowed step is terminal, not truncated
    else:
        assert out["done"][:, 4::5].bool().all()      # the walled-in task: every item doubled
    if res == (256, 256):
        assert roll.cache_info()["hits_in_global"]
    for e in (roll, twin, plain):
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. against the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
@pytest.mark.parametrize("kind", ["D3D", "C3D"])
def test_terminal_frames_vs_oracle(torch_mod, textures, tasks, monkeypatch, kind, task_type):
    """Per finished env: final_obs is the oracle's step observation, obs is the oracle's reset(), truncated is the step
    limit rule on the oracle's state.  The continuous rollout draws its actions on the device, restated with
    maze_continuous_rollout_actions; two chunks, so the second starts at t_base = T."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    n, res, dtype, seed = 25, (40, 24), "int32", 2 ** 33 + 5
    env = ready(make_env(kind, task_type, n, res, dtype, textures, monkeypatch), tasks)
    oracles = []
    for e in range(n):
        o = OracleMaze("C3D" if kind == "C3D" else "3D", task_type, MAX_STEPS, 1, res, textures=textures)
        o.set_task(tasks[e % 5])
        o.reset()
        oracles.append(o)
    rng = np.random.RandomState(4)
    t_base, n_done, n_trunc = 0, 0, 0
    for T in (30, 20):
        if kind == "C3D":
            out = env.rollout(T, act_seed=seed, final_obs=True)
            acts = [maze_continuous_rollout_actions(seed, np.arange(n), t_base + t) for t in range(T)]
        else:
            a = rng.randint(0, 4, (T, n)).astype(np.int32)
            out = env.rollout(T, actions=torch.as_tensor(a).cuda(), final_obs=True)
            acts = list(a)
        obs, rew, done = out["obs"].cpu().numpy(), out["rew"].cpu().numpy(), out["done"].cpu().numpy()
        fin, trunc = out["final_obs"].cpu().numpy(), out["truncated"].cpu().numpy()
        for t in range(T):
            for e in range(n):
                o = oracles[e]
                _, r2, d2, _ = o.step(acts[t][e], render=False)
                assert rew[t, e] == r2 and bool(done[t, e]) == d2, (t_base + t, e)
                if d2:
                    over = o.env.steps > MAX_STEPS - 1
                    goal = tuple(tasks[e % 5].goal)
                    ended = o.life < 0 if task_type == "SURVIVAL" else (o.env.gx, o.env.gy) == goal
                    assert trunc[t, e] == (over and not ended), (t_base + t, e)
                    assert np.array_equal(fin[t, e], oracle_frame(dtype, o)), (t_base + t, e)
                    o.reset()
                    n_done += 1
                    n_trunc += int(trunc[t, e])
                else:
                    assert trunc[t, e] == 0, (t_base + t, e)
                assert np.array_equal(obs[t, e], oracle_frame(dtype, o)), (t_base + t, e)
        t_base += T
    assert n_done > n_trunc > 0
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. drawn actions and the generator's step counter
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["D3D", "C3D"])
def test_drawn_actions_do_not_move(torch_mod, textures, tasks, monkeypatch, kind):
    """Two drawn chunks with final_obs on and off: the same actions, frames, rewards and dones, so t_base advanced
    identically; and the same state afterwards."""
    torch = torch_mod
    n, res = 30, (32, 32)
    on, off = (ready(make_env(kind, "ESCAPE", n, res, "uint8", textures, monkeypatch, env_index_base=500), tasks)
               for _ in range(2))
    for T in (13, 9):
        a = on.rollout(T, act_seed=77, want_actions=True, final_obs=True)
        b = off.rollout(T, act_seed=77, want_actions=True)
        for k in ("act", "obs", "rew", "done"):
            assert torch.equal(a[k], b[k]), (T, k)
        assert int(a["done"].sum()) > 0
    assert_same_state(torch, on, off)
    on.close(); off.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. CUDA-graph capture
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,pipe", [("D3D", None), ("C3D", "1"), ("C3D", "0")])
def test_graph_replay_equals_eager_rollouts(torch_mod, textures, tasks, monkeypatch, kind, pipe):
    """rollout(final_obs=True, out=...) captured in a CUDA graph right after reset() and replayed K times equals K eager
    rollouts into an identically initialised out dict."""
    torch = torch_mod
    n, T, K = 40, 6, 5
    g_env, e_env = (ready(make_env(kind, "SURVIVAL", n, (32, 32), "int32", textures, monkeypatch, pipe), tasks)
                    for _ in range(2))
    acts = random_actions(torch, kind, np.random.RandomState(2), T, n)
    g_out, e_out = full_out(torch, g_env, T), full_out(torch, e_env, T)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            g_env.rollout(T, actions=acts, out=g_out, final_obs=True)
    torch.cuda.synchronize()
    n_done = 0
    for k in range(K):
        graph.replay()
        e_env.rollout(T, actions=acts, out=e_out, final_obs=True)
        torch.cuda.synchronize()
        n_done += int(e_out["done"].sum())
        for key in ("obs", "rew", "done", "final_obs", "truncated"):
            assert torch.equal(g_out[key], e_out[key]), (k, key)
    assert n_done > 0
    assert_same_state(torch, g_env, e_env)
    g_env.close(); e_env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. sharding
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,pipe", [("D3D", None), ("C3D", "1")])
def test_sharded_handles_equal_one_handle(torch_mod, textures, tasks, monkeypatch, kind, pipe):
    """Two handles over env_index_base halves, drawn actions: the outputs of one handle over all envs."""
    torch = torch_mod
    n, T, res = 40, 30, (32, 32)
    whole = ready(make_env(kind, "SURVIVAL", n, res, "uint8", textures, monkeypatch, pipe), tasks)
    halves = [ready(make_env(kind, "SURVIVAL", n // 2, res, "uint8", textures, monkeypatch, pipe, env_index_base=b), tasks)
              for b in (0, n // 2)]
    ref = full_out(torch, whole, T, drawn=True)
    whole.rollout(T, act_seed=31, out=ref, final_obs=True)
    parts = []
    for h in halves:
        parts.append(full_out(torch, h, T, drawn=True))
        h.rollout(T, act_seed=31, out=parts[-1], final_obs=True)
    for k in ("obs", "rew", "done", "act", "final_obs", "truncated"):
        assert torch.equal(ref[k], torch.cat([p[k] for p in parts], dim=1)), k
    assert int(ref["truncated"].sum()) > 0
    for x, y in zip(state(whole), zip(*(state(h) for h in halves))):
        assert torch.equal(x, torch.cat(y))
    for e in [whole] + halves:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def test_final_obs_rollout_refusals(torch_mod, textures, tasks, monkeypatch):
    """T <= 0, final_obs without auto-reset (truncated alone is fine), either output with mirrors or multicast, and the
    Python ValueError; the rollout works afterwards.  A MetaMaze2D handle runs its own rollout with the outputs, and a
    discrete handle without a pose cache runs on the direct renderer, as its step() would."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D
    n, T, res = 8, 3, (32, 32)
    u8 = torch.zeros((T, n), dtype=torch.uint8, device="cuda")
    envs = {kind: ready(make_env(kind, "SURVIVAL", n, res, "uint8", textures, monkeypatch), tasks)
            for kind in ("D3D", "C3D")}
    m2 = ready(BatchedMetaMaze2D(max_steps=MAX_STEPS, num_envs=n, squeeze=False, auto_reset=True), tasks[:4])
    lib = m2._lib
    fo = torch.zeros((T, n) + res + (3,), dtype=torch.uint8, device="cuda")
    obs = torch.zeros_like(fo)
    rew = torch.zeros((T, n), dtype=torch.float64, device="cuda")
    done = torch.zeros((T, n), dtype=torch.uint8, device="cuda")

    def call(h, steps, f, tr, stream):
        return lib.mgb_maze_rollout(h, steps, None, 0, None, obs.data_ptr(), rew.data_ptr(), done.data_ptr(), _ptr(f),
                                    _ptr(tr), None, 0, stream)

    assert call(m2._h, T, fo, u8, m2._stream()) == 0                  # the 2-D rollout (test_final_obs_rollout_gpu.py)
    torch.cuda.synchronize()
    for env in envs.values():
        h, st = env._h, env._stream()
        for steps in (0, -1):
            assert call(h, steps, fo, u8, st) == MGB_ERR_ARG
            assert b"T must be positive" in lib.mgb_last_error()
        delta = np.array([16], np.int64)
        for arm in (lambda: lib.mgb_maze_set_mirrors(h, 1, delta.ctypes.data),
                    lambda: lib.mgb_maze_set_multicast(h, 16)):
            assert arm() == 0
            for f, tr in ((fo, None), (None, u8)):
                assert call(h, T, f, tr, st) == MGB_ERR_ARG
                assert b"mirrors" in lib.mgb_last_error()
            assert lib.mgb_maze_set_mirrors(h, 0, None) == 0
        out = env.rollout(T, final_obs=True)                  # usable again
        assert "final_obs" in out and "truncated" in out
        torch.cuda.synchronize()
        # final_obs without auto-reset; truncated alone is fine
        assert lib.mgb_maze_set_options(h, 0) == 0
        env.auto_reset = False
        assert call(h, T, fo, None, st) == MGB_ERR_ARG
        assert b"auto_reset" in lib.mgb_last_error()
        assert call(h, T, None, u8, st) == 0
        torch.cuda.synchronize()
        with pytest.raises(ValueError, match="auto_reset"):
            env.rollout(T, final_obs=True)
        assert "truncated" not in env.rollout(T)
        torch.cuda.synchronize()
    # a discrete handle without a pose cache: the direct renderer, equal to step() with final_obs on a twin
    nc = ready(make_env("D3D", "SURVIVAL", n, res, "uint8", textures, monkeypatch, cache=False), tasks)
    twin = ready(make_env("D3D", "SURVIVAL", n, res, "uint8", textures, monkeypatch, cache=False, final_obs=True), tasks)
    acts = random_actions(torch, "D3D", np.random.RandomState(4), T, n)
    assert lib.mgb_maze_rollout(nc._h, T, acts.data_ptr(), 0, None, obs.data_ptr(), rew.data_ptr(), done.data_ptr(),
                                fo.data_ptr(), u8.data_ptr(), None, 0, nc._stream()) == 0
    for t in range(T):
        o, r, d, _ = twin.step(acts[t])
        assert torch.equal(obs[t], o) and torch.equal(rew[t], r) and torch.equal(done[t].bool(), d), t
        assert torch.equal(u8[t].bool(), twin.truncated) and torch.equal(fo[t][d], twin.final_observation[d]), t
    for e in list(envs.values()) + [m2, nc, twin]:
        e.close()
