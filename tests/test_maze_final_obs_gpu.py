"""GPU tests of the terminal observations and truncation flags of auto-reset MetaMaze steps (final_obs=True, the
optional outputs of mgb_maze_step) on every step path, against the CPU oracle (oracle/maze_oracle.c):
the terminal frame of every finished env, the first frame of its next episode, and why the episode ended."""
import numpy as np
import pytest

from util import task_from_arrays

pytestmark = pytest.mark.gpu

MAX_STEPS = 17      # with step_reward = -1/16 and no food eaten, life 1.0 runs out exactly on the last allowed step


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
    """Four 15x15 tasks whose episodes end in all three ways.  SURVIVAL, step_reward -1/16 and initial life 1.0 (tasks 0,
    3: an env that eats nothing dies on step 17, the last allowed one, so that death and time-out coincide) or 2.0 (task 1:
    time-out alive); task 2 loses 0.5 per step from 0.5 and dies on step 2 with life -0.5, whose life-bar end index is
    negative and wraps like a Python slice (maze_discrete_3d.py:118-126).  ESCAPE: the goal of tasks 0 and 2 is an open
    cell next to the start, so random walks reach it; tasks 1 and 3 keep their far goal and time out."""
    g = maze_golden
    out = []
    for k in range(4):
        t = task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                             g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k])
        t = t._replace(step_reward=(-0.0625, -0.0625, -0.5, -0.0625)[k], initial_life=(1.0, 2.0, 0.5, 1.0)[k], max_life=2.0)
        if k % 2 == 0:
            w = np.asarray(t.cell_walls)
            sx, sy = t.start
            near = [(sx + dx, sy + dy) for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1)) if w[sx + dx, sy + dy] == 0]
            t = t._replace(goal=near[0])
        out.append(t)
    return out


# path id -> (kind, obs dtype, resolution, constructor kwargs, environment)
PATHS = {
    "2d": ("2D", "float32", None, {}, {}),
    "fused_u8": ("3D", "uint8", (32, 32), {}, {}),
    "two_kernel_i32": ("3D", "int32", (40, 24), {}, {}),
    "two_kernel_f32": ("3D", "float32", (40, 24), {}, {}),
    "unfused_u8": ("3D", "uint8", (40, 24), {}, {"MGB_MAZE_FUSED_STEP": "0"}),
    "direct_pipe": ("3D", "int32", (40, 24), {"cache": False}, {"MGB_MAZE_RENDER_PIPE": "1"}),
    "direct_seq": ("3D", "uint8", (40, 24), {"cache": False}, {"MGB_MAZE_RENDER_PIPE": "0"}),
    # a screen whose two record sets do not fit in shared memory with their crossing lists: the lists go to global scratch
    "direct_global": ("3D", "uint8", (256, 256), {"cache": False}, {"MGB_MAZE_RENDER_PIPE": "1"}),
    "cont_pipe": ("C3D", "int32", (40, 24), {}, {"MGB_MAZE_RENDER_PIPE": "1"}),
    "cont_seq": ("C3D", "uint8", (40, 24), {}, {"MGB_MAZE_RENDER_PIPE": "0"}),
}


def make_env(path, task_type, n, textures, monkeypatch, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    kind, dtype, res, extra, env = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    kw = dict(dict(max_steps=MAX_STEPS, task_type=task_type, num_envs=n, squeeze=False, auto_reset=True), **kw)
    if kind == "2D":
        return BatchedMetaMaze2D(view_grid=2, **kw)
    cls = BatchedMetaMazeContinuous3D if kind == "C3D" else BatchedMetaMazeDiscrete3D
    return cls(resolution=res, obs_dtype=dtype, textures=textures, **dict(extra, **kw))


def oracle_frame(path, o):
    """The oracle's observation in the path's obs dtype (uint8 = min(value, 255))."""
    v = o._observe()
    dtype = PATHS[path][1]
    if dtype == "uint8":
        return np.minimum(v, 255).astype(np.uint8)
    return v.astype(np.float32) if dtype == "float32" else v


def actions(path, rng, n):
    if PATHS[path][0] == "C3D":
        return rng.uniform(-1.3, 1.3, (n, 2)).astype(np.float32)
    return rng.randint(0, 4, n).astype(np.int32)


def snapshot(env, kind, obs, rew, done):
    """Every primary output of a step and the env state it leaves, on the host."""
    ag, life = env.agent_state()
    out = [obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy(), ag.cpu().numpy(), life.cpu().numpy()]
    if kind == "C3D":
        pos, ori = env.pose()
        out += [pos.cpu().numpy(), ori.cpu().numpy()]
    return out


@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
@pytest.mark.parametrize("path", list(PATHS))
def test_terminal_frames_and_truncation_vs_oracle(torch_mod, textures, tasks, monkeypatch, path, task_type):
    """Many envs over four tasks, random actions, auto-reset: for every env that finishes in every step, final_observation
    is the oracle's step() observation, obs is the oracle's reset(), truncated is the step-limit rule on the oracle's
    state; with the same actions, obs / rew / done / agent state (and pose) equal those of a final_obs=False handle."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    kind = PATHS[path][0]
    if path == "direct_global" and task_type == "ESCAPE":
        pytest.skip("ESCAPE records at most two crossings per column: its lists fit in shared memory")
    if kind == "C3D" and task_type == "ESCAPE":
        # a continuous walk covers a tenth of a cell per step: the goal of tasks 0 and 2 is the start cell itself, so
        # those episodes end on the goal in their first step and the other two time out
        tasks = [t._replace(goal=tuple(t.start)) if k % 2 == 0 else t for k, t in enumerate(tasks)]
    n, T = (64, 60) if kind == "2D" else (24, 40)
    env = make_env(path, task_type, n, textures, monkeypatch, final_obs=True)
    ref = make_env(path, task_type, n, textures, monkeypatch)
    assert ref.final_observation is None and ref.truncated is None
    for e in (env, ref):
        e.set_task(tasks)
        e.reset()
    res = PATHS[path][2] or (8, 8)
    oracles = []
    for e in range(n):
        o = OracleMaze(kind, task_type, MAX_STEPS, 2, res, textures=textures if kind != "2D" else None)
        o.set_task(tasks[e % 4])
        o.reset()
        oracles.append(o)
    rng = np.random.RandomState(11)
    deaths = timeouts = goals = death_at_limit = 0
    prev = env.final_observation.cpu().numpy()
    for t in range(T):
        act = actions(path, rng, n)
        a_dev = torch.as_tensor(act).cuda()
        got = snapshot(env, kind, *env.step(a_dev)[:3])
        want = snapshot(ref, kind, *ref.step(a_dev)[:3])
        for x, y in zip(got, want):
            assert np.array_equal(x, y), (path, t)
        obs, done = got[0], got[2]
        fin = env.final_observation.cpu().numpy()
        trunc = env.truncated.cpu().numpy()
        assert trunc.dtype == np.bool_
        for e in range(n):
            o = oracles[e]
            _, _, d, _ = o.step(act[e], render=False)
            assert bool(done[e]) == d, (t, e)
            if not d:
                assert not trunc[e], (t, e)
                assert np.array_equal(fin[e], prev[e]), (t, e)       # rows of envs that did not finish stay untouched
                continue
            over = o.env.steps > MAX_STEPS - 1
            if task_type == "SURVIVAL":
                ended = o.life < 0
            else:
                ended = (o.env.gx, o.env.gy) == tuple(tasks[e % 4].goal)
            assert bool(trunc[e]) == (over and not ended), (t, e, over, ended)
            deaths += ended and task_type == "SURVIVAL"
            goals += ended and task_type == "ESCAPE"
            timeouts += over and not ended
            death_at_limit += ended and over
            assert np.array_equal(fin[e], oracle_frame(path, o)), (t, e)
            o.reset()
            assert np.array_equal(obs[e], oracle_frame(path, o)), (t, e)
        prev = fin
    if path == "direct_global":
        assert env.cache_info()["hits_in_global"]
    assert timeouts > 0
    if task_type == "SURVIVAL":
        assert deaths > 0 and death_at_limit > 0
    else:
        assert goals > 0
    env.close()
    ref.close()


@pytest.mark.parametrize("path", ["2d", "fused_u8", "two_kernel_i32", "direct_pipe", "cont_seq"])
def test_graph_replay_equals_eager_steps(torch_mod, textures, tasks, monkeypatch, path):
    """step() with final_obs=True captured in a CUDA graph right after reset() (no step before it) and replayed K times
    equals K eager steps."""
    torch = torch_mod
    n, K = 40, 24
    g_env = make_env(path, "SURVIVAL", n, textures, monkeypatch, final_obs=True)
    e_env = make_env(path, "SURVIVAL", n, textures, monkeypatch, final_obs=True)
    for e in (g_env, e_env):
        e.set_task(tasks)
        e.reset()
    rng = np.random.RandomState(3)
    act = torch.as_tensor(actions(path, rng, n)).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            g_env.step(act)
    torch.cuda.synchronize()
    n_done = 0
    for k in range(K):
        graph.replay()
        obs, rew, done, _ = e_env.step(act)
        torch.cuda.synchronize()
        n_done += int(done.sum())
        assert torch.equal(g_env._obs, e_env._obs) and torch.equal(g_env._done, e_env._done), k
        assert torch.equal(g_env.final_observation, e_env.final_observation), k
        assert torch.equal(g_env.truncated, e_env.truncated), k
    assert n_done > 0
    g_env.close()
    e_env.close()


def test_task_churn_keeps_the_old_task_terminal_frames(torch_mod, textures, tasks, monkeypatch):
    """update_tasks between steps (direct renderer, one task slot per env): the terminal frames are the old task's, the
    next observation is the new task's first frame."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    n, T, path = 12, 30, "direct_pipe"
    env = make_env(path, "SURVIVAL", n, textures, monkeypatch, final_obs=True)
    env.set_task([tasks[e % 4] for e in range(n)], env2task=np.arange(n))
    env.reset()
    res = PATHS[path][2]
    oracles = []
    for e in range(n):
        o = OracleMaze("3D", "SURVIVAL", MAX_STEPS, 2, res, textures=textures)
        o.set_task(tasks[e % 4])
        o.reset()
        oracles.append(o)
    rng = np.random.RandomState(5)
    churned = seen_new = 0
    fresh = np.zeros(n, dtype=bool)          # re-tasked in the step before
    for t in range(T):
        act = rng.randint(0, 4, n).astype(np.int32)
        obs, _, done, _ = env.step(torch.as_tensor(act).cuda())
        obs, done = obs.cpu().numpy(), done.cpu().numpy()
        ids = np.nonzero(done)[0]
        new = [tasks[(int(e) + 1 + t) % 4] for e in ids]
        if len(ids):
            env.update_tasks(ids, new)
        fin = env.final_observation.cpu().numpy()
        for e in range(n):
            _, _, d, _ = oracles[e].step(int(act[e]), render=False)
            assert bool(done[e]) == d, (t, e)
            if d:          # the terminal frame of the old task, still there after update_tasks
                assert np.array_equal(fin[e], oracle_frame(path, oracles[e])), (t, e)
            else:          # includes the first step on a new task
                assert np.array_equal(obs[e], oracle_frame(path, oracles[e])), (t, e)
                seen_new += fresh[e]
        fresh[:] = False
        for e, tk in zip(ids, new):
            oracles[e].set_task(tk)
            oracles[e].reset()
            fresh[e] = True
            churned += 1
    assert churned > 0 and seen_new > 0
    env.close()


@pytest.mark.parametrize("path", ["2d", "fused_u8", "direct_seq"])
def test_sharded_handles_equal_one_handle(torch_mod, textures, tasks, monkeypatch, path):
    """Two handles over env_index_base halves give the final_observation / truncated of one handle."""
    torch = torch_mod
    n, T = 32, 30
    whole = make_env(path, "SURVIVAL", n, textures, monkeypatch, final_obs=True)
    halves = [make_env(path, "SURVIVAL", n // 2, textures, monkeypatch, final_obs=True, env_index_base=b)
              for b in (0, n // 2)]
    for e in [whole] + halves:
        e.set_task(tasks)
        e.reset()
    rng = np.random.RandomState(9)
    n_trunc = 0
    for t in range(T):
        act = torch.as_tensor(actions(path, rng, n)).cuda()
        whole.step(act)
        halves[0].step(act[:n // 2].contiguous())
        halves[1].step(act[n // 2:].contiguous())
        assert torch.equal(whole.final_observation, torch.cat([h.final_observation for h in halves])), t
        assert torch.equal(whole.truncated, torch.cat([h.truncated for h in halves])), t
        n_trunc += int(whole.truncated.sum())
    assert n_trunc > 0
    for e in [whole] + halves:
        e.close()


def test_final_obs_step_refusals(torch_mod, textures, tasks, monkeypatch):
    """final_obs needs auto_reset, in Python (ValueError) and in the C ABI (MGB_ERR_ARG)."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    with pytest.raises(ValueError, match="auto_reset"):
        BatchedMetaMaze2D(num_envs=2, final_obs=True)
    with pytest.raises(ValueError, match="auto_reset"):
        BatchedMetaMazeDiscrete3D(num_envs=2, resolution=(32, 32), final_obs=True, auto_reset=False)
    with pytest.raises(ValueError, match="auto_reset"):
        BatchedMetaMazeContinuous3D(num_envs=2, resolution=(32, 32), final_obs=True)
    for path in ("2d", "fused_u8", "cont_seq"):
        env = make_env(path, "SURVIVAL", 2, textures, monkeypatch, auto_reset=False)
        env.set_task(tasks)
        env.reset()
        final = torch.zeros_like(env._obs)
        trunc = torch.zeros(2, dtype=torch.uint8, device="cuda")
        if PATHS[path][0] == "C3D":
            act = torch.zeros((2, 2), dtype=torch.float32, device="cuda")
        else:
            act = torch.zeros(2, dtype=torch.int32, device="cuda")
        fn = env._lib.mgb_maze_step
        args = (env._h, act.data_ptr(), env._obs.data_ptr(), env._rew.data_ptr(), env._done.data_ptr())
        assert fn(*args, final.data_ptr(), trunc.data_ptr(), env._stream()) == -1       # MGB_ERR_ARG
        assert b"auto_reset" in env._lib.mgb_last_error()
        assert fn(*args, None, trunc.data_ptr(), env._stream()) == 0                    # truncated alone is fine
        torch.cuda.synchronize()
        env.close()
