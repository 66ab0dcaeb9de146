"""GPU tests of mgb_maze_rollout on the direct raycaster: T steps of a MetaMazeDiscrete3D or MetaMazeContinuous3D handle
in one launch of maze3d_kernel<false, true, FIN, RS>, optionally giving every finished env a freshly drawn maze in
the same launch (rollout(T, resample=...)).

Against T step() calls of a cache=False twin, against the pose-cache rollout of a cached twin, against the loop
step + resample_tasks(done) + reset(mask=done) that returns the frame on the new maze, against the CPU oracle fed the
restated tasks (tests/maze_sampler_draws.py), refusals, and CUDA-graph capture."""
import ctypes

import numpy as np
import pytest

from maze_sampler_draws import restated_tasks, same_task
from util import task_from_arrays

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
BASE_HI = 2 ** 32 - 70                   # env_index_base: the batch straddles genv = 2^32
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
    """Four 15x15 golden tasks with step_reward -1/8 and a near goal in two of them, so that SURVIVAL envs die and time
    out and ESCAPE envs reach the goal and time out within a few dozen steps."""
    g = maze_golden
    out = []
    for k in range(4):
        t = task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                             g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k])
        t = t._replace(step_reward=-0.125, initial_life=(1.0, 2.0, 1.0, 1.5)[k], max_life=2.0)
        w = np.array(t.cell_walls)
        sx, sy = t.start
        near = [c for c in ((sx + 1, sy), (sx - 1, sy), (sx, sy + 1), (sx, sy - 1)) if w[c] == 0]
        if k in (0, 2):
            t = t._replace(goal=near[0])
        out.append(t)
    return out


def make_env(kind, n, res, dtype, textures, monkeypatch, pipe=None, **kw):
    from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    if pipe is not None:
        monkeypatch.setenv("MGB_MAZE_RENDER_PIPE", pipe)       # read when the handle is created
    else:
        monkeypatch.delenv("MGB_MAZE_RENDER_PIPE", raising=False)
    cls = BatchedMetaMazeContinuous3D if kind == "C3D" else BatchedMetaMazeDiscrete3D
    kw = dict(dict(num_envs=n, squeeze=False), **kw)
    return cls(resolution=res, obs_dtype=dtype, textures=textures, **kw)


def out_dict(torch, env, T, final=True, drawn=False):
    """A caller's out dict; final_obs pre-filled with a sentinel (rows with done = 0 must keep it)."""
    n, shape, dt = env.num_envs, tuple(env._obs.shape[1:]), env._obs.dtype
    out = {"obs": torch.empty((T, n) + shape, dtype=dt, device="cuda"),
           "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
           "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"),
           "act": None}
    if drawn:
        out["act"] = torch.empty((T, n, 2) if env.KIND == 2 else (T, n), device="cuda",
                                 dtype=torch.float32 if env.KIND == 2 else torch.int32)
    if final:
        out["final_obs"] = torch.full((T, n) + shape, SENTINEL[env.obs_dtype], dtype=dt, device="cuda")
        out["truncated"] = torch.full((T, n), 9, dtype=torch.uint8, device="cuda")
    return out


def actions(torch, kind, rng, T, n):
    if kind == "C3D":
        return torch.as_tensor(rng.uniform(-1.3, 1.3, (T, n, 2)).astype(np.float32)).cuda()
    return torch.as_tensor(rng.randint(0, 4, (T, n)).astype(np.int32)).cuda()


def t_base(env):
    v = ctypes.c_uint64()
    assert env._lib.mgb_maze_counters(env._h, ctypes.byref(v), 0) == 0
    return v.value


def assert_same_state(torch, a, b):
    for x, y in zip(a.agent_state(), b.agent_state()):
        assert torch.equal(x, y)
    if a.KIND == 2:
        for x, y in zip(a.pose(), b.pose()):
            assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------------------------
# 1. discrete direct rollout = T step() calls of a cache=False twin
# ---------------------------------------------------------------------------------------------------------------------
# dtype, task type, drawn actions, auto-reset, screen, envs, MGB_MAZE_RENDER_PIPE
DISC = [("uint8", "SURVIVAL", False, True, (32, 32), 24, None),
        ("int32", "ESCAPE", True, True, (40, 24), 200, None),
        ("float32", "SURVIVAL", True, False, (32, 32), 24, None),
        ("uint8", "ESCAPE", False, False, (40, 24), 150, "0"),
        ("int32", "SURVIVAL", True, True, (32, 32), 150, "0"),
        ("uint8", "SURVIVAL", False, True, (256, 256), 20, None)]   # two record sets do not fit: lists in global scratch


@pytest.mark.parametrize("dtype,task_type,drawn,auto,res,n,pipe", DISC)
def test_discrete_direct_rollout_equals_single_steps(torch_mod, textures, tasks, monkeypatch, dtype, task_type, drawn,
                                                     auto, res, n, pipe):
    """rollout() of a cache=False MetaMazeDiscrete3D env against T step() calls of a cache=False twin, bit for bit: obs,
    rew, done, final_obs where done (the sentinel elsewhere), truncated, agent state, life and the recorded paths."""
    torch = torch_mod
    kw = dict(max_steps=13, task_type=task_type, auto_reset=auto, cache=False, record_path=True)
    roll = make_env("D3D", n, res, dtype, textures, monkeypatch, pipe, **kw)
    twin = make_env("D3D", n, res, dtype, textures, monkeypatch, pipe, final_obs=auto, **kw)
    for e in (roll, twin):
        e.set_task(tasks)
        e.reset()
    T = 30
    acts = None if drawn else actions(torch, "D3D", np.random.RandomState(n + res[0]), T, n)
    out = out_dict(torch, roll, T, final=auto, drawn=drawn)
    roll.rollout(T, actions=acts, act_seed=17, out=out, final_obs=auto)
    if drawn:
        acts = out["act"]
    n_done = 0
    for t in range(T):
        o, r, d, _ = twin.step(acts[t])
        assert torch.equal(out["obs"][t], o), (t, int((out["obs"][t] != o).sum()))
        assert torch.equal(out["rew"][t], r) and torch.equal(out["done"][t].bool(), d), t
        if auto:
            assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
            assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
            assert (out["final_obs"][t][~d] == SENTINEL[dtype]).all(), t
        n_done += int(d.sum())
    assert n_done > 0
    assert_same_state(torch, roll, twin)
    for x, y in zip(roll.trajectory(), twin.trajectory()):
        assert torch.equal(x, y)
    if res == (256, 256):
        assert roll.cache_info()["hits_in_global"] or not roll.cache_info()["pipelined"]
    roll.close(); twin.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. discrete direct rollout = the pose-cache rollout
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype,task_type", [("uint8", "SURVIVAL"), ("int32", "ESCAPE")])
def test_discrete_direct_rollout_equals_pose_cache_rollout(torch_mod, textures, tasks, monkeypatch, dtype, task_type):
    """Drawn actions, two consecutive rollouts: the cache=False handle (direct renderer) and a cached twin (pose cache)
    give the same act_out, obs, rew, done, final_obs, truncated, state and step counter."""
    torch = torch_mod
    n, res = 40, (32, 32)
    kw = dict(max_steps=11, task_type=task_type, auto_reset=True, env_index_base=BASE_HI)
    direct = make_env("D3D", n, res, dtype, textures, monkeypatch, cache=False, **kw)
    cached = make_env("D3D", n, res, dtype, textures, monkeypatch, cache=True, **kw)
    for e in (direct, cached):
        e.set_task(tasks)
        e.reset()
    assert cached.cache_info()["in_use"]
    for T, seed in ((20, 5), (9, 5)):
        a, b = out_dict(torch, direct, T, drawn=True), out_dict(torch, cached, T, drawn=True)
        direct.rollout(T, act_seed=seed, out=a, final_obs=True)
        cached.rollout(T, act_seed=seed, out=b, final_obs=True)
        for k in ("act", "obs", "rew", "done", "final_obs", "truncated"):
            assert torch.equal(a[k], b[k]), (T, k)
        assert int(a["done"].sum()) > 0
        assert t_base(direct) == t_base(cached)
    assert t_base(direct) == 29
    assert_same_state(torch, direct, cached)
    direct.close(); cached.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. the resampling rollout = step + resample_tasks(done) + reset(mask=done)
# ---------------------------------------------------------------------------------------------------------------------
def slot_table(n, N, food_cells=40):
    """N open-interior tasks, one table slot per env; task 0 has `food_cells` food cells (the table's food cap)."""
    from metagym_b200 import TaskConfig
    walls = np.ones((n, n), dtype=np.int32)
    walls[1:-1, 1:-1] = 0
    texts = np.where(walls > 0, 1, 0)
    base = TaskConfig(start=(1, 1), goal=(n - 2, n - 2), cell_walls=walls, cell_texts=texts, cell_size=2.0,
                      wall_height=3.2, agent_height=1.6, initial_life=1.0, max_life=2.0, step_reward=-0.2,
                      goal_reward=1.0, food_rewards=np.zeros((n, n)), food_interval=np.zeros((n, n), dtype=np.int32))
    food = np.zeros(n * n)
    fc = min(food_cells, (n - 2) ** 2 - 1)
    food[np.nonzero(walls.ravel() == 0)[0][1:1 + fc]] = 0.3
    first = base._replace(food_rewards=food.reshape(n, n), food_interval=np.where(food > 0, 5, 0).reshape(n, n))
    return [first] + [base] * (N - 1), fc


CFG = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.08, food_interval=3, cell_size=2.5, agent_height=1.2,
           wall_height=2.8, step_reward=-0.25, initial_life=1.0, max_life=1.5)

# kind, task type, n, env_index_base, MGB_MAZE_RENDER_PIPE, final_obs, drawn actions
RESAMPLE = [("D3D", "SURVIVAL", 9, BASE_HI, None, True, False),
            ("D3D", "ESCAPE", 15, 1000, None, True, True),
            ("D3D", "SURVIVAL", 15, 7, "0", True, False),
            ("D3D", "ESCAPE", 9, BASE_HI, "0", False, True),
            ("C3D", "SURVIVAL", 15, BASE_HI, None, True, False),
            ("C3D", "ESCAPE", 9, 1000, None, False, True),
            ("C3D", "SURVIVAL", 9, 7, "0", True, True),
            ("C3D", "ESCAPE", 15, BASE_HI, "0", True, False)]


@pytest.mark.parametrize("kind,task_type,n,base,pipe,final,drawn", RESAMPLE)
def test_resampling_rollout_equals_the_correct_frame_loop(torch_mod, textures, monkeypatch, kind, task_type, n, base,
                                                          pipe, final, drawn):
    """rollout(32, resample=dict(seed, **CFG)) against a twin that runs, per step, step(act[t]),
    resample_tasks(done, seed, **CFG) and obs_t = reset(mask=done): obs, rew, done, final_obs where done, truncated per
    step; afterwards the snapshot records byte for byte (agent, life, resample count, slot, food stamps, task), the
    continuous pose, and every re-tasked slot against restated_tasks at the env's resample count.  max_steps = 5: every
    env finishes several times."""
    torch = torch_mod
    N, T, seed, res = 150, 32, (0xfeed << 32) | 21, (24, 16)
    table, fc = slot_table(n, N)
    kw = dict(max_steps=5, task_type=task_type, auto_reset=True, env_index_base=base)
    if kind == "D3D":
        kw["cache"] = False
    roll = make_env(kind, N, res, "int32", textures, monkeypatch, pipe, **kw)
    twin = make_env(kind, N, res, "int32", textures, monkeypatch, pipe, final_obs=True, **kw)
    for e in (roll, twin):
        e.set_task(table, env2task=np.arange(N))
        e.reset()
    acts = None if drawn else actions(torch, kind, np.random.RandomState(n), T, N)
    out = out_dict(torch, roll, T, final=final, drawn=drawn)
    roll.rollout(T, actions=acts, act_seed=3, out=out, final_obs=final, resample=dict(seed=seed, **CFG))
    if drawn:
        acts = out["act"]
    count = np.zeros(N, np.int64)
    for t in range(T):
        _, r, d, _ = twin.step(acts[t])
        assert torch.equal(out["rew"][t], r) and torch.equal(out["done"][t].bool(), d), t
        if final:
            assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
            assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
            assert (out["final_obs"][t][~d] == SENTINEL["int32"]).all(), t
        twin.resample_tasks(d, seed=seed, **CFG)
        o = twin.reset(mask=d)
        assert torch.equal(out["obs"][t], o), (t, int((out["obs"][t] != o).sum()))
        count += d.cpu().numpy()
    assert count.min() >= 3, count.min()
    assert torch.equal(roll.snapshot()["records"], twin.snapshot()["records"])
    assert_same_state(torch, roll, twin)
    want = restated_tasks(seed, np.arange(N) + base, count, n, fc, **CFG)
    got = roll.get_tasks(np.arange(N))
    bad = [e for e in range(N) if not same_task(got[e], want[e])]
    assert not bad, bad[:5]
    assert (roll.snapshot()["records"].view(torch.int32)[:, 6].cpu().numpy() == count).all()
    roll.close(); twin.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. frames on the resampled tasks = the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["D3D", "C3D"])
@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
def test_frames_on_resampled_tasks_equal_the_oracle(torch_mod, textures, kind, task_type, monkeypatch):
    """A few envs, one resampling rollout with terminal frames: every obs, final_obs, reward and done equals an
    OracleMaze that is given the restated task whenever its episode ends (heights the table does not have: the
    renderer's per-pixel path)."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    N, n, seed, res, max_steps, T = 6, 9, 41, (24, 16), 7, 24
    table, fc = slot_table(n, N)
    kw = dict(max_steps=max_steps, task_type=task_type, auto_reset=True)
    if kind == "D3D":
        kw["cache"] = False
    env = make_env(kind, N, res, "int32", textures, monkeypatch, **kw)
    env.set_task(table, env2task=np.arange(N))
    env.reset()
    oras = [OracleMaze("3D" if kind == "D3D" else "C3D", task_type, max_steps, 1, res, textures=textures) for _ in range(N)]
    for o, t in zip(oras, table):
        o.set_task(t)
        o.reset()
    rng = np.random.RandomState(6)
    acts = torch.as_tensor(rng.randint(0, 4, (T, N)).astype(np.int32) if kind == "D3D" else
                           rng.uniform(-1, 1, (T, N, 2)).astype(np.float32)).cuda()
    out = env.rollout(T, actions=acts, final_obs=True, resample=dict(seed=seed, **CFG))
    obs, fin = out["obs"].cpu().numpy(), out["final_obs"].cpu().numpy()
    rew, done = out["rew"].cpu().numpy(), out["done"].cpu().numpy().astype(bool)
    a_h = acts.cpu().numpy()
    count = np.zeros(N, np.int64)
    for t in range(T):
        for e, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(a_h[t, e]) if kind == "D3D" else a_h[t, e])
            assert rew[t, e] == r2 and done[t, e] == d2, (t, e)
            if d2:
                assert np.array_equal(fin[t, e], o2), (t, e)
                count[e] += 1
                o.set_task(restated_tasks(seed, np.array([e]), np.array([count[e]]), n, fc, **CFG)[0])
                o2 = o.reset()
            assert np.array_equal(obs[t, e], o2), (t, e, int((obs[t, e] != o2).sum()))
    assert count.min() >= 2
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def test_direct_rollout_refusals_leave_the_handle_untouched(torch_mod, textures, tasks, monkeypatch):
    """Each refusal of mgb_maze_rollout on the direct renderer returns MGB_ERR_ARG with its message (the sampler-cfg
    ones with the text mgb_maze_resample_tasks gives for the same cfg) and leaves snapshot() as it was; a MetaMaze2D
    handle runs its own rollout; rollout(resample=dict(goal_reward=-1)) raises ValueError."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, _lib
    n, T, res, N9 = 8, 3, (24, 16), 9
    table, _ = slot_table(N9, n)
    u8 = torch.zeros((T, n), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((T, n) + res + (3,), dtype=torch.int32, device="cuda")
    obs = torch.zeros_like(fo)
    rew = torch.zeros((T, n), dtype=torch.float64, device="cuda")
    done = torch.zeros((T, n), dtype=torch.uint8, device="cuda")
    lib = _lib.load()

    def cfg(**over):
        return BatchedMetaMaze2D._sampler_cfg(**dict(dict(seed=3), **over))[0]

    def call(env, steps=T, f=None, tr=None, c=None):
        return lib.mgb_maze_rollout(env._h, steps, None, 0, None, obs.data_ptr(), rew.data_ptr(), done.data_ptr(),
                                    _ptr(f), _ptr(tr), None if c is None else ctypes.byref(c), 9, env._stream())

    def refused(env, text, **kw):
        before = env.snapshot()["records"].clone()
        assert call(env, **kw) == MGB_ERR_ARG
        msg = lib.mgb_last_error().decode()
        assert msg.startswith("mgb_maze_rollout: ") and text in msg, msg
        assert torch.equal(env.snapshot()["records"], before)
        return msg[len("mgb_maze_rollout: "):]

    def mk(kind, **kw):
        e = make_env(kind, n, res, "int32", textures, monkeypatch, **dict(dict(max_steps=9, auto_reset=True), **kw))
        e.set_task(table, env2task=np.arange(n))
        e.reset()
        return e

    m2 = BatchedMetaMaze2D(max_steps=9, num_envs=n, squeeze=False, auto_reset=True)
    m2.set_task(table, env2task=np.arange(n))
    m2.reset()
    assert call(m2) == 0                                                   # the 2-D rollout
    torch.cuda.synchronize()
    envs = [mk("D3D", cache=False), mk("C3D")]
    for env in envs:
        for steps in (0, -1):
            refused(env, "T must be positive", steps=steps)
        for k in range(3):                                                 # obs, rew or done missing
            ptrs = [obs.data_ptr(), rew.data_ptr(), done.data_ptr()]
            ptrs[k] = None
            before = env.snapshot()["records"].clone()
            rc = lib.mgb_maze_rollout(env._h, T, None, 0, None, *ptrs, None, None, None, 0, env._stream())
            assert rc == MGB_ERR_ARG
            assert lib.mgb_last_error().decode() == "mgb_maze_rollout: null argument"
            assert torch.equal(env.snapshot()["records"], before)
        delta = np.array([16], np.int64)
        for arm in (lambda: lib.mgb_maze_set_mirrors(env._h, 1, delta.ctypes.data),
                    lambda: lib.mgb_maze_set_multicast(env._h, 16)):
            assert arm() == 0
            refused(env, "mirrors")
            refused(env, "mirrors", c=cfg())
            assert lib.mgb_maze_set_mirrors(env._h, 0, None) == 0
        # the sampler-cfg checks: the message of mgb_maze_resample_tasks
        for bad in (dict(step_reward=0.0), dict(agent_height=3.5), dict(cell_size=1.0), dict(n_texts=1),
                    dict(n_texts=99), dict(food_reward=0.0), dict(crowd_ratio=-1.0)):
            text = refused(env, "", c=cfg(**bad))
            assert env._lib.mgb_maze_resample_tasks(env._h, None, ctypes.byref(cfg(**bad)), 3, env._stream()) == MGB_ERR_ARG
            assert lib.mgb_last_error().decode() == "mgb_maze_resample_tasks: " + text
        with pytest.raises(ValueError, match="goal reward"):
            env.rollout(T, resample=dict(seed=1, goal_reward=-1.0))
        assert call(env, f=fo, tr=u8, c=cfg()) == 0                       # usable again
        torch.cuda.synchronize()
        # final_obs without auto-reset; resampling without auto-reset
        assert lib.mgb_maze_set_options(env._h, 0) == 0
        refused(env, "auto_reset", f=fo)
        refused(env, "auto_reset", c=cfg())
        assert call(env, tr=u8) == 0
        torch.cuda.synchronize()
        assert lib.mgb_maze_set_options(env._h, 1) == 0
    # no slot per env: a shared table
    shared = make_env("D3D", n, res, "int32", textures, monkeypatch, max_steps=9, auto_reset=True, cache=False)
    shared.set_task(tasks)
    shared.reset()
    refused(shared, "one task-table slot per env", c=cfg())
    assert call(shared) == 0                                               # without resampling it runs
    # a discrete handle whose pose cache is in use refuses resampling, runs without it
    cached = mk("D3D", cache=True)
    assert cached.cache_info()["in_use"]
    refused(cached, "the direct renderer", c=cfg())
    assert call(cached, f=fo, tr=u8) == 0
    torch.cuda.synchronize()
    # a cache-less discrete handle without a cfg runs on the direct renderer: one launch, step counter + T
    nc = envs[0]
    launches, t0 = nc.launch_count, t_base(nc)
    assert call(nc, f=fo, tr=u8) == 0
    torch.cuda.synchronize()
    assert nc.launch_count == launches + 1 and t_base(nc) == t0 + T
    for e in envs + [m2, shared, cached]:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. CUDA-graph capture
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,pipe", [("D3D", None), ("C3D", "0")])
def test_graph_replay_equals_eager_resampling_rollouts(torch_mod, textures, monkeypatch, kind, pipe):
    """rollout(T, resample=..., final_obs=True, out=...) captured in a CUDA graph right after reset() and replayed K
    times equals K eager calls on a twin: every output of every replay, then the snapshot records."""
    torch = torch_mod
    N, n, T, K, res = 64, 9, 6, 4, (24, 16)
    table, _ = slot_table(n, N)
    kw = dict(max_steps=4, task_type="SURVIVAL", auto_reset=True)
    if kind == "D3D":
        kw["cache"] = False
    g_env, e_env = (make_env(kind, N, res, "uint8", textures, monkeypatch, pipe, **kw) for _ in range(2))
    for e in (g_env, e_env):
        e.set_task(table, env2task=np.arange(N))
        e.reset()
    acts = actions(torch, kind, np.random.RandomState(2), T, N)
    g_out, e_out = out_dict(torch, g_env, T), out_dict(torch, e_env, T)
    rs = dict(seed=12, **CFG)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            g_env.rollout(T, actions=acts, out=g_out, final_obs=True, resample=rs)
    torch.cuda.synchronize()
    n_done = 0
    for k in range(K):
        graph.replay()
        e_env.rollout(T, actions=acts, out=e_out, final_obs=True, resample=rs)
        torch.cuda.synchronize()
        n_done += int(e_out["done"].sum())
        for key in ("obs", "rew", "done", "final_obs", "truncated"):
            assert torch.equal(g_out[key], e_out[key]), (k, key)
    assert n_done > 0
    assert torch.equal(g_env.snapshot()["records"], e_env.snapshot()["records"])
    assert_same_state(torch, g_env, e_env)
    g_env.close(); e_env.close()
