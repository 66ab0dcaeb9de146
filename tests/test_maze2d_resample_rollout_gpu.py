"""GPU tests of mgb_maze_rollout with a sampler cfg: T MetaMaze2D steps in one launch of
maze2d_rollout_kernel<0, FIN, REC, RS> that give every finished env a freshly drawn maze in the same launch (BatchedMetaMaze2D.rollout(T, resample=...)).

Against the loop step + resample_tasks(done) + reset(mask=done) that returns the window on the new maze, against the CPU
oracle fed the restated tasks (tests/maze_sampler_draws.py), across calls and a snapshot restore, refusals, and CUDA-graph
capture."""
import ctypes

import numpy as np
import pytest

from maze_sampler_draws import restated_tasks, same_task

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
BASE_HI = 2 ** 32 - 70                   # env_index_base: the batch straddles genv = 2^32
SEED_HI = (0xfeed << 32) | 21            # a seed with both 32-bit halves set
SENTINEL = -7.0

CFG = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.08, food_interval=3, cell_size=2.5, agent_height=1.2,
           wall_height=2.8, step_reward=-0.25, initial_life=1.0, max_life=1.5)


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


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


def make_env(N, n, table, **kw):
    from metagym_b200 import BatchedMetaMaze2D
    env = BatchedMetaMaze2D(**dict(dict(num_envs=N, squeeze=False, auto_reset=True), **kw))
    env.set_task(table, env2task=np.arange(N))
    env.reset()
    return env


def out_dict(torch, env, T, final=True, drawn=False):
    """A caller's out dict; final_obs pre-filled with a sentinel (rows with done = 0 must keep it)."""
    n, shape = env.num_envs, tuple(env._obs.shape[1:])
    out = {"obs": torch.empty((T, n) + shape, dtype=torch.float32, device="cuda"),
           "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
           "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"),
           "act": torch.empty((T, n), dtype=torch.int32, device="cuda") if drawn else None}
    if final:
        out["final_obs"] = torch.full((T, n) + shape, SENTINEL, dtype=torch.float32, device="cuda")
        out["truncated"] = torch.full((T, n), 9, dtype=torch.uint8, device="cuda")
    return out


def run_twin(torch, twin, out, acts, seed, final):
    """The correct-frame loop step(act[t]) + resample_tasks(done) + reset(mask=done) on `twin` for the T steps of `out`,
    compared step by step with the rollout's outputs -> done counts per env."""
    N = twin.num_envs
    count = np.zeros(N, np.int64)
    for t in range(out["obs"].shape[0]):
        _, r, d, _ = twin.step(acts[t])
        assert torch.equal(out["rew"][t], r) and torch.equal(out["done"][t].bool(), d), t
        if final:
            assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
            assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
            assert (out["final_obs"][t][~d] == SENTINEL).all(), t
        twin.resample_tasks(d, seed=seed, **CFG)
        o = twin.reset(mask=d)
        assert torch.equal(out["obs"][t], o), (t, int((out["obs"][t] != o).sum()))
        count += d.cpu().numpy()
    return count


def records(env):
    """snapshot() records written into zeroed memory: the padding behind the path entries is not written."""
    snap = env.snapshot()
    snap["records"].zero_()
    return env.snapshot(out=snap)["records"]


def assert_same_envs(torch, a, b, record):
    assert torch.equal(records(a), records(b))
    for x, y in zip(a.agent_state(), b.agent_state()):
        assert torch.equal(x, y)
    if record:
        for x, y in zip(a.trajectory(), b.trajectory()):
            assert torch.equal(x, y)


def assert_restated(env, seed, base, count, n, fc):
    N = env.num_envs
    want = restated_tasks(seed, np.arange(N) + base, count, n, fc, **CFG)
    got = env.get_tasks(np.arange(N))
    bad = [e for e in range(N) if not same_task(got[e], want[e])]
    assert not bad, bad[:5]
    assert (records(env).view(env._torch.int32)[:, 6].cpu().numpy() == count).all()


# ---------------------------------------------------------------------------------------------------------------------
# 1. the resampling rollout = step + resample_tasks(done) + reset(mask=done)
# ---------------------------------------------------------------------------------------------------------------------
# task type, n, view_grid, drawn actions, final_obs, record_path, (env_index_base, seed), envs: every pair of values of
# any two parameters occurs.  N = 150 and 1027 leave the tail warp with inactive lanes.
LO, HI = (7, 5), (BASE_HI, SEED_HI)
RESAMPLE = [("SURVIVAL", 7, 1, False, False, False, LO, 150),
            ("ESCAPE", 7, 2, False, True, True, HI, 1027),
            ("SURVIVAL", 7, 5, True, True, True, LO, 1027),
            ("ESCAPE", 15, 1, True, False, True, LO, 1027),
            ("SURVIVAL", 15, 2, True, True, False, HI, 150),
            ("ESCAPE", 15, 5, False, False, False, HI, 1027),
            ("ESCAPE", 31, 1, True, True, False, HI, 150),
            ("SURVIVAL", 31, 2, False, False, True, HI, 1027),
            ("ESCAPE", 31, 5, False, True, True, LO, 150)]


@pytest.mark.parametrize("task_type,n,view_grid,drawn,final,record,base_seed,N", RESAMPLE)
def test_resampling_rollout_equals_the_correct_frame_loop(torch_mod, task_type, n, view_grid, drawn, final, record,
                                                          base_seed, N):
    """rollout(32, resample=dict(seed, **CFG)) against a twin that runs, per step, step(act[t]),
    resample_tasks(done, seed, **CFG) and obs_t = reset(mask=done): obs, rew, done and, with final_obs, truncated and
    final_obs where done (the sentinel elsewhere).  Afterwards the snapshot records byte for byte, the agent state, the
    recorded paths, and every slot against restated_tasks at the env's resample count.  max_steps = 5: every env finishes
    at least three times; in ESCAPE whole warps time out together in one step."""
    torch = torch_mod
    T = 32
    base, seed = base_seed
    table, fc = slot_table(n, N)
    kw = dict(max_steps=5, task_type=task_type, view_grid=view_grid, env_index_base=base, record_path=record)
    roll = make_env(N, n, table, final_obs=final, **kw)
    twin = make_env(N, n, table, final_obs=True, **kw)
    acts = None if drawn else torch.as_tensor(np.random.RandomState(n + N).randint(0, 4, (T, N)).astype(np.int32)).cuda()
    out = out_dict(torch, roll, T, final=final, drawn=drawn)
    launches = roll.launch_count
    roll.rollout(T, actions=acts, act_seed=3, out=out, resample=dict(seed=seed, **CFG))
    assert roll.launch_count == launches + 1
    if drawn:
        acts = out["act"]
    count = run_twin(torch, twin, out, acts, seed, final)
    assert count.min() >= 3, count.min()
    if task_type == "ESCAPE":
        d = out["done"].cpu().numpy()[:, :N // 32 * 32].reshape(T, -1, 32)
        assert d.all(axis=2).any()                     # all 32 lanes of a warp drew a task in the same step
    assert_same_envs(torch, roll, twin, record)
    assert_restated(roll, seed, base, count, n, fc)
    roll.close(); twin.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. windows on the resampled tasks = the CPU oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task_type,view_grid", [("SURVIVAL", 2), ("ESCAPE", 1)])
def test_windows_on_resampled_tasks_equal_the_oracle(torch_mod, task_type, view_grid):
    """A few envs, one resampling rollout with terminal windows: every obs, final_obs, reward and done equals an
    OracleMaze("2D") that is given the restated task whenever its episode ends."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    N, n, seed, max_steps, T = 6, 9, 41, 7, 24
    table, fc = slot_table(n, N)
    env = make_env(N, n, table, max_steps=max_steps, task_type=task_type, view_grid=view_grid, final_obs=True)
    oras = [OracleMaze("2D", task_type, max_steps, view_grid) for _ in range(N)]
    for o, t in zip(oras, table):
        o.set_task(t)
        o.reset()
    acts = torch.as_tensor(np.random.RandomState(6).randint(0, 4, (T, N)).astype(np.int32)).cuda()
    out = env.rollout(T, actions=acts, resample=dict(seed=seed, **CFG))
    obs, fin = out["obs"].cpu().numpy(), out["final_obs"].cpu().numpy()
    rew, done = out["rew"].cpu().numpy(), out["done"].cpu().numpy().astype(bool)
    a_h = acts.cpu().numpy()
    count = np.zeros(N, np.int64)
    for t in range(T):
        for e, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(a_h[t, e]))
            assert rew[t, e] == r2 and done[t, e] == d2, (t, e)
            if d2:
                assert np.array_equal(fin[t, e], o2), (t, e)
                count[e] += 1
                o.set_task(restated_tasks(seed, np.array([e]), np.array([count[e]]), n, fc, **CFG)[0])
                o2 = o.reset()
            assert np.array_equal(obs[t, e], o2), (t, e)
    assert count.min() >= 2
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. consecutive calls and a restore in between
# ---------------------------------------------------------------------------------------------------------------------
def test_consecutive_rollouts_and_restore_continue_the_loop(torch_mod):
    """Two resampling rollouts with drawn actions equal one twin loop over both; a snapshot taken between them and
    restored into a fresh handle continues bit for bit (outputs, drawn actions, records, tasks)."""
    torch = torch_mod
    N, n, seed, T1, T2 = 150, 9, SEED_HI, 13, 19
    table, fc = slot_table(n, N)
    kw = dict(max_steps=6, task_type="SURVIVAL", view_grid=2, env_index_base=BASE_HI, record_path=True, final_obs=True)
    roll, twin = make_env(N, n, table, **kw), make_env(N, n, table, **kw)
    rs = dict(seed=seed, **CFG)
    a = out_dict(torch, roll, T1, drawn=True)
    roll.rollout(T1, act_seed=11, out=a, resample=rs)
    snap = roll.snapshot()
    b = out_dict(torch, roll, T2, drawn=True)
    roll.rollout(T2, act_seed=11, out=b, resample=rs)
    count = run_twin(torch, twin, a, a["act"], seed, True) + run_twin(torch, twin, b, b["act"], seed, True)
    assert count.min() >= 3
    assert_same_envs(torch, roll, twin, True)
    assert_restated(roll, seed, BASE_HI, count, n, fc)
    fresh = make_env(N, n, table, **kw)
    fresh.restore(snap)
    c = out_dict(torch, fresh, T2, drawn=True)
    fresh.rollout(T2, act_seed=11, out=c, resample=rs)
    for k in ("act", "obs", "rew", "done", "final_obs", "truncated"):
        assert torch.equal(b[k], c[k]), k
    assert_same_envs(torch, roll, fresh, True)
    for e in (roll, twin, fresh):
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _ptr(t):
    return None if t is None else t.data_ptr()


def test_resampling_refusals_leave_the_handle_untouched(torch_mod, maze_golden):
    """Each refusal of mgb_maze_rollout with a sampler cfg returns MGB_ERR_ARG with its message (the sampler-cfg ones
    with the text mgb_maze_resample_tasks gives for the same cfg) and leaves snapshot() as it was, and the handle runs afterwards;
    rollout(resample=dict(goal_reward=-1)) raises ValueError."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, _lib
    from util import task_from_arrays
    N, T, n = 8, 3, 9
    table, _ = slot_table(n, N)
    lib = _lib.load()

    def bufs(env):
        shape = (T, N) + tuple(env._obs.shape[1:])
        return (torch.zeros(shape, dtype=env._obs.dtype, device="cuda"), torch.zeros((T, N), dtype=torch.float64, device="cuda"),
                torch.zeros((T, N), dtype=torch.uint8, device="cuda"), torch.zeros(shape, dtype=env._obs.dtype, device="cuda"),
                torch.zeros((T, N), dtype=torch.uint8, device="cuda"))

    def cfg(**over):
        return BatchedMetaMaze2D._sampler_cfg(**dict(dict(seed=3), **over))[0]

    def call(env, steps=T, f=False, tr=False, c="default"):
        obs, rew, done, fo, u8 = bufs(env)
        c = cfg() if c == "default" else c
        return lib.mgb_maze_rollout(env._h, steps, None, 0, None, obs.data_ptr(), rew.data_ptr(), done.data_ptr(),
                                    _ptr(fo) if f else None, _ptr(u8) if tr else None,
                                    None if c is None else ctypes.byref(c), 9, env._stream())

    def refused(env, text, **kw):
        before = records(env).clone()
        assert call(env, **kw) == MGB_ERR_ARG
        msg = lib.mgb_last_error().decode()
        assert msg.startswith("mgb_maze_rollout: ") and text in msg, msg
        assert torch.equal(records(env), before)
        return msg[len("mgb_maze_rollout: "):]

    env = make_env(N, n, table, max_steps=9, view_grid=2)
    # a 3-D handle resamples on the direct renderer (tests/test_maze3d_direct_rollout_gpu.py checks its outputs)
    d3 = BatchedMetaMazeDiscrete3D(resolution=(24, 16), max_steps=9, num_envs=N, squeeze=False, auto_reset=True, cache=False)
    d3.set_task(table, env2task=np.arange(N))
    d3.reset()
    assert call(d3) == 0
    torch.cuda.synchronize()
    for steps in (0, -1):
        refused(env, "T must be positive", steps=steps)
    assert call(env, c=None) == 0                                           # without a cfg: the plain rollout
    torch.cuda.synchronize()
    delta = np.array([16], np.int64)
    for arm in (lambda: lib.mgb_maze_set_mirrors(env._h, 1, delta.ctypes.data),
                lambda: lib.mgb_maze_set_multicast(env._h, 16)):
        assert arm() == 0
        refused(env, "mirrors")
        refused(env, "mirrors", f=True, tr=True)
        assert lib.mgb_maze_set_mirrors(env._h, 0, None) == 0
    # the sampler-cfg checks: the message of mgb_maze_resample_tasks
    for bad in (dict(step_reward=0.0), dict(agent_height=3.5), dict(cell_size=1.0), dict(n_texts=1),
                dict(food_reward=0.0), dict(crowd_ratio=-1.0), dict(food_density=-0.5)):
        text = refused(env, "", c=cfg(**bad))
        assert lib.mgb_maze_resample_tasks(env._h, None, ctypes.byref(cfg(**bad)), 3, env._stream()) == MGB_ERR_ARG
        assert lib.mgb_last_error().decode() == "mgb_maze_resample_tasks: " + text
    with pytest.raises(ValueError, match="goal reward"):
        env.rollout(T, resample=dict(seed=1, goal_reward=-1.0))
    assert call(env, f=True, tr=True) == 0                                   # usable again
    torch.cuda.synchronize()
    # auto-reset off: with or without final_obs
    assert lib.mgb_maze_set_options(env._h, 0) == 0
    refused(env, "auto_reset")
    refused(env, "auto_reset", f=True)
    assert lib.mgb_maze_set_options(env._h, 1) == 0
    # no slot per env: a shared table (odd n >= 7 holds for every handle that has a table)
    g = maze_golden
    shared = BatchedMetaMaze2D(max_steps=9, num_envs=N, squeeze=False, auto_reset=True)
    shared.set_task([task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                                      g["tasks15.interval"][k], g["tasks15.scalars"][k]) for k in range(2)])
    shared.reset()
    text = refused(shared, "one task-table slot per env")
    assert lib.mgb_maze_resample_tasks(shared._h, None, ctypes.byref(cfg()), 3, shared._stream()) == MGB_ERR_ARG
    assert lib.mgb_last_error().decode() == "mgb_maze_resample_tasks: " + text
    # shared memory: n = 31 with view_grid = 7 (the two tiles alone take 230 400 bytes)
    t31, _ = slot_table(31, N)
    big = make_env(N, 31, t31, max_steps=9, view_grid=7)
    refused(big, "shared memory")
    assert big.rollout(T)["obs"].shape == (T, N, 15, 15)                  # the plain rollout runs
    ok = make_env(N, 31, t31, max_steps=9, view_grid=6)
    assert call(ok, f=True, tr=True) == 0
    assert call(env) == 0
    torch.cuda.synchronize()
    for e in (env, d3, shared, big, ok):
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. CUDA-graph capture
# ---------------------------------------------------------------------------------------------------------------------
def test_graph_replay_equals_eager_resampling_rollouts(torch_mod):
    """rollout(T, resample=..., out=...) with terminal outputs, captured in a CUDA graph right after reset() and replayed
    K times, equals K eager calls on a twin: every output of every replay, then the snapshot records."""
    torch = torch_mod
    N, n, T, K = 200, 9, 6, 4
    table, _ = slot_table(n, N)
    kw = dict(max_steps=4, task_type="SURVIVAL", view_grid=2, final_obs=True)
    g_env, e_env = make_env(N, n, table, **kw), make_env(N, n, table, **kw)
    acts = torch.as_tensor(np.random.RandomState(2).randint(0, 4, (T, N)).astype(np.int32)).cuda()
    g_out, e_out = out_dict(torch, g_env, T), out_dict(torch, e_env, T)
    rs = dict(seed=12, **CFG)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            g_env.rollout(T, actions=acts, out=g_out, resample=rs)
    torch.cuda.synchronize()
    n_done = 0
    for k in range(K):
        graph.replay()
        e_env.rollout(T, actions=acts, out=e_out, resample=rs)
        torch.cuda.synchronize()
        n_done += int(e_out["done"].sum())
        for key in ("obs", "rew", "done", "final_obs", "truncated"):
            assert torch.equal(g_out[key], e_out[key]), (k, key)
    assert n_done > 0
    assert torch.equal(records(g_env), records(e_env))
    g_env.close(); e_env.close()
