"""The device task sampler (resample_tasks / mgb_maze_resample_tasks) task for task against its exact NumPy restatement
(tests/maze_sampler_draws.py): every field get_tasks returns, the restarted state, resample counts under masks and
restore, the task blob bytes a snapshot carries, frames stepped on the sampled tasks, CUDA-graph capture and the
goal_reward refusal."""
import numpy as np
import pytest

from maze_sampler_draws import restated_tasks, same_task

pytestmark = pytest.mark.gpu

SEED64 = (0xdeadbeef << 32) | 0x01234567
BASE_HI = 2 ** 32 - 500                  # env_index_base: the batch straddles genv = 2^32


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def table(n, N, food_cells):
    """N open-interior tasks, one slot per env; task 0 has `food_cells` food cells, the others none, so the table's
    f_max (the cap of the sampler's thinning) is food_cells."""
    from metagym_b200 import TaskConfig
    walls = np.ones((n, n), dtype=np.int32)
    walls[1:-1, 1:-1] = 0
    texts = np.where(walls > 0, 1, 0)
    base = TaskConfig(start=(1, 1), goal=(n - 2, n - 2), cell_walls=walls, cell_texts=texts, cell_size=2.0,
                      wall_height=3.2, agent_height=1.6, initial_life=1.0, max_life=2.0, step_reward=-0.01,
                      goal_reward=1.0, food_rewards=np.zeros((n, n)), food_interval=np.zeros((n, n), dtype=np.int32))
    food = np.zeros(n * n)
    free = np.nonzero(walls.ravel() == 0)[0][1:1 + food_cells]
    food[free] = 0.3
    first = base._replace(food_rewards=food.reshape(n, n), food_interval=np.where(food > 0, 5, 0).reshape(n, n))
    return [first] + [base] * (N - 1)


def make(kind, N, n, food_cells=127, base=0, textures=None, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    args = dict(num_envs=N, squeeze=False, env_index_base=base, max_steps=kw.pop("max_steps", 50),
                task_type=kw.pop("task_type", "SURVIVAL"))
    args.update(kw)
    if kind == "2D":
        env = BatchedMetaMaze2D(view_grid=1, **args)
    elif kind == "D3":
        env = BatchedMetaMazeDiscrete3D(resolution=args.pop("resolution", (16, 12)), textures=textures, cache=False, **args)
    else:
        env = BatchedMetaMazeContinuous3D(resolution=args.pop("resolution", (16, 12)), textures=textures, **args)
    fc = min(food_cells, (n - 2) ** 2 - 1)
    env.set_task(table(n, N, fc), env2task=np.arange(N))
    return env, fc


def check_tasks(env, want, envs=None):
    envs = np.arange(env.num_envs) if envs is None else np.asarray(envs)
    got = env.get_tasks(envs)
    bad = [int(e) for e, g, w in zip(envs, got, want) if not same_task(g, w)]
    assert not bad, ("%d env(s) differ, first %d" % (len(bad), bad[0]), got[envs.tolist().index(bad[0])], want[envs.tolist().index(bad[0])])


def check_restarted(env, tasks, envs):
    ag, life = env.agent_state()
    ag, life = ag.cpu().numpy()[envs], life.cpu().numpy()[envs]
    want = np.array([[t.start[0], t.start[1], 0, 0] for t in tasks])
    assert np.array_equal(ag, want) and (life == np.array([t.initial_life for t in tasks])).all()
    if env.KIND == 2:
        pos, ori = env.pose()
        pos, ori = pos.cpu().numpy()[envs], ori.cpu().numpy()[envs]
        cs = np.array([t.cell_size for t in tasks])
        centre = np.stack([want[:, 0] * cs + 0.5 * cs, want[:, 1] * cs + 0.5 * cs], axis=1).astype(np.float32)
        assert np.array_equal(pos, centre) and (ori == 0.0).all()


# n, allow_loops, crowd_ratio, food_density, food_reward, n_texts, goal_reward, kind, envs, base, seed, f_max: a
# pairwise cover of the parameter grid (every pair of values of any two parameters occurs in some row)
GRID = [
    (7, True, 0.0, 0.0, 0.5, 7, 3.5, "2D", 1027, 0, 11, 127),
    (7, True, 0.35, 0.01, 0.05, 2, None, "2D", 1027, BASE_HI, SEED64, 127),
    (7, False, 1.0, 0.2, 0.5, 7, None, "2D", 1027, 0, 12, 0),
    (15, False, 0.0, 0.01, 0.5, 2, None, "C3", 1027, 0, 13, 127),
    (15, True, 0.35, 0.2, 0.5, 7, 3.5, "D3", 1027, BASE_HI, SEED64, 127),
    (15, False, 1.0, 0.0, 0.05, 2, 3.5, "2D", 1027, 0, 14, 127),
    (31, True, 0.0, 0.2, 0.05, 2, 3.5, "2D", 1027, 0, 15, 1),
    (31, False, 0.35, 0.0, 0.5, 7, None, "2D", 1027, 0, 16, 127),
    (31, True, 1.0, 0.01, 0.5, 7, 3.5, "2D", 1027, BASE_HI, SEED64, 127),
    (31, True, 0.35, 0.01, 0.05, 7, 3.5, "2D", 4099, BASE_HI, SEED64, 127),
]


@pytest.mark.parametrize("n,loops,crowd,density,reward,n_texts,goal,kind,N,base,seed,f_max", GRID)
def test_resampled_tasks_equal_the_restatement(torch_mod, textures, n, loops, crowd, density, reward, n_texts, goal,
                                               kind, N, base, seed, f_max):
    """One resample of every env: each field of get_tasks equals the restated task (float64 by ==), and every env
    restarted on it (start cell, heading 0, step 0, initial life; the continuous kind at the cell centre, heading 0).
    The table's f_max of 0 and 1 makes the food cap drive the thinning."""
    env, fc = make(kind, N, n, food_cells=f_max, base=base, textures=textures)
    env.reset()
    kw = dict(allow_loops=loops, crowd_ratio=crowd, food_density=density, food_reward=reward, n_texts=n_texts,
              goal_reward=goal, food_interval=7, cell_size=2.5 if kind != "2D" else 2.0, agent_height=1.2,
              wall_height=2.8, initial_life=1.5, max_life=3.0, step_reward=-0.02)
    env.resample_tasks(None, seed=seed, **kw)
    want = restated_tasks(seed, np.arange(N) + base, 1, n, fc, **kw)
    check_tasks(env, want)
    check_restarted(env, want, np.arange(N))
    if f_max <= 1:
        assert max(int((t.food_rewards > 0).sum()) for t in want) <= f_max
    env.close()


def test_masks_and_counts(torch_mod):
    """Three resamples under different masks: the k-th resample of an env equals the restatement at ep = k; envs left
    out keep their task, their state and their next step bit for bit (against a twin restored from a snapshot taken
    just before the call)."""
    torch = torch_mod
    N, n, seed = 1027, 15, 77
    kw = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.05, food_interval=3)
    env, fc = make("2D", N, n, max_steps=40, auto_reset=True)
    twin, _ = make("2D", N, n, max_steps=40, auto_reset=True)
    env.reset()
    rs = np.random.RandomState(8)
    count = np.zeros(N, dtype=np.int64)
    for call, p in enumerate((0.5, 0.2, 0.9)):
        for _ in range(3):
            env.step(torch.from_numpy(rs.randint(0, 4, N).astype(np.int32)).cuda())
        mask = rs.rand(N) < p
        before = env.get_tasks(np.arange(N))
        ag0, life0 = [x.cpu().numpy() for x in env.agent_state()]
        twin.restore(env.snapshot())
        env.resample_tasks(torch.from_numpy(mask.astype(np.uint8)).cuda(), seed=seed, **kw)
        count += mask
        ids = np.nonzero(mask)[0]
        want = restated_tasks(seed, ids, count[ids], n, fc, **kw)
        check_tasks(env, want, ids)
        check_restarted(env, want, ids)
        out = np.nonzero(~mask)[0]
        assert all(same_task(a, before[e]) for a, e in zip(env.get_tasks(out), out))
        ag, life = [x.cpu().numpy() for x in env.agent_state()]
        assert np.array_equal(ag[out], ag0[out]) and np.array_equal(life[out], life0[out])
        act = torch.from_numpy(rs.randint(0, 4, N).astype(np.int32)).cuda()
        r1 = [x.cpu().numpy()[out] for x in env.step(act)[:3]]
        r2 = [x.cpu().numpy()[out] for x in twin.step(act)[:3]]
        assert all(np.array_equal(x, y) for x, y in zip(r1, r2)), call
    assert (env.snapshot()["records"].view(torch.int32)[:, 6].cpu().numpy() == count).all()
    env.close()
    twin.close()


def blob_bytes(n, f_max):
    off = 104 + 3 * n * n
    off = (off + 7) // 8 * 8 + max(f_max, 1) * 12
    return (off + 15) // 16 * 16


def test_sampled_blob_is_the_blob_of_the_same_task_given_by_update_tasks(torch_mod):
    """A twin gets the restated tasks through update_tasks; the task-blob part of every snapshot record is byte for byte
    the same as the sampling handle's, after two resamples (so slots past the second task's food count once held the
    first's) -- this covers the header fields get_tasks does not return (n_food, cls, inv_cell, inv_t2c, the
    power-of-two flags) and the zeroed tail of the food slots."""
    N, n, seed = 257, 15, 5
    kw = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.1, food_interval=4, cell_size=2.5)
    env, fc = make("2D", N, n, food_cells=60)
    twin, _ = make("2D", N, n, food_cells=60)
    for e in (env, twin):
        e.reset()
    env.resample_tasks(None, seed=seed, **kw)
    env.resample_tasks(None, seed=seed + 1, **kw)
    want = restated_tasks(seed + 1, np.arange(N), 2, n, fc, **kw)
    check_tasks(env, want)
    twin.update_tasks(np.arange(N), want)
    a, b = env.snapshot()["records"].cpu().numpy(), twin.snapshot()["records"].cpu().numpy()
    bb = blob_bytes(n, fc)
    assert a.shape == b.shape and a.shape[1] == 48 + (fc + 3) // 4 * 16 + bb
    assert np.array_equal(a[:, -bb:], b[:, -bb:])
    env.close()
    twin.close()


def test_continuation_after_restore(torch_mod):
    """Restore into a fresh handle that never resampled, then resample: every env equals the restatement at its
    restored count + 1."""
    torch = torch_mod
    N, n, seed = 1027, 9, 31
    kw = dict(allow_loops=False, food_density=0.05)
    env, fc = make("2D", N, n)
    env.reset()
    rs = np.random.RandomState(2)
    count = np.zeros(N, dtype=np.int64)
    for _ in range(2):
        mask = rs.rand(N) < 0.6
        env.resample_tasks(torch.from_numpy(mask.astype(np.uint8)).cuda(), seed=seed, **kw)
        count += mask
    snap = env.snapshot()
    fresh, _ = make("2D", N, n)
    fresh.restore(snap)
    fresh.resample_tasks(None, seed=seed, **kw)
    check_tasks(fresh, restated_tasks(seed, np.arange(N), count + 1, n, fc, **kw))
    env.close()
    fresh.close()


@pytest.mark.parametrize("kind", ["D3", "C3"])
@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
def test_frames_on_sampled_tasks_equal_the_oracle(torch_mod, textures, kind, task_type):
    """Episodes with auto-reset on tasks drawn on the device with heights the table does not have (agent 1.2, wall 2.8:
    the renderer's per-pixel path) and cell_size 2.5: every frame, reward and done equals an OracleMaze fed the
    restated task (not the device read-back)."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    N, n, seed, res, max_steps = 12, 9, 41, (24, 16), 15
    kw = dict(allow_loops=True, crowd_ratio=0.3, food_density=0.08, food_interval=3, cell_size=2.5, agent_height=1.2,
              wall_height=2.8)
    env, fc = make(kind, N, n, textures=textures, max_steps=max_steps, task_type=task_type, auto_reset=True,
                   resolution=res)
    oras = [OracleMaze("3D" if kind == "D3" else "C3D", task_type, max_steps, 1, res, textures=textures) for _ in range(N)]
    env.reset()
    count = np.ones(N, dtype=np.int64)
    env.resample_tasks(None, seed=seed, **kw)
    for o, t in zip(oras, restated_tasks(seed, np.arange(N), 1, n, fc, **kw)):
        o.set_task(t)
        o.reset()
    rs = np.random.RandomState(6)
    retasked = 0
    for t in range(45):
        if kind == "D3":
            act = rs.randint(0, 4, N).astype(np.int32)
        else:
            act = rs.uniform(-1, 1, (N, 2)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.from_numpy(act).cuda())
        obs, rew_h, done_h = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy().astype(bool)
        for e, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(act[e]) if kind == "D3" else act[e])
            assert rew_h[e] == r2 and bool(done_h[e]) == d2, (t, e)
            if d2:
                o2 = o.reset()
            assert np.array_equal(obs[e], o2), (t, e, int((obs[e] != o2).sum()))
        if done_h.any():
            env.resample_tasks(done, seed=seed, **kw)
            ids = np.nonzero(done_h)[0]
            count[ids] += 1
            for e, nt in zip(ids, restated_tasks(seed, ids, count[ids], n, fc, **kw)):
                oras[e].set_task(nt)
                oras[e].reset()
                retasked += 1
    assert retasked >= N // 2
    env.close()


def test_capture_step_resample_and_restore_on_handles_that_never_resampled(torch_mod):
    """step + resample_tasks(done) captured in a CUDA graph on a handle that never resampled, replayed, equals the
    eager calls; so does a restore captured into a handle that never resampled."""
    torch = torch_mod
    from metagym_b200 import _lib
    N, n, seed = 300, 9, 3
    kw = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.05)
    g_env, _ = make("2D", N, n, max_steps=6, auto_reset=True)
    eager, _ = make("2D", N, n, max_steps=6, auto_reset=True)
    for e in (g_env, eager):
        e.reset()
    act = torch.zeros(N, dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            _, _, done, _ = g_env.step(act)
            g_env.resample_tasks(done, seed=seed, **kw)
    torch.cuda.synchronize()
    rs = np.random.RandomState(1)
    for t in range(14):
        a = torch.from_numpy(rs.randint(0, 4, N).astype(np.int32)).cuda()
        act.copy_(a)
        graph.replay()
        _, _, d, _ = eager.step(a)
        eager.resample_tasks(d, seed=seed, **kw)
        torch.cuda.synchronize()
        assert torch.equal(g_env._obs, eager._obs) and torch.equal(g_env._rew, eager._rew), t
    a1, a2 = g_env.snapshot()["records"], eager.snapshot()["records"]
    assert torch.equal(a1, a2) and int(a1.view(torch.int32)[:, 6].max()) >= 2
    # restore into a fresh handle, captured
    snap = g_env.snapshot()
    dst, _ = make("2D", N, n, max_steps=6, auto_reset=True)
    ref, _ = make("2D", N, n, max_steps=6, auto_reset=True)
    for e in (dst, ref):
        e.reset()
    ref.restore(snap)
    row = torch.arange(N, dtype=torch.int64, device="cuda")
    rec = snap["records"]
    with torch.cuda.stream(s):
        graph2 = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph2, stream=s):
            _lib.check(dst._lib.mgb_maze_restore(dst._h, rec.data_ptr(), N, row.data_ptr(), dst._stream()))
    graph2.replay()
    torch.cuda.synchronize()
    assert torch.equal(dst.snapshot()["records"], ref.snapshot()["records"])
    dst.resample_tasks(None, seed=seed, **kw)
    ref.resample_tasks(None, seed=seed, **kw)
    assert torch.equal(dst.snapshot()["records"], ref.snapshot()["records"])
    for e in (g_env, eager, dst, ref):
        e.close()


def test_goal_reward_refusal_leaves_the_handle_untouched(torch_mod):
    """resample_tasks(goal_reward=-1.0) (and 0.0) raises ValueError, as the host sampler refuses it, and changes
    neither the handle's fingerprint nor its next step."""
    torch = torch_mod
    N, n = 64, 9
    env, _ = make("2D", N, n, max_steps=30)
    twin, _ = make("2D", N, n, max_steps=30)
    for e in (env, twin):
        e.reset()
        e.resample_tasks(None, seed=4)
    for bad in (-1.0, 0.0):
        with pytest.raises(ValueError, match="goal reward"):
            env.resample_tasks(None, seed=5, goal_reward=bad)
    assert np.array_equal(env._fingerprint(), twin._fingerprint())
    assert torch.equal(env.snapshot()["records"], twin.snapshot()["records"])
    act = torch.from_numpy(np.random.RandomState(0).randint(0, 4, N).astype(np.int32)).cuda()
    r1, r2 = env.step(act), twin.step(act)
    assert all(torch.equal(x, y) for x, y in zip(r1[:3], r2[:3]))
    env.close()
    twin.close()
