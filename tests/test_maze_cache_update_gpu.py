"""update_tasks on the pose cache of MetaMazeDiscrete3D: the replaced tasks' region of the slot-strided cache is rebuilt in
place on the stream.  Checked against the CPU oracle, against a direct-renderer twin bit for bit at the benchmark shape,
against a cache freshly built from the final table, and for refusals, stream order and snapshots."""
import numpy as np
import pytest

from util import task_from_arrays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


@pytest.fixture(scope="module")
def pool(maze_golden):
    g = maze_golden
    return [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                             g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(8)]


def free_cells(task):
    """Free cells as the pose cache counts them: every non-wall cell and the start cell."""
    walls = np.asarray(task.cell_walls) == 0
    walls[task.start[0], task.start[1]] = True
    return int(walls.sum())


def maze3d(n, textures, **kw):
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    kw.setdefault("resolution", (32, 24))
    kw.setdefault("max_steps", 30)
    kw.setdefault("task_type", "SURVIVAL")
    return BatchedMetaMazeDiscrete3D(num_envs=n, squeeze=False, textures=textures, **kw)


@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
def test_updates_on_the_cache_follow_the_oracle(torch_mod, pool, textures, task_type):
    """One table slot per env on the cache: every env's obs, reward and done equal the oracle of its current task through
    updates between steps (twice in a row too), including a replacement with other cell, wall and agent heights."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    N = 12
    env = maze3d(N, textures, task_type=task_type, obs_dtype="uint8")
    oras = [OracleMaze("3D", task_type, 30, 1, (32, 24), textures=textures) for _ in range(N)]
    cur = [pool[i % 4] for i in range(N)]
    env.set_task(cur, env2task=np.arange(N))
    obs = env.reset().cpu().numpy()
    assert env.cache_info()["in_use"]
    for i, o in enumerate(oras):
        o.set_task(cur[i])
        assert np.array_equal(obs[i], np.minimum(o.reset(), 255))
    cell = max(t.cell_size for t in cur)
    odd = pool[5]._replace(cell_size=cell * 1.25, wall_height=4.5, agent_height=1.2)
    choices = pool[4:] + [odd]
    rs = np.random.RandomState(4)
    for t in range(40):
        if t in (3, 7, 8, 19, 33):
            ids = rs.choice(N, size=4, replace=False)
            new = [choices[int(rs.randint(len(choices)))] for _ in ids]
            if t == 3:
                new[0] = odd
            env.update_tasks(ids, new)
            for i, nt in zip(ids, new):
                oras[i].set_task(nt)
                oras[i].reset()
        act = rs.randint(0, 4, size=N)
        obs, rew, done, _ = env.step(torch.as_tensor(act, dtype=torch.int32).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for i, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(act[i]))
            assert np.array_equal(obs[i], np.minimum(o2, 255)) and rew[i] == r2 and bool(done[i]) == d2, (t, i)
            if d2:
                o.reset()
        if done.any():
            env.reset(mask=torch.as_tensor(done).cuda())
    env.close()


def bench_tasks(k, seed):
    from metagym_b200 import MazeTaskSampler
    rs = np.random.RandomState(seed)
    return [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=rs) for _ in range(k)]


@pytest.mark.parametrize("path", ["u8_fused", "u8_two_kernels", "int32", "float32"])
def test_cache_equals_direct_renderer_through_updates(torch_mod, textures, monkeypatch, path):
    """1024 envs, 64 tasks x 16 envs, 128x128, episodes that end: staggered updates of 8 slots every few steps (no host
    synchronisation in the loop) go to a cached handle and a cache=False twin alike; obs, rewards, dones, terminal frames,
    truncation flags, recorded paths, and a rollout with drawn actions replayed by the twin's steps agree bit for bit."""
    torch = torch_mod
    monkeypatch.setenv("MGB_MAZE_FUSED_STEP", "0" if path == "u8_two_kernels" else "1")
    dtype = {"u8_fused": "uint8", "u8_two_kernels": "uint8"}.get(path, path)
    N, K = 1024, 64
    table = bench_tasks(K, 3)
    most = max(free_cells(t) for t in table)
    foods = max(int((np.asarray(t.food_rewards) > 0).sum()) for t in table)
    fresh = [t for t in bench_tasks(160, 5)
             if free_cells(t) <= most and int((np.asarray(t.food_rewards) > 0).sum()) <= foods]
    assert len(fresh) >= 16
    envs = [maze3d(N, textures, resolution=(128, 128), max_steps=12, obs_dtype=dtype, auto_reset=True, final_obs=True,
                   record_path=True, cache=c) for c in (True, False)]
    e2t = np.repeat(np.arange(K), N // K)
    for env in envs:
        env.set_task(table, env2task=e2t)
        env.reset()
    assert envs[0].cache_info()["in_use"] and not envs[1].cache_info()["in_use"]
    g = torch.Generator(device="cuda").manual_seed(9)
    acts = torch.randint(0, 4, (40, N), device="cuda", dtype=torch.int32, generator=g)
    bad = torch.zeros((), dtype=torch.bool, device="cuda")
    rs = np.random.RandomState(2)
    for t in range(40):
        if t % 3 == 1:
            slots = rs.choice(K, size=8, replace=False)
            new = [fresh[int(rs.randint(len(fresh)))] for _ in slots]
            for env in envs:
                env.update_tasks(slots, new)
        a, b = [env.step(acts[t])[:3] for env in envs]
        for x, y in zip(a, b):
            bad |= (x != y).any()
        d = a[2].view(-1)
        fa, fb = envs[0].final_observation, envs[1].final_observation
        bad |= (fa[d] != fb[d]).any()
        bad |= (envs[0].truncated != envs[1].truncated).any()
    assert not bool(bad)
    ta, tb = envs[0].trajectory(), envs[1].trajectory()
    assert torch.equal(ta[0], tb[0]) and torch.equal(ta[1], tb[1])
    slots = np.arange(8) * 8
    for env in envs:
        env.update_tasks(slots, fresh[:8])
    T = 16
    out = envs[0].rollout(T, act_seed=5, want_actions=True, final_obs=True)
    for t in range(T):
        obs, rew, done, _ = envs[1].step(out["act"][t])
        d = done.view(-1)
        assert torch.equal(out["obs"][t], obs) and torch.equal(out["rew"][t], rew), t
        assert torch.equal(out["done"][t].bool(), done) and torch.equal(out["truncated"][t], envs[1].truncated), t
        assert torch.equal(out["final_obs"][t][d], envs[1].final_observation[d]), t
    for env in envs:
        env.close()


def test_rebuilt_regions_equal_a_fresh_build(torch_mod, pool, textures):
    """After several updates (one slot twice) a cached handle behaves exactly like a handle given set_task(final table):
    the same outputs under the same actions, and the same pose and variant-frame counts -- every replaced task, a task of
    the original table in another slot, gets all its variant frames."""
    torch = torch_mod
    N = 16
    table = list(pool)
    a = maze3d(N, textures, obs_dtype="uint8", auto_reset=True)
    a.set_task(table, env2task=np.arange(N) % 8)
    a.reset()
    info0 = a.cache_info()
    assert info0["in_use"] and info0["variant_frames"] > 0
    acts = torch.randint(0, 4, (30, N), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(1))
    for t, (slots, new) in enumerate([([2, 6], [5, 0]), ([2], [7]), ([1, 3, 4], [6, 6, 2])]):
        a.step(acts[t])
        a.update_tasks(slots, [pool[k] for k in new])
        for s, k in zip(slots, new):
            table[s] = pool[k]
    b = maze3d(N, textures, obs_dtype="uint8", auto_reset=True)
    b.set_task(table, env2task=np.arange(N) % 8)
    oa, ob = a.reset(), b.reset()
    assert torch.equal(oa, ob)
    ia, ib = a.cache_info(), b.cache_info()
    for k in ("poses", "variant_frames", "variant_bits", "poses_by_food_count"):
        assert ia[k] == ib[k], (k, ia[k], ib[k])
    for t in range(30):
        ra, rb = a.step(acts[t])[:3], b.step(acts[t])[:3]
        for x, y in zip(ra, rb):
            assert torch.equal(x, y), t
    a.close()
    b.close()


def test_refusals_on_the_cache_leave_the_handle_untouched(torch_mod, pool, textures):
    """A replacement with more free cells than the table's largest task, and one with a texture no loaded texture has, are
    refused on a cached handle before anything is written: fingerprint and the next step equal an untouched twin's."""
    torch = torch_mod
    from metagym_b200._lib import MgbError
    small = pool[:4]
    dst, twin = [maze3d(4, textures, obs_dtype="uint8") for _ in range(2)]
    for env in (dst, twin):
        env.set_task(small, env2task=np.arange(4))
        env.reset()
    walls = np.asarray(small[0].cell_walls).copy()
    walls[1:-1, 1:-1] = 0                                   # no inner walls: more free cells than any task of the table
    big = small[0]._replace(cell_walls=walls)
    assert free_cells(big) > max(free_cells(t) for t in small)
    with pytest.raises(MgbError, match="free cells"):
        dst.update_tasks([1], [big])
    texts = np.asarray(small[0].cell_texts).copy()
    texts[0, 0] = 15
    with pytest.raises(MgbError, match="texture that is not loaded"):
        dst.update_tasks([2], [small[0]._replace(cell_texts=texts)])
    assert np.array_equal(dst._fingerprint(), twin._fingerprint())
    act = torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda")
    for x, y in zip(dst.step(act)[:3], twin.step(act)[:3]):
        assert torch.equal(x, y)
    dst.close()
    twin.close()


def test_update_on_the_cache_does_not_synchronise(torch_mod, pool, textures):
    """update_tasks on a cached handle enqueues its work behind what the stream already holds and returns at once."""
    torch = torch_mod
    env = maze3d(8, textures, obs_dtype="uint8")
    env.set_task(pool, env2task=np.arange(8))
    env.reset()
    assert env.cache_info()["in_use"]
    env.update_tasks([1, 2], [pool[3], pool[4]])         # both staging halves exist from here on
    env.update_tasks([5], [pool[6]])
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream()
    torch.cuda._sleep(2_000_000_000)
    env.update_tasks([0, 7], [pool[5], pool[2]])
    assert not stream.query()
    torch.cuda.synchronize()
    env.close()


def test_snapshot_after_an_update_restores_into_a_twin(torch_mod, pool, textures):
    """A snapshot taken after update_tasks on the cache restores into a handle holding the same table and both continue
    bit for bit."""
    torch = torch_mod
    N = 8
    src = maze3d(N, textures, obs_dtype="uint8", auto_reset=True)
    table = list(pool)
    src.set_task(table, env2task=np.arange(N))
    src.reset()
    acts = torch.randint(0, 4, (20, N), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(3))
    for t in range(5):
        src.step(acts[t])
    src.update_tasks([2, 6], [pool[1], pool[0]])      # the table keeps its largest food count: the same record layout
    table[2], table[6] = pool[1], pool[0]
    src.step(acts[5])
    snap = src.snapshot()
    dst = maze3d(N, textures, obs_dtype="uint8", auto_reset=True)
    dst.set_task(table, env2task=np.arange(N))
    dst.reset()
    dst.restore(snap)
    for t in range(6, 20):
        for x, y in zip(src.step(acts[t])[:3], dst.step(acts[t])[:3]):
            assert torch.equal(x, y), t
    src.close()
    dst.close()
