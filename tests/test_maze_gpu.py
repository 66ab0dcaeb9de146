"""GPU parity tests of the MetaMaze path: libmgb200 against golden episodes recorded from the unmodified reference
(tests/golden/maze_golden.npz) and against the CPU oracle (oracle/maze_oracle.c).  Everything is compared bit for bit:
grid indices, heading, step counters, done flags, float64 rewards / life, float32 2-D observations, int32 raycast images
(and the uint8 mode as min(reference, 255))."""
import numpy as np
import pytest

from util import MAZE_CASES, maze_case, task_from_arrays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def make_env(c, n, textures, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D
    if c["kind"] == "2D":
        return BatchedMetaMaze2D(max_steps=c["max_steps"], task_type=c["task_type"], view_grid=c["view_grid"],
                                 num_envs=n, squeeze=False, **kw)
    return BatchedMetaMazeDiscrete3D(resolution=c["resolution"], max_steps=c["max_steps"], task_type=c["task_type"],
                                     num_envs=n, squeeze=False, textures=textures, **kw)


@pytest.fixture(params=["pose_cache", "direct_render"])
def render_path(request, monkeypatch):
    """3-D observations come either from the memoised pose cache (default) or from the direct float64 renderer
    (MGB_MAZE_CACHE=0); both must reproduce the reference bit for bit."""
    monkeypatch.setenv("MGB_MAZE_CACHE", "1" if request.param == "pose_cache" else "0")
    return request.param


GEOM_CASES = ["g3d_surv", "g3d_esc"]      # non-default cell / wall / eye heights (tests/golden/gen_maze_geom.py)


@pytest.mark.parametrize("name", MAZE_CASES + GEOM_CASES)
@pytest.mark.parametrize("n", [1, 3])
def test_reference_episode(torch_mod, maze_golden, geom_golden, textures, name, n, render_path):
    """Replay the recorded reference episode on n identical envs (manual reset after done, like the reference user)."""
    torch = torch_mod
    c = maze_case(geom_golden if name in GEOM_CASES else maze_golden, name)
    if c["kind"] == "2D" and render_path == "direct_render":
        pytest.skip("2-D has a single path")
    env = make_env(c, n, textures)
    with pytest.raises(Exception, match="set_task"):
        env.reset()
    env.set_task(c["task"])
    with pytest.raises(Exception, match="reset"):
        env.step(torch.zeros(n, dtype=torch.int32, device="cuda"))
    obs0 = env.reset().cpu().numpy()
    for k in range(n):
        assert np.array_equal(obs0[k], c["reset_obs"].astype(obs0.dtype))
    kept = {int(t): k for k, t in enumerate(c["obs_idx"])}
    for t, a in enumerate(c["act"]):
        obs, rew, done, info = env.step(torch.full((n,), int(a), dtype=torch.int32, device="cuda"))
        ag, life = env.agent_state()
        ag, life, rew_h, done_h = ag.cpu().numpy(), life.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for k in range(n):
            assert rew_h[k] == c["rew"][t], (t, rew_h[k], c["rew"][t])
            assert bool(done_h[k]) == bool(c["done"][t]), t
            assert tuple(ag[k]) == tuple(int(x) for x in c["agent"][t]), (t, ag[k], c["agent"][t])
            if c["task_type"] == "SURVIVAL":
                assert life[k] == c["life"][t], t
        if t in kept:
            o = obs.cpu().numpy()
            ref = c["obs"][kept[t]]
            for k in range(n):
                assert np.array_equal(o[k], ref.astype(o.dtype)), (t, int((o[k] != ref).sum()))
        assert int(info["steps"][0]) == int(c["agent"][t][3])
        if c["done"][t]:
            env.reset()
    env.close()


def test_uint8_mode_is_clamped_reference(torch_mod, maze_golden, textures, render_path):
    torch = torch_mod
    c = maze_case(maze_golden, "m3d_big")
    bright = (textures[0].copy(), textures[1])
    bright[0][0] = 255          # bright ground -> exact values exceed 255 near the bottom of the screen
    a = make_env(c, 1, bright, obs_dtype="int32")
    b = make_env(c, 1, bright, obs_dtype="uint8")
    for e in (a, b):
        e.set_task(c["task"])
        e.reset()
    for t in range(10):
        act = torch.full((1,), int(c["act"][t]), dtype=torch.int32, device="cuda")
        o32 = a.step(act)[0].cpu().numpy()
        o8 = b.step(act)[0].cpu().numpy()
        assert o8.dtype == np.uint8 and np.array_equal(o8, np.minimum(o32, 255).astype(np.uint8))
    assert o32.max() > 255
    a.close()
    b.close()


@pytest.mark.parametrize("kind,task_type", [("2D", "SURVIVAL"), ("2D", "ESCAPE"), ("3D", "SURVIVAL"), ("3D", "ESCAPE")])
def test_random_batch_vs_oracle(torch_mod, maze_golden, textures, kind, task_type, render_path):
    """Many envs, several tasks, independent random actions, auto-reset on: every env equals its own oracle instance."""
    torch = torch_mod
    if kind == "2D" and render_path == "direct_render":
        pytest.skip("2-D has a single path")
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(4)]
    n, T, max_steps, res = (96, 120, 40, None) if kind == "2D" else (20, 45, 25, (40, 24))
    if kind == "2D":
        env = BatchedMetaMaze2D(max_steps=max_steps, task_type=task_type, view_grid=2, num_envs=n, squeeze=False,
                                auto_reset=True)
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=res, max_steps=max_steps, task_type=task_type, num_envs=n,
                                        squeeze=False, auto_reset=True, textures=textures)
    env.set_task(tasks)
    oracles = []
    for e in range(n):
        o = OracleMaze(kind, task_type, max_steps, 2, res or (8, 8), textures=textures if kind == "3D" else None)
        o.set_task(tasks[e % 4])
        oracles.append(o)
    obs = env.reset().cpu().numpy()
    for e in range(n):
        assert np.array_equal(obs[e], oracles[e].reset())
    rng = np.random.RandomState(7)
    n_done = 0
    for t in range(T):
        act = rng.randint(0, 4, n)
        obs, rew, done, _ = env.step(torch.as_tensor(act, dtype=torch.int32).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for e in range(n):
            o2, r2, d2, _ = oracles[e].step(int(act[e]))
            assert rew[e] == r2 and bool(done[e]) == d2, (t, e)
            if d2:
                o2 = oracles[e].reset()         # auto-reset publishes the first observation of the next episode
                n_done += 1
            assert np.array_equal(obs[e], o2), (t, e)
    assert n_done > 0
    env.close()


def test_masked_reset(torch_mod, maze_golden):
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D
    c = maze_case(maze_golden, "m2d_surv")
    env = BatchedMetaMaze2D(max_steps=60, view_grid=1, num_envs=4, squeeze=False)
    env.set_task(c["task"])
    env.reset()
    for a in c["act"][:10]:
        env.step(torch.full((4,), int(a), dtype=torch.int32, device="cuda"))
    before, _ = env.agent_state()
    env.reset(mask=torch.tensor([1, 0, 0, 1], device="cuda"))
    after, life = env.agent_state()
    after, before = after.cpu().numpy(), before.cpu().numpy()
    assert tuple(after[0]) == (c["task"].start[0], c["task"].start[1], 0, 0) and np.array_equal(after[0], after[3])
    assert np.array_equal(after[1], before[1]) and np.array_equal(after[2], before[2])
    env.close()


def test_pose_cache_equals_direct_render_at_config4_shape(torch_mod, maze_golden, textures, monkeypatch):
    """1024 envs, 15x15, 128x128 uint8 (BASELINE config 4 per GPU): memoised path == direct float64 renderer."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 20, g["tasks15.scalars"][k]) for k in range(8)]
    N = 1024
    kw = dict(resolution=(128, 128), max_steps=60, task_type="SURVIVAL", squeeze=False, auto_reset=True,
              obs_dtype="uint8", textures=textures, num_envs=N)
    monkeypatch.setenv("MGB_MAZE_CACHE", "1")
    a = BatchedMetaMazeDiscrete3D(**kw)
    monkeypatch.setenv("MGB_MAZE_CACHE", "0")
    b = BatchedMetaMazeDiscrete3D(**kw)
    for e in (a, b):
        e.set_task(tasks)
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator(device="cuda").manual_seed(3)
    for t in range(80):
        act = torch.randint(0, 4, (N,), device="cuda", generator=gen, dtype=torch.int32)
        o1, r1, d1, _ = a.step(act)
        o2, r2, d2, _ = b.step(act)
        assert torch.equal(o1, o2), (t, int((o1 != o2).sum()))
        assert torch.equal(r1, r2) and torch.equal(d1, d2)
    a.close()
    b.close()


@pytest.mark.parametrize("res,task_type,vbits", [((128, 128), "SURVIVAL", None), ((64, 48), "SURVIVAL", None),
                                                 ((96, 80), "ESCAPE", None), ((256, 256), "SURVIVAL", None),
                                                 ((128, 128), "SURVIVAL", "0"), ((64, 48), "SURVIVAL", "2")])
def test_fused_step_kernel_equals_two_kernel_path(torch_mod, maze_golden, textures, monkeypatch, res, task_type, vbits):
    """uint8 frames take maze3d_step_kernel (logic + TMA-moved baked frame + in-smem patches, one launch); it must equal the
    logic + compose kernel pair bit for bit: partial last chunk (64x48 = one 9 KB chunk), many chunks (256x256 = 16),
    tinted groups under the life bar, auto-reset, reset() frames.  vbits = MGB_MAZE_VARIANT_BITS: with 0 or 2 variant bits
    most frames with an eaten food in view keep float64 tints, i.e. the kernel's three-warp tint group runs for real."""
    torch = torch_mod
    if vbits is not None:
        monkeypatch.setenv("MGB_MAZE_VARIANT_BITS", vbits)
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 20, g["tasks15.scalars"][k]) for k in range(6)]
    N = 300
    kw = dict(resolution=res, max_steps=50, task_type=task_type, squeeze=False, auto_reset=True, obs_dtype="uint8",
              textures=textures, num_envs=N)
    monkeypatch.setenv("MGB_MAZE_FUSED_STEP", "1")
    a = BatchedMetaMazeDiscrete3D(**kw)
    monkeypatch.setenv("MGB_MAZE_FUSED_STEP", "0")
    b = BatchedMetaMazeDiscrete3D(**kw)
    monkeypatch.delenv("MGB_MAZE_FUSED_STEP")
    for e in (a, b):
        e.set_task(tasks)
    assert torch.equal(a.reset(), b.reset())
    gen = torch.Generator(device="cuda").manual_seed(13)
    changed = 0
    for t in range(70):
        act = torch.randint(0, 4, (N,), device="cuda", generator=gen, dtype=torch.int32)
        o1, r1, d1, _ = a.step(act)
        o2, r2, d2, _ = b.step(act)
        assert torch.equal(o1, o2), (t, int((o1 != o2).sum()))
        assert torch.equal(r1, r2) and torch.equal(d1, d2)
        changed += int(d1.sum())
    assert changed > 0
    ag1, l1 = a.agent_state()
    ag2, l2 = b.agent_state()
    assert torch.equal(ag1, ag2) and torch.equal(l1, l2)
    a.close()
    b.close()


def test_maze2d_large_view_grid(torch_mod, maze_golden):
    """view_grid = 5: the 2-D step kernel needs 62 KB of dynamic shared memory (round-1 advice: the attribute was only
    raised on the rollout path, every step()/reset() failed with 'invalid argument')."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    task = task_from_arrays(g["tasks15.walls"][0], g["tasks15.texts"][0], g["tasks15.food"][0], g["tasks15.interval"][0] // 10,
                            g["tasks15.scalars"][0])
    env = BatchedMetaMaze2D(max_steps=30, task_type="SURVIVAL", view_grid=5, num_envs=3, squeeze=False)
    ora = OracleMaze("2D", "SURVIVAL", 30, 5)
    env.set_task(task)
    ora.set_task(task)
    assert np.array_equal(env.reset().cpu().numpy()[0], ora.reset())
    rs = np.random.RandomState(2)
    for t in range(12):
        act = int(rs.randint(4))
        obs, rew, done, _ = env.step(torch.full((3,), act, device="cuda", dtype=torch.int32))
        o2, r2, d2, _ = ora.step(act)
        assert np.array_equal(obs.cpu().numpy()[2], o2) and float(rew[1]) == r2 and bool(done[0]) == d2
    env.close()


@pytest.mark.parametrize("kind", ["2D", "3D"])
def test_update_tasks_equals_fresh_env(torch_mod, maze_golden, textures, kind):
    """Per-episode task resampling: update_tasks() on a subset of slots (stream-ordered, no device sync) must leave the batch
    exactly where a fresh env with the final task table, reset on those envs, would be -- the untouched envs keep their
    episodes, the re-tasked envs restart, and every later step matches the oracle of each env's current task."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    pool = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                             g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(8)]
    N = 12
    if kind == "2D":
        env = BatchedMetaMaze2D(max_steps=30, task_type="SURVIVAL", view_grid=1, num_envs=N, squeeze=False)
        oras = [OracleMaze("2D", "SURVIVAL", 30, 1) for _ in range(N)]
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=(32, 24), max_steps=30, task_type="SURVIVAL", num_envs=N, squeeze=False,
                                        textures=textures, cache=False)
        oras = [OracleMaze("3D", "SURVIVAL", 30, 1, (32, 24), textures=textures) for _ in range(N)]
    cur = [pool[i % 4] for i in range(N)]                       # one table slot per env
    env.set_task(cur, env2task=np.arange(N))
    obs = env.reset().cpu().numpy()
    for i, o in enumerate(oras):
        o.set_task(cur[i])
        assert np.array_equal(obs[i], o.reset())
    rs = np.random.RandomState(4)
    for t in range(40):
        if t in (7, 8, 19, 33):                                  # re-task a few envs between steps, twice in a row too
            ids = rs.choice(N, size=4, replace=False)
            new = [pool[4 + int(rs.randint(4))] for _ in ids]
            env.update_tasks(ids, new)
            for i, nt in zip(ids, new):
                oras[i].set_task(nt)
                oras[i].reset()
        act = rs.randint(0, 4, size=N)
        obs, rew, done, _ = env.step(torch.as_tensor(act, dtype=torch.int32).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for i, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(act[i]))
            assert np.array_equal(obs[i], o2) and rew[i] == r2 and bool(done[i]) == d2, (t, i)
            if d2:
                o.reset()
        if done.any():
            env.reset(mask=torch.as_tensor(done).cuda())
    env.close()


@pytest.mark.parametrize("cache", [True, False])
def test_float32_observation_view_equals_int32(torch_mod, maze_golden, textures, cache):
    """obs_dtype='float32' (the dtype the reference's observation_space declares, maze_env.py:37-39) holds exactly the
    int32 values, on the pose-cache path, the direct renderer, reset() and the fused rollout."""
    torch = torch_mod
    c = maze_case(maze_golden, "m3d_surv")
    envs = [make_env(c, 3, textures, obs_dtype=dt, cache=cache) for dt in ("int32", "float32")]
    for e in envs:
        e.set_task(c["task"])
    o_i, o_f = [e.reset() for e in envs]
    assert o_f.dtype == torch.float32 and torch.equal(o_i.to(torch.float32), o_f)
    for t in range(25):
        act = torch.full((3,), int(c["act"][t]), dtype=torch.int32, device="cuda")
        o_i, o_f = [e.step(act)[0] for e in envs]
        assert torch.equal(o_i.to(torch.float32), o_f), t
    if cache:
        r_i, r_f = [e.rollout(4, act_seed=3)["obs"] for e in envs]
        assert torch.equal(r_i.to(torch.float32), r_f)
    for e in envs:
        e.close()


@pytest.mark.parametrize("kind", ["2D", "3D"])
def test_device_resampled_tasks_step_like_the_oracle(torch_mod, maze_golden, textures, kind):
    """Episodes on device-sampled tasks: after each resample_tasks(done) the re-tasked envs' tasks are read back and given to
    an oracle instance; every later observation / reward / done must match it bit for bit (the blobs the sampler writes are
    exactly what the step and render kernels consume)."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, MazeTaskSampler
    from oracle.maze_oracle import OracleMaze
    N = 10
    rs = np.random.RandomState(3)
    init = [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.3, food_density=0.05, food_interval=5, rng=rs) for _ in range(N)]
    if kind == "2D":
        env = BatchedMetaMaze2D(max_steps=12, task_type="SURVIVAL", view_grid=2, num_envs=N, squeeze=False)
        oras = [OracleMaze("2D", "SURVIVAL", 12, 2) for _ in range(N)]
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=(32, 32), max_steps=12, task_type="SURVIVAL", num_envs=N, squeeze=False,
                                        textures=textures, cache=False)
        oras = [OracleMaze("3D", "SURVIVAL", 12, 1, (32, 32), textures=textures) for _ in range(N)]
    env.set_task(init, env2task=np.arange(N))
    obs = env.reset().cpu().numpy()
    for i, o in enumerate(oras):
        o.set_task(init[i])
        assert np.array_equal(obs[i], o.reset())
    retasked = 0
    for t in range(40):
        act = rs.randint(0, 4, size=N)
        obs, rew, done, _ = env.step(torch.as_tensor(act, dtype=torch.int32).cuda())
        obs, rew, done_h = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for i, o in enumerate(oras):
            o2, r2, d2, _ = o.step(int(act[i]))
            assert np.array_equal(obs[i], o2) and rew[i] == r2 and bool(done_h[i]) == d2, (t, i)
        if done_h.any():
            env.resample_tasks(done, seed=21, allow_loops=True, crowd_ratio=0.3, food_density=0.05, food_interval=5)
            ids = np.nonzero(done_h)[0]
            for i, nt in zip(ids, env.get_tasks(ids)):
                oras[i].set_task(nt)
                oras[i].reset()
                retasked += 1
    assert retasked >= N
    env.close()


def test_config4_shape_properties(torch_mod, maze_golden, textures):
    """BASELINE config 4 shape per GPU (1024 envs, 15x15, 128x128, uint8): sharding invariance + determinism."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k], g["tasks15.scalars"][k]) for k in range(8)]
    N = 1024
    kw = dict(resolution=(128, 128), max_steps=200, task_type="SURVIVAL", squeeze=False, auto_reset=True,
              obs_dtype="uint8", textures=textures)
    full = BatchedMetaMazeDiscrete3D(num_envs=N, **kw)
    lo = BatchedMetaMazeDiscrete3D(num_envs=N // 2, env_index_base=0, **kw)
    hi = BatchedMetaMazeDiscrete3D(num_envs=N // 2, env_index_base=N // 2, **kw)
    for e in (full, lo, hi):
        e.set_task(tasks)
        e.reset()
    gen = torch.Generator(device="cuda").manual_seed(1)
    for t in range(6):
        act = torch.randint(0, 4, (N,), device="cuda", generator=gen, dtype=torch.int32)
        o, r, d, _ = full.step(act)
        o1, r1, d1, _ = lo.step(act[: N // 2])
        o2, r2, d2, _ = hi.step(act[N // 2:])
        assert torch.equal(o, torch.cat([o1, o2])) and torch.equal(r, torch.cat([r1, r2]))
        assert torch.equal(d, torch.cat([d1, d2]))
    # envs that share a task and received the same actions render the same image: env i and i+8 differ only by action
    assert int(o.max()) <= 255 and int(o.float().mean()) > 5
    for e in (full, lo, hi):
        e.close()


@pytest.mark.parametrize("res", [(256, 256), (320, 320), (320, 200)])
def test_reference_default_resolutions_vs_oracle(torch_mod, maze_golden, textures, res, render_path):
    """The reference registers 256x256 and defaults to 320x320 (metamaze/__init__.py:33-43, maze_env.py:20): screens
    whose per-column tables no longer fit shared memory next to the textures (hit lists spill to a global scratch)."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    task = task_from_arrays(g["tasks15.walls"][0], g["tasks15.texts"][0], g["tasks15.food"][0],
                            g["tasks15.interval"][0] // 20, g["tasks15.scalars"][0])
    env = BatchedMetaMazeDiscrete3D(resolution=res, max_steps=30, task_type="SURVIVAL", num_envs=2, squeeze=False,
                                    textures=textures)
    ora = OracleMaze("3D", "SURVIVAL", 30, 1, res, textures=textures)
    env.set_task(task)
    ora.set_task(task)
    assert np.array_equal(env.reset().cpu().numpy()[1], ora.reset())
    rng = np.random.RandomState(11)
    for t in range(8):
        a = int(rng.randint(4))
        obs, rew, done, _ = env.step(torch.full((2,), a, dtype=torch.int32, device="cuda"))
        o2, r2, d2, _ = ora.step(a)
        assert np.array_equal(obs.cpu().numpy()[0], o2), (t, int((obs.cpu().numpy()[0] != o2).sum()))
        assert float(rew[1]) == r2 and bool(done[1]) == d2
    env.close()


@pytest.mark.parametrize("name", ["c3d_surv", "c3d_esc", "gc3d"])
def test_continuous_maze_reference_episode(torch_mod, cont_golden, geom_golden, textures, name):
    """MetaMazeContinuous3D (SURVEY.md 8f row 2): reference episodes replayed on the GPU -- float32 positions, float64
    headings, cells, rewards, dones, life and every recorded frame bit for bit."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D
    from util import cont_case
    c = cont_case(geom_golden if name == "gc3d" else cont_golden, name)
    n = 3
    env = BatchedMetaMazeContinuous3D(resolution=c["resolution"], max_steps=c["max_steps"], task_type=c["task_type"],
                                      num_envs=n, squeeze=False, textures=textures)
    env.set_task(c["task"])
    obs0 = env.reset().cpu().numpy()
    assert np.array_equal(obs0[2], c["reset_obs"].astype(np.int32))
    kept = {int(t): k for k, t in enumerate(c["obs_idx"])}
    for t, a in enumerate(c["act"]):
        obs, rew, done, info = env.step(torch.as_tensor(np.tile(a, (n, 1))).cuda())
        pos, ori = env.pose()
        ag, life = env.agent_state()
        pos, ori, ag, life = pos.cpu().numpy(), ori.cpu().numpy(), ag.cpu().numpy(), life.cpu().numpy()
        for k in range(n):
            assert np.array_equal(pos[k], c["pos"][t]) and ori[k] == c["ori"][t], (t, pos[k], c["pos"][t], ori[k], c["ori"][t])
            assert float(rew[k]) == c["rew"][t] and bool(done[k]) == bool(c["done"][t]), t
            assert tuple(ag[k][:2]) == tuple(int(x) for x in c["grid"][t]) and int(ag[k][3]) == int(c["steps"][t])
            if c["task_type"] == "SURVIVAL":
                assert life[k] == c["life"][t]
        if t in kept:
            o = obs.cpu().numpy()
            ref = c["obs"][kept[t]].astype(np.int32)
            assert np.array_equal(o[0], ref) and np.array_equal(o[n - 1], ref), (t, int((o[0] != ref).sum()))
        if c["done"][t]:
            env.reset()
    env.close()


def test_continuous_maze_random_batch_vs_oracle(torch_mod, maze_golden, textures):
    """64 envs over 4 tasks, independent random float32 actions, auto-reset: every env equals its oracle instance."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(4)]
    n, T, max_steps, res = 64, 60, 25, (40, 24)
    env = BatchedMetaMazeContinuous3D(resolution=res, max_steps=max_steps, task_type="SURVIVAL", num_envs=n,
                                      squeeze=False, auto_reset=True, textures=textures)
    env.set_task(tasks)
    oracles = []
    for e in range(n):
        o = OracleMaze("C3D", "SURVIVAL", max_steps, 1, res, textures=textures)
        o.set_task(tasks[e % 4])
        oracles.append(o)
    obs = env.reset().cpu().numpy()
    for e in range(n):
        assert np.array_equal(obs[e], oracles[e].reset())
    rng = np.random.RandomState(17)
    for t in range(T):
        act = rng.uniform(-1.3, 1.3, (n, 2)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        pos, ori = env.pose()
        pos, ori = pos.cpu().numpy(), ori.cpu().numpy()
        for e in range(n):
            o2, r2, d2, _ = oracles[e].step(act[e])
            assert rew[e] == r2 and bool(done[e]) == d2, (t, e)
            if d2:
                o2 = oracles[e].reset()
            p2, a2 = oracles[e].pose
            assert np.array_equal(pos[e], p2) and ori[e] == a2, (t, e)
            assert np.array_equal(obs[e], o2), (t, e, int((obs[e] != o2).sum()))
    env.close()


@pytest.mark.parametrize("cache", [True, False])
def test_set_task_again_on_the_same_handle(torch_mod, maze_golden, textures, cache):
    """set_task() on a handle that already ran (the reference's meta-RL loop: sample_task / set_task / reset per
    episode, maze_env.py:44-57) rebuilds the task table and the pose cache -- every device table of the old cache is freed.
    The envs must behave exactly like a fresh handle given the second task list (use-after-rebuild regression)."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    g = maze_golden
    def tasks_of(ks):
        return [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                                 g["tasks15.interval"][k] // 20, g["tasks15.scalars"][k]) for k in ks]
    first, second = tasks_of([0, 1, 2, 3, 4, 5]), tasks_of([5, 3, 1])
    kw = dict(resolution=(128, 128), max_steps=40, squeeze=False, auto_reset=True, obs_dtype="uint8", textures=textures,
              num_envs=96, cache=None if cache else False)
    gen = torch.Generator(device="cuda").manual_seed(5)
    acts = torch.randint(0, 4, (30, 96), device="cuda", generator=gen, dtype=torch.int32)
    a = BatchedMetaMazeDiscrete3D(**kw)
    a.set_task(first); a.reset()
    for t in range(10):
        a.step(acts[t])
    a.set_task(second)                      # different table size: every cache array changes size and address
    b = BatchedMetaMazeDiscrete3D(**kw)
    b.set_task(second)
    assert torch.equal(a.reset(), b.reset())
    for t in range(30):
        o1, r1, d1, _ = a.step(acts[t])
        o2, r2, d2, _ = b.step(acts[t])
        assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2), t
    a.set_task(first); a.reset()            # and back again
    a.step(acts[0])
    torch.cuda.synchronize()
    a.close()
    b.close()


def test_handles_with_different_shared_memory_needs_interleave(torch_mod, maze_golden, textures):
    """Handles are independent: kernels' shared-memory opt-ins are device-wide properties, so a handle that needs little must
    not lower what a handle that needs a lot has set.  Big and small screens / view grids are stepped alternately and must
    reproduce what each gives when it runs alone."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(2)]
    acts = torch.randint(0, 4, (12, 8), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(3))

    def make(kind, arg):
        if kind == "3D":
            e = BatchedMetaMazeDiscrete3D(resolution=arg, max_steps=30, num_envs=8, squeeze=False, auto_reset=True,
                                          obs_dtype="uint8", textures=textures, cache=False)
        else:
            e = BatchedMetaMaze2D(max_steps=30, view_grid=arg, num_envs=8, squeeze=False, auto_reset=True)
        e.set_task(tasks)
        return e

    specs = [("3D", (256, 256)), ("3D", (32, 32)), ("2D", 6), ("2D", 1), ("3D", (128, 128))]
    alone = []
    for kind, arg in specs:
        e = make(kind, arg)
        frames = [e.reset().clone()] + [e.step(acts[t])[0].clone() for t in range(12)]
        alone.append(frames)
        e.close()
    envs = [make(kind, arg) for kind, arg in specs]
    for k in (0, 1, 2, 3, 4):                    # big first, then small: the small one must not shrink the big one's limit
        assert torch.equal(envs[k].reset(), alone[k][0])
    for t in range(12):
        for k in (1, 0, 3, 2, 4):
            assert torch.equal(envs[k].step(acts[t])[0], alone[k][t + 1]), (t, specs[k])
    for e in envs:
        e.close()


@pytest.mark.parametrize("cell_size", [0.5, 1.0, 2.0, 4.0, 8.0, 3.0, 1.25])
def test_direct_renderer_cell_size_family_vs_oracle(torch_mod, textures, cell_size):
    """The direct renderer's integer texel / cell index path is taken for power-of-two cell sizes >= text_size (1.0); smaller
    and non-power-of-two sizes take the reference expressions.  Each family member: 48 envs random-walk one sampled task
    for 50 steps (most free poses get visited), every frame against the env's own oracle instance, bit for bit."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D, MazeTaskSampler
    from oracle.maze_oracle import OracleMaze
    rs = np.random.RandomState(int(cell_size * 100))
    task = MazeTaskSampler(n=9, allow_loops=True, crowd_ratio=0.4, cell_size=cell_size, wall_height=1.6 * cell_size,
                           agent_height=0.8 * cell_size, food_density=0.05, food_interval=7, rng=rs)
    n, res, max_steps = 48, (48, 32), 30
    env = BatchedMetaMazeDiscrete3D(resolution=res, max_steps=max_steps, num_envs=n, squeeze=False, auto_reset=True,
                                    textures=textures, cache=False)
    env.set_task(task)
    oracles = []
    for e in range(n):
        o = OracleMaze("3D", "SURVIVAL", max_steps, 1, res, textures=textures)
        o.set_task(task)
        oracles.append(o)
    obs = env.reset().cpu().numpy()
    for e in range(n):
        assert np.array_equal(obs[e], oracles[e].reset())
    poses = set()
    for t in range(50):
        act = rs.randint(0, 4, n)
        obs, rew, done, _ = env.step(torch.as_tensor(act, dtype=torch.int32).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        ag = env.agent_state()[0].cpu().numpy() if hasattr(env, "agent_state") else None
        for e in range(n):
            o2, r2, d2, _ = oracles[e].step(int(act[e]))
            assert rew[e] == r2 and bool(done[e]) == d2, (t, e)
            if d2:
                o2 = oracles[e].reset()
            assert np.array_equal(obs[e], o2), (cell_size, t, e)
            if ag is not None:
                poses.add((int(ag[e][0]), int(ag[e][1]), int(ag[e][2])))
    if ag is not None:
        assert len(poses) >= 40, len(poses)
    env.close()


@pytest.mark.parametrize("kind", ["2D", "3D", "C3D"])
def test_maximum_maze_size_vs_oracle(torch_mod, textures, kind):
    """n = 31 cells per side (the engine's maximum; the reference's own smoke script grows n from 9 upwards,
    metamaze/test.py:17-26), dense food, tasks from the host sampler: GPU == oracle, bit for bit."""
    torch = torch_mod
    from metagym_b200 import (BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D,
                              MazeTaskSampler)
    from oracle.maze_oracle import OracleMaze
    rs = np.random.RandomState(31)
    task = MazeTaskSampler(n=31, allow_loops=True, crowd_ratio=0.3, food_density=0.03, food_interval=5, rng=rs)
    n, res = 4, (64, 40)
    if kind == "2D":
        env = BatchedMetaMaze2D(max_steps=80, view_grid=3, num_envs=n, squeeze=False)
    elif kind == "3D":
        env = BatchedMetaMazeDiscrete3D(resolution=res, max_steps=80, num_envs=n, squeeze=False, textures=textures)
    else:
        env = BatchedMetaMazeContinuous3D(resolution=res, max_steps=80, num_envs=n, squeeze=False, textures=textures)
    ora = OracleMaze(kind, "SURVIVAL", 80, 3, res, textures=textures if kind != "2D" else None)
    env.set_task(task)
    ora.set_task(task)
    assert np.array_equal(env.reset().cpu().numpy()[0], ora.reset())
    for t in range(40):
        if kind == "C3D":
            a = rs.uniform(-1, 1, 2).astype(np.float32)
            act = torch.as_tensor(np.tile(a, (n, 1))).cuda()
        else:
            a = int(rs.randint(4))
            act = torch.full((n,), a, dtype=torch.int32, device="cuda")
        obs, rew, done, _ = env.step(act)
        o2, r2, d2, _ = ora.step(a)
        assert np.array_equal(obs.cpu().numpy()[n - 1], o2), t
        assert float(rew[0]) == r2 and bool(done[0]) == d2
    env.close()


@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
@pytest.mark.parametrize("n,view_grid", [(300, 2), (77, 1), (128, 3)])
def test_fused_2d_rollout_equals_single_steps(torch_mod, maze_golden, task_type, n, view_grid):
    """mgb_maze_rollout (T steps, one launch) == T mgb_maze_step calls, bit for bit, auto-reset included; with
    device-drawn actions the drawn actions replayed through step() give the same trajectory; state hand-over between
    two consecutive rollouts and a following single step is exact."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMaze2D
    from oracle import philox
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(4)]
    T = 90

    def fresh():
        env = BatchedMetaMaze2D(max_steps=35, task_type=task_type, view_grid=view_grid, num_envs=n, squeeze=False,
                                auto_reset=True)
        env.set_task(tasks)
        env.reset()
        return env

    a_env, b_env = fresh(), fresh()
    rng = np.random.RandomState(n + view_grid)
    act = torch.as_tensor(rng.randint(0, 4, (T, n)), dtype=torch.int32).cuda()
    out = a_env.rollout(T, actions=act)
    n_done = 0
    for t in range(T):
        obs, rew, done, _ = b_env.step(act[t])
        assert torch.equal(out["obs"][t], obs), t
        assert torch.equal(out["rew"][t], rew), t
        assert torch.equal(out["done"][t].bool(), done.bool()), t
        n_done += int(done.sum())
    assert n_done > 0
    # device-drawn actions: two chunks, then one ordinary step
    o1 = a_env.rollout(40, act_seed=11, want_actions=True)
    o2 = a_env.rollout(25, act_seed=11, want_actions=True)
    drawn = torch.cat([o1["act"], o2["act"]])
    genv = a_env.env_index_base + np.arange(n)
    for t in range(65):          # the given-action rollout above advanced the step counter by T
        assert np.array_equal(drawn[t].cpu().numpy(), philox.maze_rollout_actions(11, genv, T + t)), t
    ref_obs = torch.cat([o1["obs"], o2["obs"]]); ref_rew = torch.cat([o1["rew"], o2["rew"]])
    for t in range(65):
        obs, rew, done, _ = b_env.step(drawn[t])
        assert torch.equal(ref_obs[t], obs) and torch.equal(ref_rew[t], rew), t
    last = torch.as_tensor(rng.randint(0, 4, n), dtype=torch.int32).cuda()
    ra, rb = a_env.step(last), b_env.step(last)
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])
    sa, sb = a_env.agent_state(), b_env.agent_state()
    assert torch.equal(sa[0], sb[0]) and torch.equal(sa[1], sb[1])
    a_env.close(); b_env.close()


@pytest.mark.parametrize("task_type,obs_dtype,res,n", [("SURVIVAL", "uint8", (64, 48), 37), ("SURVIVAL", "int32", (32, 32), 20),
                                                       ("ESCAPE", "uint8", (40, 24), 9), ("SURVIVAL", "uint8", (128, 128), 800)])
def test_fused_3d_rollout_equals_single_steps(torch_mod, maze_golden, textures, task_type, obs_dtype, res, n):
    """mgb_maze_rollout on MetaMazeDiscrete3D (one CTA per env, logic + compose per step, one launch) == T mgb_maze_step
    calls bit for bit: frames, rewards, dones, final agent state; given actions and device-drawn ones; more envs than
    resident CTAs (800 > 132 x 5 on an H100) exercises the env loop of a CTA."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    from oracle import philox
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(4)]
    T = 12 if n > 100 else 45

    def fresh():
        env = BatchedMetaMazeDiscrete3D(resolution=res, max_steps=20, task_type=task_type, num_envs=n, squeeze=False,
                                        auto_reset=True, obs_dtype=obs_dtype, textures=textures)
        env.set_task(tasks)
        env.reset()
        return env

    a_env, b_env = fresh(), fresh()
    rng = np.random.RandomState(n)
    act = torch.as_tensor(rng.randint(0, 4, (T, n)), dtype=torch.int32).cuda()
    out = a_env.rollout(T, actions=act)
    assert out["obs"].dtype == (torch.uint8 if obs_dtype == "uint8" else torch.int32)
    n_done = 0
    for t in range(T):
        obs, rew, done, _ = b_env.step(act[t])
        assert torch.equal(out["obs"][t], obs), t
        assert torch.equal(out["rew"][t], rew) and torch.equal(out["done"][t].bool(), done.bool()), t
        n_done += int(done.sum())
    assert n_done > 0 or n > 100
    o2 = a_env.rollout(7, act_seed=4, want_actions=True)
    genv = a_env.env_index_base + np.arange(n)
    for t in range(7):           # the given-action rollout above advanced the step counter by T
        assert np.array_equal(o2["act"][t].cpu().numpy(), philox.maze_rollout_actions(4, genv, T + t)), t
    for t in range(7):
        obs, rew, done, _ = b_env.step(o2["act"][t])
        assert torch.equal(o2["obs"][t], obs) and torch.equal(o2["rew"][t], rew), t
    sa, sb = a_env.agent_state(), b_env.agent_state()
    assert torch.equal(sa[0], sb[0]) and torch.equal(sa[1], sb[1])
    last = torch.as_tensor(rng.randint(0, 4, n), dtype=torch.int32).cuda()
    ra, rb = a_env.step(last), b_env.step(last)
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1])
    a_env.close(); b_env.close()
