"""snapshot() / restore() / clone_envs() of the quadrotor and the three mazes (metagym_b200/snapshot.py).  Every
comparison is bitwise: a restored handle must continue exactly like the handle the snapshot was taken from, in a fresh
handle, in place, in another sharding, for masked envs, after device re-tasking, through torch.save and from a CUDA graph.
The row-map builder and the ctypes bindings are tested without a GPU."""
import io

import numpy as np
import pytest

from util import task_from_arrays

gpu = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------------------------
# CPU: row maps and bindings
# ---------------------------------------------------------------------------------------------------------------


def test_row_map_matches_records_by_global_index():
    from metagym_b200.snapshot import build_row_map
    gi = np.array([13, 10, 11, 12, 14, 15])
    assert build_row_map(gi, 10, 4).tolist() == [1, 2, 3, 0]
    assert build_row_map(gi, 12, 4).tolist() == [3, 0, 4, 5]
    assert build_row_map(gi, 13, 3, mask=[True, False, True]).tolist() == [0, -1, 5]
    # masked-out envs need no record
    assert build_row_map(gi, 14, 4, mask=[1, 1, 0, 0]).tolist() == [4, 5, -1, -1]


def test_row_map_refusals():
    from metagym_b200.snapshot import build_row_map
    with pytest.raises(ValueError, match="does not cover"):
        build_row_map([0, 1, 2], 0, 4)
    with pytest.raises(ValueError, match="global index 5"):
        build_row_map([0, 1, 2], 3, 4, mask=[0, 0, 1, 0])
    with pytest.raises(ValueError, match="twice"):
        build_row_map([0, 1, 1, 2], 0, 3)
    with pytest.raises(ValueError, match="one entry per local env"):
        build_row_map([0, 1, 2], 0, 3, mask=[1, 1])


def test_clone_row_map():
    from metagym_b200.snapshot import clone_row_map
    assert clone_row_map([0, 0, 3], [1, 2, 0], 5).tolist() == [3, 0, 0, -1, -1]
    with pytest.raises(ValueError, match="twice"):
        clone_row_map([0, 1], [2, 2], 4)
    with pytest.raises(ValueError, match="outside"):
        clone_row_map([0, 4], [1, 2], 4)
    with pytest.raises(ValueError, match="same length"):
        clone_row_map([0, 1], [2], 4)


def test_bindings_of_the_snapshot_entry_points():
    import ctypes
    import __graft_entry__
    __graft_entry__.build()
    from metagym_b200 import _lib
    lib = _lib.load()
    for kind in ("quad", "maze"):
        assert getattr(lib, "mgb_%s_record_bytes" % kind).restype is _lib.c_i64
        assert getattr(lib, "mgb_%s_snapshot" % kind).argtypes == [_lib.vp] * 3
        assert getattr(lib, "mgb_%s_restore" % kind).argtypes == [_lib.vp, _lib.vp, _lib.c_i64, _lib.vp, _lib.vp]
        assert getattr(lib, "mgb_%s_counters" % kind).argtypes[1] is ctypes.POINTER(_lib.c_u64)
        # a null handle is refused without touching a device
        assert getattr(lib, "mgb_%s_record_bytes" % kind)(None) < 0
        assert getattr(lib, "mgb_%s_snapshot" % kind)(None, None, None) < 0
        assert getattr(lib, "mgb_%s_restore" % kind)(None, None, 0, None, None) < 0
        t = _lib.c_u64(0)
        assert getattr(lib, "mgb_%s_counters" % kind)(None, ctypes.byref(t), 0) < 0
        assert getattr(lib, "mgb_%s_fingerprint" % kind)(None, (_lib.c_u64 * 4)()) < 0


# ---------------------------------------------------------------------------------------------------------------
# GPU fixtures
# ---------------------------------------------------------------------------------------------------------------
QUAD_TASKS = ["no_collision", "hovering_control", "velocity_control"]
K1 = [("step", 25), ("roll", 30)]          # every env auto-resets (nt = 40) and rollout actions are drawn
K2 = [("step", 20), ("roll", 30)]          # ... and again


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def make_quad(task="velocity_control", n=64, base=0, **kw):
    from metagym_b200 import BatchedQuadrotor
    args = dict(task=task, dt=0.01, nt=40, seed=[1, 2, 3] if task == "velocity_control" else 0, num_envs=n,
                device=0, auto_reset=True, final_obs=True, rng_seed=7, env_index_base=base, squeeze=False)
    args.update(kw)
    return BatchedQuadrotor(**args)


def quad_actions(env, seed, n_global):
    lo, hi = env.action_space.low, env.action_space.high
    rs = np.random.RandomState(seed)
    return rs.uniform(lo, hi, size=(n_global, 4)).astype(np.float32)[env.env_index_base:env.env_index_base + env.num_envs]


def run_quad(env, plan, seed=0, n_global=None):
    """Outputs of a plan, each with the env axis first (numpy).  Terminal observations are kept where done only (zero
    elsewhere, also for a negative value: the comparison is bitwise)."""
    import torch
    n_global = n_global or env.num_envs
    out = []
    for i, (what, k) in enumerate(plan):
        if what == "step":
            for t in range(k):
                a = torch.from_numpy(quad_actions(env, 1000 * seed + 100 * i + t, n_global)).cuda()
                obs, rew, done, _ = env.step(a)
                d = done.cpu().numpy()
                out += [obs.cpu().numpy(), rew.cpu().numpy(), d, env.truncated.cpu().numpy(), env.fail_code.cpu().numpy(),
                        np.where(d[:, None], env.final_observation.cpu().numpy(), 0)]
        else:
            r = env.rollout(k, actions=None, act_seed=5 + i, want_actions=True)
            d = r["done"].cpu().numpy()
            fo = np.where(d[..., None], r["final_obs"].cpu().numpy(), 0)
            out += [np.swapaxes(x, 0, 1) for x in (r["obs"].cpu().numpy(), r["rew"].cpu().numpy(), d,
                                                   r["act"].cpu().numpy(), fo, r["truncated"].cpu().numpy())]
    return out


def same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and np.array_equal(np.ascontiguousarray(x).view(np.uint8),
                                                                                 np.ascontiguousarray(y).view(np.uint8))
                                    for x, y in zip(a, b))


def cat(parts):
    return [np.concatenate(xs, axis=0) for xs in zip(*parts)]


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


@pytest.fixture(scope="module")
def maze_tasks(maze_golden):
    """Four 15x15 tasks with food on every third free cell and a respawn interval of 4 steps, so that food is eaten and
    grows back inside a test window."""
    g = maze_golden
    out = []
    for j in range(4):
        t = task_from_arrays(g["tasks15.walls"][j], g["tasks15.texts"][j], g["tasks15.food"][j],
                             g["tasks15.interval"][j], g["tasks15.scalars"][j])
        w = np.asarray(t.cell_walls)
        ii, jj = np.meshgrid(np.arange(15), np.arange(15), indexing="ij")
        food = np.where((w == 0) & ((ii + jj) % 3 == 0), 0.2, 0.0)
        food[tuple(t.start)] = 0.0
        out.append(t._replace(food_rewards=food, food_interval=np.where(food > 0, 4, 0).astype(np.int32),
                              step_reward=-0.05, initial_life=1.0, max_life=2.0))
    return out


MAZES = {   # name -> (class, constructor kwargs, has a fused rollout)
    "2d_surv": ("BatchedMetaMaze2D", dict(task_type="SURVIVAL", max_steps=30, view_grid=2), True),
    "2d_esc": ("BatchedMetaMaze2D", dict(task_type="ESCAPE", max_steps=30, view_grid=1), True),
    "d3_cache": ("BatchedMetaMazeDiscrete3D", dict(task_type="SURVIVAL", max_steps=30, resolution=(32, 24),
                                                   obs_dtype="uint8", cache=True), True),
    "d3_direct": ("BatchedMetaMazeDiscrete3D", dict(task_type="SURVIVAL", max_steps=30, resolution=(24, 16),
                                                    obs_dtype="int32", cache=False), False),
    "c3": ("BatchedMetaMazeContinuous3D", dict(task_type="SURVIVAL", max_steps=30, resolution=(16, 16),
                                               obs_dtype="uint8"), True),
}


def make_maze(name, tasks, textures, n=24, base=0, env2task=None, **kw):
    from metagym_b200 import metamaze
    cls, args, _ = MAZES[name]
    args = dict(args, num_envs=n, device=0, auto_reset=True, final_obs=True, env_index_base=base, squeeze=False)
    if cls != "BatchedMetaMaze2D":
        args["textures"] = textures
    args.update(kw)
    env = getattr(metamaze, cls)(**args)
    env.set_task(tasks, env2task=env2task)
    return env


def maze_actions(env, seed, n_global):
    rs = np.random.RandomState(seed)
    b, n = env.env_index_base, env.num_envs
    if env.KIND == 2:
        return rs.uniform(-1, 1, size=(n_global, 2)).astype(np.float32)[b:b + n]
    return rs.randint(0, 4, size=n_global).astype(np.int32)[b:b + n]


def run_maze(env, plan, seed=0, n_global=None, roll=True):
    import torch
    n_global = n_global or env.num_envs
    out = []
    for i, (what, k) in enumerate(plan):
        if what == "step" or not roll:
            for t in range(k):
                a = torch.from_numpy(maze_actions(env, 1000 * seed + 100 * i + t, n_global)).cuda()
                obs, rew, done, _ = env.step(a)
                d = done.cpu().numpy()
                fo = env.final_observation.cpu().numpy()
                out += [obs.cpu().numpy(), rew.cpu().numpy(), d, env.truncated.cpu().numpy(),
                        np.where(d.reshape((-1,) + (1,) * (fo.ndim - 1)), fo, 0)]
        else:
            kw = {} if env.KIND == 0 else {"final_obs": True}
            r = env.rollout(k, actions=None, act_seed=5 + i, want_actions=True, **kw)
            d = r["done"].cpu().numpy()
            fo = r["final_obs"].cpu().numpy()
            fo = np.where(d.reshape(d.shape + (1,) * (fo.ndim - 2)), fo, 0)
            out += [np.swapaxes(x, 0, 1) for x in (r["obs"].cpu().numpy(), r["rew"].cpu().numpy(), d,
                                                   r["act"].cpu().numpy(), fo, r["truncated"].cpu().numpy())]
    return out


# ---------------------------------------------------------------------------------------------------------------
# 1. resume in a fresh handle
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("task", QUAD_TASKS)
def test_quad_resume_in_fresh_handle(torch_mod, task):
    a = make_quad(task)
    a.reset()
    run_quad(a, K1, seed=1)
    snap = a.snapshot()
    sd = a.state_dict()
    assert (snap["records"].view(torch_mod.int32)[:, 23] > 0).all()       # every env has auto-reset (episode counter)
    assert int(snap["counters"][0]) == 30                                  # rollout actions were drawn
    ref = run_quad(a, K2, seed=2)
    b = make_quad(task)
    b.restore(snap)
    assert same(run_quad(b, K2, seed=2), ref)
    # control: the existing state_dict leaves episode counter and rollout action counter behind
    c = make_quad(task)
    c.load_state_dict(sd)
    assert not same(run_quad(c, K2, seed=2), ref)
    if task == "velocity_control":
        assert torch_mod.equal(b.env2task, a.env2task)


@gpu
@pytest.mark.parametrize("name", sorted(MAZES))
def test_maze_resume_in_fresh_handle(torch_mod, name, maze_tasks, textures):
    roll = MAZES[name][2]
    a = make_maze(name, maze_tasks, textures)
    a.reset()
    run_maze(a, K1, seed=1, roll=roll)
    snap = a.snapshot()
    ref = run_maze(a, K2, seed=2, roll=roll)
    if name in ("2d_surv", "d3_cache", "d3_direct"):      # food was eaten in the window (rewards: the float64 outputs)
        assert any((x > 0).any() for x in ref if x.dtype == np.float64)
    b = make_maze(name, maze_tasks, textures)             # fresh: set_task, no reset()
    b.restore(snap)
    assert not b.need_reset
    assert same(run_maze(b, K2, seed=2, roll=roll), ref)


# ---------------------------------------------------------------------------------------------------------------
# 2. in-place rewind
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_in_place_rewind(torch_mod, maze_tasks, textures):
    q = make_quad("hovering_control")
    q.reset()
    run_quad(q, K1, seed=1)
    snap = q.snapshot()
    ref = run_quad(q, K2, seed=2)
    q.restore(snap)
    assert same(run_quad(q, K2, seed=2), ref)
    m = make_maze("2d_surv", maze_tasks, textures)
    m.reset()
    run_maze(m, K1, seed=1)
    snap = m.snapshot()
    ref = run_maze(m, K2, seed=2)
    m.restore(snap)
    assert same(run_maze(m, K2, seed=2), ref)


# ---------------------------------------------------------------------------------------------------------------
# 3. resharding
# ---------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kind", ["quad", "d3_cache"])
def test_resharding_both_ways(torch_mod, kind, maze_tasks, textures):
    N = 64 if kind == "quad" else 24
    if kind == "quad":
        make = lambda n, base: make_quad("velocity_control", n=n, base=base)        # noqa: E731
        run = lambda env, plan, seed: run_quad(env, plan, seed, n_global=N)          # noqa: E731
    else:
        make = lambda n, base: make_maze(kind, maze_tasks, textures, n=n, base=base)  # noqa: E731
        run = lambda env, plan, seed: run_maze(env, plan, seed, n_global=N)          # noqa: E731
    # one handle -> two shards
    one = make(N, 0)
    one.reset()
    run(one, K1, 1)
    snap = one.snapshot()
    ref = run(one, K2, 2)
    shards = [make(N // 2, 0), make(N // 2, N // 2)]
    for s in shards:
        s.restore(snap)
    assert same(cat([run(s, K2, 2) for s in shards]), ref)
    # two shards -> one handle, from the list of both snapshots
    shards = [make(N // 2, 0), make(N // 2, N // 2)]
    for s in shards:
        s.reset()
        run(s, K1, 3)
    snaps = [s.snapshot() for s in shards]
    ref = cat([run(s, K2, 4) for s in shards])
    one = make(N, 0)
    one.restore(snaps[::-1])
    assert same(run(one, K2, 4), ref)


# ---------------------------------------------------------------------------------------------------------------
# 4. masked restore
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_masked_restore(torch_mod):
    a, twin = make_quad("hovering_control"), make_quad("hovering_control")
    for e in (a, twin):
        e.reset()
        run_quad(e, K1, seed=1)
    snap = a.snapshot()
    for e in (a, twin):
        run_quad(e, [("step", 17)], seed=5)
    mask = np.arange(64) % 3 == 0
    t_base = a._counters()
    a.restore(snap, mask=torch_mod.from_numpy(mask).cuda())
    assert a._counters() == t_base                        # a masked restore leaves the counters alone
    cont = make_quad("hovering_control")
    cont.restore(snap)
    plan = [("step", 30)]
    out, out_twin, out_cont = run_quad(a, plan, 6), run_quad(twin, plan, 6), run_quad(cont, plan, 6)
    assert same([x[~mask] for x in out], [x[~mask] for x in out_twin])
    assert same([x[mask] for x in out], [x[mask] for x in out_cont])


# ---------------------------------------------------------------------------------------------------------------
# 5. clone_envs
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_clone_envs_quad_across_tasks(torch_mod):
    env = make_quad("velocity_control", n=16, nt=400)
    env.reset()
    run_quad(env, [("step", 5)], seed=1)
    src, dst = np.array([0, 1, 5]), np.array([4, 8, 7])
    assert (env.env2task.cpu().numpy()[src] != env.env2task.cpu().numpy()[dst]).all()
    env.clone_envs(src, dst)
    e2t = env.env2task.cpu().numpy()
    assert (e2t[dst] == e2t[src]).all()
    for t in range(10):
        a = quad_actions(env, t, 16)
        a[dst] = a[src]
        obs, rew, done, _ = env.step(torch_mod.from_numpy(a).cuda())
        o, r, d = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        assert not d.any()
        assert np.array_equal(o[dst], o[src]) and np.array_equal(r[dst], r[src])


@gpu
@pytest.mark.parametrize("per_env", [False, True])
def test_clone_envs_maze_across_slots(torch_mod, maze_tasks, textures, per_env):
    n = 8
    tasks = [maze_tasks[k % 4] for k in range(n)] if per_env else maze_tasks
    env = make_maze("2d_surv", tasks, textures, n=n, env2task=np.arange(n) if per_env else None, max_steps=1000)
    env.reset()
    run_maze(env, [("step", 3)], seed=1)
    src, dst = np.array([0, 2]), np.array([1, 7])
    env.clone_envs(src, dst)
    if per_env:      # the task was copied into the destination env's own slot
        assert (env.env2task == np.arange(n)).all()
        got = env.get_tasks(dst)
        for k, s in enumerate(src):
            assert np.array_equal(got[k].cell_walls, np.asarray(tasks[s].cell_walls)) and got[k].start == tuple(tasks[s].start)
    else:
        assert (env.env2task[dst] == env.env2task[src]).all()
    for t in range(6):
        a = maze_actions(env, t, n)
        a[dst] = a[src]
        obs, rew, done, _ = env.step(torch_mod.from_numpy(a).cuda())
        o, r, d = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        assert not d.any()
        assert np.array_equal(o[dst], o[src]) and np.array_equal(r[dst], r[src])


# ---------------------------------------------------------------------------------------------------------------
# 6. re-tasked mazes
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_restore_after_device_resampling(torch_mod, maze_tasks, textures):
    n = 8
    tasks = [maze_tasks[k % 4] for k in range(n)]
    a = make_maze("d3_direct", tasks, textures, n=n, env2task=np.arange(n))
    a.reset()
    run_maze(a, [("step", 6)], seed=1, roll=False)
    a.resample_tasks(mask=torch_mod.tensor([1, 0, 1, 1, 0, 0, 1, 0], dtype=torch_mod.uint8).cuda(), seed=3)
    run_maze(a, [("step", 4)], seed=2, roll=False)
    snap = a.snapshot()
    assert int(snap["fingerprint"][3]) == 1                       # the records carry their tasks
    ref = run_maze(a, [("step", 12)], seed=3, roll=False)
    b = make_maze("d3_direct", tasks, textures, n=n, env2task=np.arange(n))      # the ORIGINAL tasks
    b.restore(snap)
    assert same(run_maze(b, [("step", 12)], seed=3, roll=False), ref)
    for x, y in zip(b.get_tasks(range(n)), a.get_tasks(range(n))):
        assert all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(x, y))
    assert not all(np.array_equal(x.cell_walls, np.asarray(t.cell_walls)) for x, t in zip(b.get_tasks(range(n)), tasks))


# ---------------------------------------------------------------------------------------------------------------
# 7. refusals
# ---------------------------------------------------------------------------------------------------------------
def step_once(env, seed):
    import torch
    if hasattr(env, "velocity_targets"):
        return env.step(torch.from_numpy(quad_actions(env, seed, env.num_envs)).cuda())[0].cpu().numpy()
    return env.step(torch.from_numpy(maze_actions(env, seed, env.num_envs)).cuda())[0].cpu().numpy()


@gpu
def test_refusals_leave_the_handle_untouched(torch_mod, maze_tasks, textures):
    src = make_quad("velocity_control", n=16)
    src.reset()
    run_quad(src, [("step", 7)], seed=1)
    snap = src.snapshot()
    for kw in (dict(dt=0.02), dict(rng_seed=8), dict(seed=[1, 2, 4])):
        dst, twin = make_quad("velocity_control", n=16, **kw), make_quad("velocity_control", n=16, **kw)
        dst.reset()
        twin.reset()
        with pytest.raises(ValueError, match="incompatible"):
            dst.restore(snap)
        assert np.array_equal(step_once(dst, 3), step_once(twin, 3))
    msrc = make_maze("d3_direct", maze_tasks, textures, n=6)
    msrc.reset()
    snap = msrc.snapshot()
    from metagym_b200.textures import synthetic_textures
    for res, tex, tasks in (((24, 18), textures, maze_tasks), ((24, 16), synthetic_textures(seed=1), maze_tasks),
                            ((24, 16), textures, maze_tasks[::-1])):
        dst, twin = [make_maze("d3_direct", tasks, tex, n=6, resolution=res) for _ in range(2)]
        dst.reset()
        twin.reset()
        with pytest.raises(ValueError, match="incompatible"):
            dst.restore(snap)
        assert np.array_equal(step_once(dst, 3), step_once(twin, 3))
    with pytest.raises(ValueError, match="quadrotor"):
        make_maze("d3_direct", maze_tasks, textures, n=6).restore(make_quad(n=6).snapshot())
    # a refused set_task: a table with more food cells (a new layout) and a texture id no loaded texture has
    from metagym_b200._lib import MgbError
    dst, twin = [make_maze("d3_direct", maze_tasks, textures, n=6) for _ in range(2)]
    dst.reset()
    twin.reset()
    t = maze_tasks[0]
    food = np.where(np.asarray(t.cell_walls) == 0, 0.3, 0.0)
    texts = np.asarray(t.cell_texts).copy()
    texts[0, 0] = 15                                       # n_tex <= 15
    with pytest.raises(MgbError, match="texture that is not loaded"):
        dst.set_task([t._replace(food_rewards=food, cell_texts=texts)])
    assert np.array_equal(dst._fingerprint(), twin._fingerprint()) and dst._record_bytes() == twin._record_bytes()
    act = torch_mod.from_numpy(maze_actions(dst, 3, 6)).cuda()
    assert same(*[[x.cpu().numpy() for x in env.step(act)[:3]] for env in (dst, twin)])
    # a refused quadrotor map (two start cells) keeps the map the handle has
    dst, twin = make_quad("hovering_control", n=16), make_quad("hovering_control", n=16)
    grid = np.zeros((6, 6), dtype=np.int32)
    grid[2, 3], grid[4, 1] = -1, 1
    for env in (dst, twin):
        assert env._lib.mgb_quad_set_map(env._h, grid.ctypes.data, 6, 6) == 0
        env.reset()
    bad = grid.copy()
    bad[0, 0] = -1
    assert dst._lib.mgb_quad_set_map(dst._h, bad.ctypes.data, 6, 6) < 0
    assert dst._fingerprint()[1] == twin._fingerprint()[1] != 0
    assert np.array_equal(step_once(dst, 3), step_once(twin, 3))


# ---------------------------------------------------------------------------------------------------------------
# 8. serialisation and capture
# ---------------------------------------------------------------------------------------------------------------
@gpu
def test_torch_save_round_trip_and_cuda_graph(torch_mod, maze_tasks, textures):
    torch = torch_mod
    for make, run in ((lambda: make_quad("velocity_control"), run_quad),
                      (lambda: make_maze("d3_cache", maze_tasks, textures), run_maze)):
        a = make()
        a.reset()
        run(a, K1, seed=1)
        buf = io.BytesIO()
        torch.save(a.snapshot(), buf)
        ref = run(a, K2, seed=2)
        buf.seek(0)
        snap = torch.load(buf, map_location="cpu")
        assert snap["records"].device.type == "cpu"
        b = make()
        b.restore(snap)
        assert same(run(b, K2, seed=2), ref)
        # snapshot(out=...) in a CUDA graph
        s = a.snapshot()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            a.snapshot(out=s)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            a.snapshot(out=s)
        run(a, [("step", 3)], seed=3)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(s["records"], a.snapshot()["records"])
