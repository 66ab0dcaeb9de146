"""GPU tests of path recording and the trajectory picture (mgb_maze_set_path / mgb_maze_path, MGB_GOD_TRAJECTORY;
record_path=True, trajectory(), god_view(trajectory=True) and save_trajectory() of the three MetaMaze classes): paths and
pictures against the unmodified reference's recorded episodes (tests/golden/maze_trajectory_golden.npz) and against
OracleMaze through resets; every entry point records what single steps record; recording changes no other output;
snapshots carry paths; the step limit; PNG files; refusals and CUDA-graph capture."""
import os

import numpy as np
import pytest

import trajectory_view as tv
from test_maze_trajectory_oracle import CASES, _decode_png, path_at, recorded
from util import task_from_arrays

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
KINDS = {0: "2D", 1: "3D", 2: "C3D"}


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def case_task(d):
    return task_from_arrays(d["task.walls"], d["task.texts"], d["task.food"], d["task.interval"], d["task.scalars"])


def make_env(kind, num_envs, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    kw = dict(dict(max_steps=1000, task_type="SURVIVAL", num_envs=num_envs, squeeze=False, record_path=True), **kw)
    if kind == 0:
        return BatchedMetaMaze2D(view_grid=2, **kw)
    cls = BatchedMetaMazeDiscrete3D if kind == 1 else BatchedMetaMazeContinuous3D
    return cls(resolution=(8, 8), obs_dtype="uint8", **kw)


def paths(env, envs=None):
    """trajectory() -> list of [L, 2] int arrays, checking the -1 padding."""
    cells, lens = env.trajectory(envs)
    cells, lens = cells.cpu().numpy(), lens.cpu().numpy()
    assert cells.shape[1] == env.max_steps + 1
    for k in range(len(lens)):
        assert (cells[k, lens[k]:] == -1).all()
    return [cells[k, :lens[k]] for k in range(len(lens))]


def rand_actions(torch, kind, rng, n):
    if kind == 2:
        a = np.stack([rng.uniform(-0.4, 0.4, n), rng.uniform(0.2, 1.0, n)], -1).astype(np.float32)
        return a, torch.as_tensor(a).cuda()
    a = rng.randint(0, 4, n).astype(np.int32)
    return a, torch.as_tensor(a).cuda()


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_replay_equals_the_reference(torch_mod, d):
    """Replay the recorded episode on a two-env batch (twins): at every recorded step trajectory() is the reference's
    _agent_trajectory and god_view(trajectory=True) is the raster of the primitives render_trajectory drew."""
    torch = torch_mod
    kind, tt, n, S, max_steps = (int(v) for v in d["meta"])
    env = make_env(kind, 2, task_type=("SURVIVAL", "ESCAPE")[tt], render_scale=S, max_steps=max_steps)
    env.set_task(case_task(d))
    env.reset()
    frames = [int(f) for f in d["frames"]]
    act = d["act"]
    for t in range(frames[-1] + 1):
        if t in frames:
            f = frames.index(t)
            want_path = path_at(d, f)
            for p in paths(env):
                assert np.array_equal(p, want_path), (d["name"], t)
            want = tv.rasterise(recorded(d, f), S)
            got = env.god_view(trajectory=True).cpu().numpy()
            for e in range(2):
                bad = np.argwhere((got[e] != want).any(-1))
                assert bad.size == 0, (d["name"], t, e, bad[:5].tolist(), got[e][tuple(bad[0])].tolist(),
                                       want[tuple(bad[0])].tolist())
        if t == frames[-1]:
            break
        if kind == 2:
            a = torch.as_tensor(np.stack([act[t], act[t]]), device=env.device)
        else:
            a = torch.full((2,), int(act[t]), dtype=torch.int32, device=env.device)
        env.step(a)
    env.close()


def _oracle_tasks(kind):
    return [case_task(d) for d in CASES if int(d["meta"][0]) == kind and int(d["meta"][2]) == 9]


@pytest.mark.parametrize("auto_reset", [True, False])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_random_batches_follow_the_oracle_through_resets(torch_mod, textures, kind, auto_reset):
    """Each env's path is the cell sequence of its own OracleMaze since its last reset: auto-resets, or (auto_reset off)
    masked resets of the finished envs."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    tasks = _oracle_tasks(kind)
    N, T, max_steps = 40, 70, 18
    env = make_env(kind, N, max_steps=max_steps, auto_reset=auto_reset)
    env.set_task(tasks)
    env.reset()
    oracles, want = [], []
    for e in range(N):
        o = OracleMaze(KINDS[kind], "SURVIVAL", max_steps, 2, (8, 8), textures=textures if kind else None)
        o.set_task(tasks[int(env.env2task[e])])
        o.reset()
        oracles.append(o)
        want.append([o.agent[:2]])
    rng = np.random.RandomState(5 + kind)
    resets = 0
    for t in range(T):
        a, a_dev = rand_actions(torch, kind, rng, N)
        _, _, done, _ = env.step(a_dev)
        done = done.cpu().numpy()
        for e in range(N):
            _, _, dn, _ = oracles[e].step(a[e], render=False)
            assert dn == bool(done[e]), (t, e)
            want[e].append(oracles[e].agent[:2])
            if dn and auto_reset:
                oracles[e].reset()
                want[e] = [oracles[e].agent[:2]]
        got = paths(env)
        for e in range(N):
            assert np.array_equal(got[e], np.asarray(want[e])), (kind, t, e)
        if not auto_reset and done.any():
            env.reset(mask=done)
            for e in np.nonzero(done)[0]:
                oracles[e].reset()
                want[e] = [oracles[e].agent[:2]]
        resets += int(done.sum())
    assert resets > N
    env.close()


def _drive(env, kind, acts, how):
    """Step env through acts [T, N(, 2)] with single steps or one rollout."""
    torch = env._torch
    if how == "step":
        for a in acts:
            env.step(torch.as_tensor(a).cuda())
    else:
        kw = {} if kind == 0 else {"final_obs": how == "rollout_fin"}
        env.rollout(len(acts), actions=torch.as_tensor(np.stack(acts)).cuda(), **kw)


ENTRY = [(0, "rollout", {}), (0, "rollout_fin", {"final_obs": True}), (0, "step", {"final_obs": True}),
         (1, "rollout", {}), (1, "rollout_fin", {}), (1, "step", {"final_obs": True}),
         (1, "step", {"cache": False}), (1, "step", {"cache": False, "final_obs": True}),
         (2, "rollout", {}), (2, "rollout_fin", {}), (2, "step", {"final_obs": True})]


@pytest.mark.parametrize("kind,how,kw", ENTRY, ids=["%s-%s-%s" % (KINDS[k], h, "-".join(sorted(kw))) for k, h, kw in ENTRY])
def test_every_entry_point_records_like_single_steps(torch_mod, kind, how, kw):
    """step / step_ex on every 3-D renderer and the 2-D / pose-cache / continuous rollouts, with and without terminal
    observations, leave the same paths and state as plain single steps of the same actions through auto-resets."""
    torch = torch_mod
    tasks = _oracle_tasks(kind)
    N, T = 48, 40
    base = dict(max_steps=15, auto_reset=True)
    env = make_env(kind, N, **dict(base, **kw))
    ref = make_env(kind, N, **dict(base, cache=kw.get("cache")) if kind else base)
    for e in (env, ref):
        e.set_task(tasks)
        e.reset()
    rng = np.random.RandomState(21)
    acts = [rand_actions(torch, kind, rng, N)[0] for _ in range(T)]
    _drive(env, kind, acts, how)
    _drive(ref, kind, acts, "step")
    for x, y in zip(paths(env), paths(ref)):
        assert np.array_equal(x, y)
    assert torch.equal(env.agent_state()[0], ref.agent_state()[0])
    env.close()
    ref.close()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_masked_reset_update_and_resample_restart_paths(torch_mod, kind):
    """A masked reset, update_tasks and resample_tasks each leave a restarted env with the one-cell path [start]; other
    envs keep theirs."""
    torch = torch_mod
    tasks = _oracle_tasks(kind)
    N = 12
    env = make_env(kind, N, max_steps=200, cache=False) if kind else make_env(kind, N, max_steps=200)
    env.set_task([tasks[e % len(tasks)] for e in range(N)], env2task=np.arange(N))
    env.reset()
    rng = np.random.RandomState(3)
    for _ in range(6):
        env.step(rand_actions(torch, kind, rng, N)[1])
    before = paths(env)
    assert all(len(p) == 7 for p in before)

    def check(restarted):
        got = paths(env)
        ag = env.agent_state()[0].cpu().numpy()
        for e in range(N):
            if e in restarted:
                assert len(got[e]) == 1 and tuple(got[e][0]) == tuple(ag[e, :2]), e
            else:
                assert np.array_equal(got[e], before[e]), e

    mask = np.zeros(N, np.uint8)
    mask[[1, 4]] = 1
    env.reset(mask=mask)
    check({1, 4})
    for e in (1, 4):
        before[e] = paths(env)[e]
    env.update_tasks([7], tasks[0])
    check({1, 4, 7})
    assert tuple(paths(env)[7][0]) == tuple(tasks[0].start)
    before[7] = paths(env)[7]
    m = torch.zeros(N, dtype=torch.uint8, device="cuda")
    m[[2, 9]] = 1
    env.resample_tasks(m, seed=4, cell_size=2.0)
    check({1, 4, 7, 2, 9})
    env.close()


@pytest.mark.parametrize("kind,kw", [(0, {}), (0, {"final_obs": True}), (1, {}), (1, {"cache": False}),
                                     (1, {"final_obs": True}), (2, {}), (2, {"final_obs": True})])
def test_recording_changes_no_other_output(torch_mod, kind, kw):
    torch = torch_mod
    tasks = _oracle_tasks(kind)
    N = 40
    on = make_env(kind, N, max_steps=12, auto_reset=True, **kw)
    off = make_env(kind, N, max_steps=12, auto_reset=True, record_path=False, **kw)
    on.set_task(tasks)
    off.set_task(tasks)
    assert torch.equal(on.reset(), off.reset())
    rng = np.random.RandomState(8)
    for t in range(30):
        a = rand_actions(torch, kind, rng, N)[1]
        x, y = on.step(a), off.step(a)
        for u, v in zip(x[:3], y[:3]):
            assert torch.equal(u, v), t
        if kw.get("final_obs"):
            assert torch.equal(on.final_observation, off.final_observation)
            assert torch.equal(on.truncated, off.truncated)
    if kind != 1 or kw.get("cache") is None:
        acts = torch.as_tensor(np.stack([rand_actions(torch, kind, rng, N)[0] for _ in range(9)])).cuda()
        x, y = on.rollout(9, actions=acts), off.rollout(9, actions=acts)
        for k in ("obs", "rew", "done"):
            assert torch.equal(x[k], y[k]), k
    for u, v in zip(on.agent_state(), off.agent_state()):
        assert torch.equal(u, v)
    assert torch.equal(on.god_view(), off.god_view())
    on.close()
    off.close()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_snapshot_restore_and_clone_carry_paths(torch_mod, kind):
    torch = torch_mod
    tasks = _oracle_tasks(kind)
    N = 10
    env = make_env(kind, N, max_steps=300)
    env.set_task(tasks)
    env.reset()
    rng = np.random.RandomState(2)
    for _ in range(9):
        env.step(rand_actions(torch, kind, rng, N)[1])
    snap = env.snapshot()
    want = paths(env)
    view = env.god_view(trajectory=True)
    for _ in range(5):
        env.step(rand_actions(torch, kind, rng, N)[1])
    env.restore(snap)
    for x, y in zip(paths(env), want):
        assert np.array_equal(x, y)
    assert torch.equal(env.god_view(trajectory=True), view)
    env.step(rand_actions(torch, kind, rng, N)[1])
    env.clone_envs([0, 5], [3, 8])
    got = paths(env)
    assert np.array_equal(got[3], got[0]) and np.array_equal(got[8], got[5]) and len(got[3]) == 11
    # a record of a recording handle does not fit a handle without recording, and the reverse
    other = make_env(kind, N, max_steps=300, record_path=False)
    other.set_task(tasks)
    other.reset()
    with pytest.raises(ValueError, match="path recording"):
        other.restore(snap)
    with pytest.raises(ValueError, match="path recording"):
        env.restore(other.snapshot())
    env.close()
    other.close()


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_steps_past_the_limit_are_not_stored(torch_mod, textures, kind):
    """auto_reset off, stepped on after the step limit: the path keeps its max_steps + 1 cells."""
    torch = torch_mod
    from oracle.maze_oracle import OracleMaze
    tasks = _oracle_tasks(kind)[:1]
    env = make_env(kind, 3, max_steps=10, task_type="ESCAPE", auto_reset=False)
    env.set_task(tasks)
    env.reset()
    o = OracleMaze(KINDS[kind], "ESCAPE", 10, 2, (8, 8), textures=textures if kind else None)
    o.set_task(tasks[0])
    o.reset()
    want = [o.agent[:2]]
    rng = np.random.RandomState(1)
    for t in range(16):
        a, _ = rand_actions(torch, kind, rng, 1)
        env.step(torch.as_tensor(np.repeat(a, 3, 0)).cuda())
        o.step(a[0], render=False)
        want.append(o.agent[:2])
    ag = env.agent_state()[0].cpu().numpy()
    assert (ag[:, 3] == 16).all()
    for p in paths(env):
        assert np.array_equal(p, np.asarray(want[:11]))
    env.god_view(trajectory=True)
    env.close()


@pytest.mark.parametrize("kind,n,S", [(0, 21, 500), (1, 15, 480), (2, 9, 500)])
def test_any_path_is_drawn_exactly(torch_mod, kind, n, S):
    """A path of arbitrary cells (long and diagonal jumps, neighbour steps, repeats) written into snapshot records and
    restored: trajectory() returns it and god_view(trajectory=True) equals the raster of its primitives."""
    torch = torch_mod
    d = [d for d in CASES if tuple(int(v) for v in d["meta"][[0, 1, 2]]) == (kind, 1, n)][0]
    task = case_task(d)
    N, L, cap = 4, 70, 301
    env = make_env(kind, N, task_type="ESCAPE", max_steps=cap - 1, render_scale=S)
    env.set_task(task)
    env.reset()
    snap = env.snapshot()
    rec = snap["records"].cpu().numpy().copy()
    off = rec.shape[1] - (2 * cap + 15) // 16 * 16
    rng = np.random.RandomState(kind)
    want = []
    for e in range(N):
        p = [rng.randint(0, n, 2)]
        for i in range(L - 1):
            r = rng.rand()
            step = rng.randint(0, n, 2) if r < 0.4 else (p[-1] if r < 0.5 else p[-1] + rng.randint(-1, 2, 2))
            p.append(np.clip(step, 0, n - 1))
        p = np.asarray(p, np.int8)
        want.append(p.astype(np.int64))
        rec[e, off:off + 2 * L] = p.reshape(-1).view(np.uint8)
        rec[e, 12:16] = np.array([L - 1], np.int32).view(np.uint8)        # steps: the path's last entry
    snap["records"] = torch.from_numpy(rec)
    env.restore(snap)
    got = env.god_view(trajectory=True).cpu().numpy()
    ag = env.agent_state()[0].cpu().numpy()
    for e, p in enumerate(paths(env)):
        assert np.array_equal(p, want[e])
        prims = tv.trajectory_primitives("ESCAPE", task.cell_walls, task.goal, S, ag[e, :2],
                                         [tuple(int(v) for v in c) for c in p])
        img = tv.rasterise(prims, S)
        bad = np.argwhere((got[e] != img).any(-1))
        assert bad.size == 0, (e, bad[:5].tolist())
    env.close()


def test_save_trajectory_files(torch_mod, tmp_path, monkeypatch):
    torch = torch_mod
    monkeypatch.chdir(tmp_path)
    d = [d for d in CASES if "add.names" in d][0]
    kind, tt, n, S, max_steps = (int(v) for v in d["meta"])
    one = make_env(0, 1, squeeze=True, render_scale=S)
    one.set_task(case_task(d))
    one.reset()
    for a in d["act"][:20]:
        one.step(int(a))
    assert one.save_trajectory("traj.png") == ["traj.png"]
    panel = one.god_view(trajectory=True)[0].cpu().numpy()
    assert np.array_equal(_decode_png(open("traj.png", "rb").read()), panel)
    # additional surfaces (maze_base.py:161-187): the sizes, positions and names the reference used
    rng = np.random.RandomState(0)
    surfs = [rng.randint(0, 256, (h, w, 3)).astype(np.uint8) for w, h in d["add.sizes"].tolist()]
    names = one.save_trajectory("traj.png", additional={"surfaces": surfs, "file_names": ["_a", "_b"]})
    assert names == [str(v) for v in d["add.names"]]
    W, H = (int(v) for v in d["add.canvas"])
    canvas = np.full((H, W, 3), 255, np.uint8)
    canvas[:S, :S] = panel
    for (x, y, w, h), s, name in zip(d["add.blits"].tolist(), surfs, names):
        canvas[y:y + min(h, H - y), x:x + min(w, W - x)] = s[:H - y, :W - x]
        assert np.array_equal(_decode_png(open(name, "rb").read()), canvas), name
    # a batch: one file per selected env
    env = make_env(1, 3, render_scale=64)
    env.set_task(case_task(d))
    env.reset()
    env.step(torch.tensor([3, 1, 2], dtype=torch.int32, device="cuda"))
    out = env.save_trajectory(str(tmp_path / "run.png"), envs=[2, 0])
    assert out == [str(tmp_path / "run_2.png"), str(tmp_path / "run_0.png")]
    views = env.god_view(envs=[2, 0], trajectory=True).cpu().numpy()
    for k, f in enumerate(out):
        assert np.array_equal(_decode_png(open(f, "rb").read()), views[k])
    assert len(env.save_trajectory("all.png")) == 3 and os.path.exists("all_1.png")
    one.close()
    env.close()


def test_refusals_and_graph_capture(torch_mod):
    from metagym_b200 import _lib
    torch = torch_mod
    d = CASES[0]
    plain = make_env(0, 3, record_path=False)
    plain.set_task(case_task(d))
    plain.reset()
    with pytest.raises(ValueError, match="record_path"):
        plain.god_view(trajectory=True)
    with pytest.raises(ValueError, match="record_path"):
        plain.trajectory()
    lib = _lib.load()
    cells = torch.empty((3, 1001, 2), dtype=torch.int8, device="cuda")
    lens = torch.empty((3,), dtype=torch.int32, device="cuda")
    assert lib.mgb_maze_path(plain._h, 3, None, cells.data_ptr(), lens.data_ptr(), None) == MGB_ERR_ARG
    out = torch.empty((3, 40, 40, 3), dtype=torch.uint8, device="cuda")
    assert lib.mgb_maze_god_view(plain._h, 3, None, 40, 2, out.data_ptr(), None) == MGB_ERR_ARG
    # an out-of-range CUDA index: length 0 and an all-zero frame
    env = make_env(1, 4, render_scale=64)
    env.set_task(case_task(d))
    env.reset()
    _, lens = env.trajectory(torch.tensor([1, 9], dtype=torch.int32, device="cuda"))
    assert lens.tolist() == [1, 0]
    assert env.god_view(envs=torch.tensor([9], dtype=torch.int32, device="cuda"), trajectory=True).eq(0).all()
    # one recording step plus the trajectory view, captured in a CUDA graph and replayed
    twin = make_env(1, 4, render_scale=64)
    twin.set_task(case_task(d))
    twin.reset()
    act = torch.tensor([3, 1, 2, 3], dtype=torch.int32, device="cuda")
    view = torch.zeros((4, 64, 64, 3), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        env.step(act)
        env.god_view(trajectory=True, out=view)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            env.step(act)
            env.god_view(trajectory=True, out=view)
    torch.cuda.synchronize()
    twin.step(act)                                # the warm-up step; capture does not run the step
    for _ in range(3):
        graph.replay()
        twin.step(act)
    torch.cuda.synchronize()
    assert torch.equal(view, twin.god_view(trajectory=True))
    for x, y in zip(paths(env), paths(twin)):
        assert np.array_equal(x, y) and len(x) == 5
    plain.close()
    env.close()
    twin.close()
