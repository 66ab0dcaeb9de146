"""GPU tests of the batched god view (mgb_maze_god_view, maze_god_view_kernel; god_view() and render("rgb_array") of
the three MetaMaze classes): frames against the oracle raster of primitives recorded from the unmodified reference, for
every kind, task type, maze size and view size of tests/golden/maze_godview_golden.npz; env selection, batch and launch
shape invariance, CUDA-graph capture, and refusals."""
import numpy as np
import pytest

from oracle import maze_godview as gv
from test_maze_godview_oracle import CASES, recorded
from util import task_from_arrays

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def case_task(d):
    return task_from_arrays(d["task.walls"], d["task.texts"], d["task.food"], d["task.interval"], d["task.scalars"])


def make_env(kind, task_type, num_envs, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    kw = dict(dict(max_steps=1000, task_type=task_type, num_envs=num_envs, squeeze=False), **kw)
    if kind == 0:
        return BatchedMetaMaze2D(view_grid=2, **kw)
    cls = BatchedMetaMazeDiscrete3D if kind == 1 else BatchedMetaMazeContinuous3D
    return cls(resolution=(8, 8), obs_dtype="uint8", **kw)


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_god_view_equals_the_reference_primitives(torch_mod, d):
    """Replay the recorded episode on a two-env batch (env 1 a twin of env 0); at every recorded step both frames equal
    the oracle raster of the primitives the reference drew there."""
    torch = torch_mod
    kind, tt, n, S = (int(v) for v in d["meta"])
    env = make_env(kind, ("SURVIVAL", "ESCAPE")[tt], 2, render_scale=S)
    env.set_task(case_task(d))
    env.reset()
    frames = [int(f) for f in d["frames"]]
    act = d["act"]
    for t in range(frames[-1] + 1):
        if t in frames:
            f = frames.index(t)
            want = gv.rasterise(recorded(d, f), S)
            got = env.god_view().cpu().numpy()
            ag, _ = env.agent_state()
            assert tuple(ag[0, :2].tolist()) == tuple(int(v) for v in d["state"][f][:2])
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


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_selection_batch_and_launch_shape(torch_mod, kind):
    """A 300-env batch on mixed tasks after random steps: god_view() of all envs, of a permuted subset (host list and
    CUDA tensor), of single envs (a launch that splits each frame over many CTAs) and with an odd view size (frames
    that are not a multiple of 16 bytes) agree frame for frame; each frame equals the oracle raster of the state."""
    torch = torch_mod
    tasks = [case_task(d) for d in CASES if int(d["meta"][0]) == kind and int(d["meta"][2]) == 15]
    N = 300
    env = make_env(kind, "SURVIVAL", N, render_scale=480)
    env.set_task(tasks)
    env.reset()
    g = torch.Generator(device="cpu").manual_seed(kind)
    for _ in range(9):
        if kind == 2:
            env.step((torch.rand((N, 2), generator=g) * 2 - 1).cuda())
        else:
            env.step(torch.randint(0, 4, (N,), generator=g, dtype=torch.int32).cuda())
    full = env.god_view()
    sel = [299, 3, 0, 150, 3]
    assert torch.equal(env.god_view(envs=sel), full[sel])
    assert torch.equal(env.god_view(envs=torch.tensor(sel, device="cuda", dtype=torch.int32)), full[sel])
    for e in (0, 77, 299):
        assert torch.equal(env.god_view(envs=[e]), full[e:e + 1])
    odd = env.god_view(envs=[1, 2, 3], view_size=37)
    for k, e in enumerate((1, 2, 3)):
        assert torch.equal(odd[k], env.god_view(envs=[e], view_size=37)[0])
    # the oracle from the batched state
    ag, _ = env.agent_state()
    ag = ag.cpu().numpy()
    pos = ori = None
    if kind == 2:
        p, o = env.pose()
        pos, ori = p.cpu().numpy(), o.cpu().numpy()
    e2t = env.env2task
    for e in (0, 5, 123, 299):
        t = tasks[int(e2t[e])]
        food = _food_now(env, e, t)
        loc, o = gv.reference_pose(kind, ag[e, :2], ag[e, 2], ag[e, 3], None if pos is None else pos[e],
                                   None if ori is None else ori[e], t.cell_size)
        prims = gv.live_primitives(kind, "SURVIVAL", t.cell_walls, t.goal, 480, t.cell_size, food, tuple(ag[e, :2]), loc, o)
        assert np.array_equal(full[e].cpu().numpy(), gv.rasterise(prims, 480)), e
    env.close()


def _food_now(env, e, task):
    """_cur_food_rewards of env e from its snapshot record (food stamps, int32 12.. of the record) and its step counter:
    a food eaten at step s is back on the grid after step t iff t >= s + interval."""
    rec = env.snapshot()["records"][e].cpu().numpy().view(np.int32)
    steps = int(rec[3])
    food = np.asarray(task.food_rewards, np.float64)
    itv = np.asarray(task.food_interval)
    cells = [tuple(c) for c in np.argwhere(food > 0)]
    out = np.zeros_like(food)
    for f, c in enumerate(cells):
        s = int(rec[12 + f])
        if s == np.iinfo(np.int32).min // 2 or steps >= s + itv[c]:
            out[c] = food[c]
    return out


def test_graph_capture_and_render(torch_mod):
    torch = torch_mod
    d = [d for d in CASES if int(d["meta"][0]) == 1][0]
    env = make_env(1, "SURVIVAL", 4, render_scale=64)
    env.set_task(case_task(d))
    env.reset()
    envs = torch.tensor([3, 1], dtype=torch.int32, device="cuda")
    out = torch.zeros((2, 64, 64, 3), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        env.god_view(envs=envs, out=out)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            env.god_view(envs=envs, out=out)
    env.step(torch.full((4,), 3, dtype=torch.int32, device="cuda"))
    env.step(torch.full((4,), 1, dtype=torch.int32, device="cuda"))
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, env.god_view()[[3, 1]])
    assert not torch.equal(out[0], torch.zeros_like(out[0]))
    # render("rgb_array"): all envs, squeezed for a one-env batch
    assert tuple(env.render("rgb_array").shape) == (4, 64, 64, 3)
    one = make_env(1, "SURVIVAL", 1, render_scale=50, squeeze=True)
    one.set_task(case_task(d))
    one.reset()
    assert tuple(one.render(mode="rgb_array").shape) == (50, 50, 3)
    with pytest.raises(NotImplementedError):
        one.render()
    one.close()
    env.close()


def test_refusals(torch_mod):
    from metagym_b200 import _lib
    torch = torch_mod
    d = CASES[0]
    env = make_env(0, "SURVIVAL", 3)
    with pytest.raises(Exception, match="set_task"):
        env.god_view()
    env.set_task(case_task(d))
    env.reset()
    for bad in (0, -5, 4097, 2.5):
        with pytest.raises(ValueError):
            env.god_view(view_size=bad)
    with pytest.raises(IndexError):
        env.god_view(envs=[0, 3])
    with pytest.raises(IndexError):
        env.god_view(envs=[-1])
    with pytest.raises(ValueError):
        env.god_view(out=torch.empty((3, 480, 480, 3), dtype=torch.int32, device="cuda"))
    # a CUDA index tensor is not checked on the host: an out-of-range entry gives an all-zero frame
    got = env.god_view(envs=torch.tensor([1, 7, -2], dtype=torch.int32, device="cuda"), view_size=40)
    assert got[1:].eq(0).all() and not got[0].eq(0).all()
    lib = _lib.load()
    out = torch.empty((3, 40, 40, 3), dtype=torch.uint8, device="cuda")
    assert lib.mgb_maze_god_view(env._h, 3, None, 40, 1, out.data_ptr(), None) == MGB_ERR_ARG
    assert lib.mgb_maze_god_view(env._h, 4, None, 40, 0, out.data_ptr(), None) == MGB_ERR_ARG
    env.close()
