"""Generate tests/golden/maze_optics_golden.npz by RUNNING THE UNMODIFIED REFERENCE with NON-default optics and screen
shapes (build container only).

    python tests/golden/gen_maze_optics.py

Every other 3-D fixture renders with the reference's default optics (max_vision_range 12.0, fol_angle 0.6 pi) on even
screens.  Here the cores are built with other vision ranges and fields of view (MazeCoreDiscrete3D /
MazeCoreContinuous3D keyword arguments, maze_discrete_3d.py:22-23; the MetaMaze*3D wrappers do not forward them, so the
wrapper's maze_core is replaced), on odd, tall and degenerate screens.  Case `xings` is a hand-built open arena with a
food band along the diagonal: columns near +45 degrees cross up to about 57 transparent cells within the vision range,
which pins that every crossing of DDA_2D is blended (ray_caster_utils.py:11-62,194-205).  Textures as in gen_maze.py.
"""
import os
import random
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _refload  # noqa: E402
from gen_maze import plan, record, task_arrays  # noqa: E402
import gen_maze_continuous as gc  # noqa: E402
from metagym_b200.textures import synthetic_textures  # noqa: E402

PI = 3.1415926                      # metagym/metamaze/envs/dynamics.py:6


def with_optics(ns, vision, fov):
    """A copy of the loader namespace whose MetaMazeDiscrete3D / MetaMazeContinuous3D run cores with these optics."""
    import importlib
    d3 = importlib.import_module("metagym.metamaze.envs.maze_discrete_3d")
    c3 = importlib.import_module("metagym.metamaze.envs.maze_continuous_3d")

    def factory(wrapper, core):
        def make(enable_render, resolution, max_steps, task_type):
            env = wrapper(enable_render=enable_render, resolution=resolution, max_steps=max_steps, task_type=task_type)
            env.maze_core = core(max_vision_range=vision, fol_angle=fov, resolution_horizon=resolution[0],
                                 resolution_vertical=resolution[1], max_steps=max_steps, task_type=task_type)
            return env
        return make

    out = types.SimpleNamespace(**vars(ns))
    out.MetaMazeDiscrete3D = factory(ns.MetaMazeDiscrete3D, d3.MazeCoreDiscrete3D)
    out.maze_env = types.SimpleNamespace(MetaMazeContinuous3D=factory(ns.maze_env.MetaMazeContinuous3D,
                                                                      c3.MazeCoreContinuous3D))
    return out


def xings_task(ns):
    """n = 31, walls on the border only, cell 0.25 / wall 0.5 / eye 0.25, food on every interior cell with |i - j| <= 1
    (85 cells), start (1, 1) facing +x.  A ray along the band lists its crossings in the order of i + j.  Each blend
    truncates to int32 (ray_caster_utils.py:205), so weak foods (0.011: blend factor 0.1055) before i + j = 49 drive a
    wall pixel to a fixed point after ~45 blends, and only the strong foods (0.5: factor 0.35) past it move the pixel
    again: a renderer that drops the crossings past the 48th changes the wall pixels of the columns along the band."""
    n = 31
    walls = np.zeros((n, n), dtype=np.int32)
    walls[0, :] = walls[-1, :] = walls[:, 0] = walls[:, -1] = 1
    rs = np.random.RandomState(31)
    texts = rs.randint(1, 7, size=(n, n)) * walls
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    band = (np.abs(i - j) <= 1) & (walls == 0)
    food = np.where(band, np.where(i + j >= 49, 0.5, 0.011), 0.0)
    interval = 6 * band.astype(np.int32)
    assert int(band.sum()) == 85
    return ns.TaskConfig(start=(1, 1), goal=(n - 2, n - 2), cell_walls=walls, cell_texts=texts, cell_size=0.25,
                         wall_height=0.5, agent_height=0.25, initial_life=1.0, max_life=2.0, step_reward=-0.12,
                         goal_reward=1.0, food_rewards=food, food_interval=interval)


def thin(rec, every):
    """Keep the frames of every `every`-th step and of every terminal step (the fixture stays small; rewards, dones and
    states are kept for every step)."""
    idx = np.asarray(rec["obs_idx"])
    sel = (idx % every == 0) | np.asarray(rec["done"])[idx]
    rec["obs"], rec["obs_idx"] = rec["obs"][sel], idx[sel]
    return rec


def main():
    ns = _refload.load_reference()
    grounds, ceil = synthetic_textures(seed=0)
    ns.MAZE_TASK_MANAGER.grounds = grounds.astype(np.float32)
    ns.MAZE_TASK_MANAGER.ceil = ceil.astype(np.uint8)
    out = {}
    g15 = dict(cell_size=1.5, wall_height=2.5, agent_height=0.9)
    cases = [
        # name, task type, sampler kwargs (None: xings arena), max_steps, actions, resolution, vision, fov, frame stride
        ("o3d_near", "SURVIVAL", dict(n=11, allow_loops=True, crowd_ratio=0.35, food_density=0.04, food_interval=9,
                                      step_reward=-0.09), 200, 90, (37, 23), 5.0, 0.35 * PI, 3),
        ("o3d_wide", "SURVIVAL", dict(n=11, allow_loops=True, crowd_ratio=0.3, food_density=0.06, food_interval=7,
                                      step_reward=-0.1, **g15), 200, 60, (64, 64), 20.0, 0.85 * PI, 15),
        ("o3d_esc", "ESCAPE", dict(n=9, step_reward=-0.02, goal_reward=1.5), 80, 70, (48, 30), 8.0, 0.5 * PI, 4),
        ("o3d_tall", "SURVIVAL", dict(n=9, food_density=0.05, food_interval=6, step_reward=-0.1), 200, 70, (6, 70),
         12.0, 0.6 * PI, 1),
        ("o3d_dot1", "SURVIVAL", dict(n=9, food_density=0.05, food_interval=6, step_reward=-0.1), 200, 60, (1, 1),
         12.0, 0.6 * PI, 1),
        ("o3d_dot3", "SURVIVAL", dict(n=9, food_density=0.05, food_interval=6, step_reward=-0.1), 200, 60, (3, 2),
         12.0, 0.6 * PI, 1),
        ("xings", "SURVIVAL", None, 200, 40, (128, 96), 12.0, 0.6 * PI, 10),
    ]
    for k, (name, tt, skw, max_steps, n_act, res, vision, fov, every) in enumerate(cases):
        if skw is None:
            task = xings_task(ns)
        else:
            random.seed(90 + k)
            np.random.seed(90 + k)
            task = ns.MazeTaskSampler(**skw)
        rng = np.random.RandomState(500 + k)
        acts = plan(task, "3D", rng, n_act, tt)
        if name == "xings":          # look along the band first: the start pose sees the longest crossing lists
            acts = [1, 0, 0, 1] + acts[:n_act - 4]
        rec = thin(record(with_optics(ns, vision, fov), "3D", tt, task, acts, max_steps, res, 1, None), every)
        for kk, v in task_arrays(task).items():
            out["%s.task.%s" % (name, kk)] = v
        for kk, v in rec.items():
            out["%s.%s" % (name, kk)] = v
        out["%s.meta" % name] = np.array([1, 0 if tt == "SURVIVAL" else 1, max_steps, 1, res[0], res[1]], dtype=np.int32)
        out["%s.optics" % name] = np.array([vision, fov], dtype=np.float64)
        if tt == "SURVIVAL":
            assert (rec["done"] & (rec["life"] < 0)).any(), name + ": no death"
        else:
            assert rec["done"].any(), name + ": goal never reached"
        print(name, "steps", len(acts), "dones", int(rec["done"].sum()), "reward>0", int((rec["rew"] > 0).sum()),
              "frames", len(rec["obs_idx"]))
    # continuous 3-D: sampled task with short, narrow optics on an odd screen, and the xings arena
    ccases = [("oc3d", dict(n=9, allow_loops=True, crowd_ratio=0.3, food_density=0.15, food_interval=20,
                            step_reward=-0.04), 300, 280, (33, 19), 7.0, 0.45 * PI, 9),
              ("xings_c", None, 200, 45, (64, 48), 12.0, 0.6 * PI, 9)]
    for k, (name, skw, max_steps, n_act, res, vision, fov, every) in enumerate(ccases):
        if skw is None:
            task = xings_task(ns)
        else:
            random.seed(120 + k)
            np.random.seed(120 + k)
            task = ns.MazeTaskSampler(**skw)
        rec = thin(gc.record(with_optics(ns, vision, fov), "SURVIVAL", task, n_act, max_steps, res,
                             np.random.RandomState(600 + k)), every)
        for kk, v in task_arrays(task).items():
            out["%s.task.%s" % (name, kk)] = v
        for kk, v in rec.items():
            out["%s.%s" % (name, kk)] = v
        out["%s.meta" % name] = np.array([0, max_steps, res[0], res[1]], dtype=np.int32)
        out["%s.optics" % name] = np.array([vision, fov], dtype=np.float64)
        assert (rec["done"] & (rec["life"] < 0)).any(), name + ": no death"
        print(name, "steps", n_act, "dones", int(rec["done"].sum()), "reward>0", int((rec["rew"] > 0).sum()),
              "frames", len(rec["obs_idx"]))
    path = os.path.join(HERE, "maze_optics_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")
    assert os.path.getsize(path) < 650_000, "fixture too large for the repository: keep fewer frames"


if __name__ == "__main__":
    main()
