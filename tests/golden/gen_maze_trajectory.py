"""Generate tests/golden/maze_trajectory_golden.npz by RUNNING THE UNMODIFIED REFERENCE (build container only).

    python tests/golden/gen_maze_trajectory.py

The reference draws save_trajectory() (MazeBase.render_trajectory, maze_base.py:159-189) with pygame, which is not
installed: this script installs the recording pygame stand-ins of gen_maze_godview.py (their Surface logs fill / blit /
draw calls and reports its size; image.save does nothing) and captures the surface each image.save call receives.  For
each case (three kinds x SURVIVAL / ESCAPE x n in {9, 15, 21} x view sizes 480 and 500) one episode is stepped through the
reference env with random actions, long enough to revisit cells, and every third case runs to done on a short step limit.
At several steps the primitives render_trajectory draws are recorded (the god surface's blit expanded into its own calls)
together with _agent_trajectory, the agent cell and the live food values.  One 2-D case also records the composite of
save_trajectory(additional=...): the canvas size, the blits and the file names.
"""
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import _refload  # noqa: E402
import gen_maze_godview as gmg  # noqa: E402
from gen_maze import task_arrays  # noqa: E402
from metagym_b200.textures import synthetic_textures  # noqa: E402
from oracle import maze_godview as gv  # noqa: E402

SAVED = []


def capture_saves():
    import pygame
    pygame.image.save = lambda surf, name: SAVED.append((name, surf))


def trajectory_calls(core, surf):
    """The drawing calls that made `surf` (a render_trajectory screen), the god surface's blit replaced by its calls
    (text labels, which are blits of font surfaces, left out)."""
    prims = []
    for op, c, co, w in surf.log:
        if op == "blit":
            if c is core._surf_god:
                assert co == (0, 0)
                prims += [(op2, "god", c2, co2, w2) for op2, c2, co2, w2 in core._surf_god.log if op2 != "blit"]
            continue
        prims.append((op, "god", c, co, w))
    return prims


def record(ns, kind, task_type, task, S, n_steps, frames, max_steps, rng):
    kw = dict(enable_render=False, max_steps=max_steps, task_type=task_type)
    if kind == 0:
        env = ns.maze_env.MetaMaze2D(view_grid=2, **kw)
    elif kind == 1:
        env = ns.maze_env.MetaMazeDiscrete3D(resolution=(8, 8), **kw)
    else:
        env = ns.maze_env.MetaMazeContinuous3D(resolution=(8, 8), **kw)
    env.set_task(task)
    env.reset()
    core = env.maze_core
    core.render_init(S)
    acts, rows, offs, grid, food, traj, traj_off, shot = [], [], [0], [], [], [], [0], []
    done = False
    for t in range(n_steps + 1):
        if t in frames or done:
            del SAVED[:]
            env.save_trajectory("traj.png")
            assert len(SAVED) == 1 and SAVED[0][0] == "traj.png" and SAVED[0][1].size == (S, S)
            prims = trajectory_calls(core, SAVED[0][1])
            rows.append(gv.encode(prims))
            offs.append(offs[-1] + len(prims))
            grid.append([int(core._agent_grid[0]), int(core._agent_grid[1]), int(core.steps)])
            food.append(np.array(core._cur_food_rewards, np.float64) if task_type == "SURVIVAL"
                        else np.zeros(np.shape(task.cell_walls)))
            tr = np.array(core._agent_trajectory)
            traj.append(tr)
            traj_off.append(traj_off[-1] + len(tr))
            shot.append(t)
        if done or t == n_steps:
            break
        a = (np.array([rng.uniform(-0.4, 0.4), rng.uniform(0.2, 1)], dtype=np.float32) if kind == 2
             else int(rng.randint(4)))
        acts.append(a)
        _, _, done, _ = env.step(a)
    return env, dict(act=np.asarray(acts), prims=np.concatenate(rows), prim_off=np.asarray(offs, np.int64),
                     grid=np.asarray(grid, np.int32), food_now=np.asarray(food), frames=np.asarray(shot, np.int32),
                     traj=np.concatenate(traj).astype(np.int32), traj_off=np.asarray(traj_off, np.int64),
                     done=np.int32(done))


def record_additional(env, S):
    """save_trajectory("traj.png", additional) with two surfaces of different sizes: canvas size, per save the blits onto
    the canvas (position, surface size) and the file name."""
    surfs = [gmg.RecSurface((120, 90)), gmg.RecSurface((80, 200))]
    del SAVED[:]
    env.save_trajectory("traj.png", additional={"surfaces": surfs, "file_names": ["_a", "_b"]})
    names = np.array([name for name, _ in SAVED])
    canvas = np.array(SAVED[0][1].size, np.int32)
    blits = np.array([[co[0], co[1], src.size[0], src.size[1]] for _, surf in SAVED[-1:] for op, src, co, w in surf.log
                      if op == "blit" and src in surfs], np.int32)
    return {"add.names": names, "add.canvas": canvas, "add.blits": blits,
            "add.sizes": np.array([s.size for s in surfs], np.int32)}


def main():
    ns = _refload.load_reference()
    gmg.install_recording_pygame()
    capture_saves()
    grounds, ceil = synthetic_textures(seed=0)
    ns.MAZE_TASK_MANAGER.grounds = grounds.astype(np.float32)
    ns.MAZE_TASK_MANAGER.ceil = ceil.astype(np.uint8)
    out = {}
    names = []
    k = 0
    for kind in (0, 1, 2):
        for tt in ("SURVIVAL", "ESCAPE"):
            for n in (9, 15, 21):
                for S in (480, 500):
                    name = "k%d_%s_n%d_s%d" % (kind, tt[:4].lower(), n, S)
                    random.seed(700 + k)
                    np.random.seed(700 + k)
                    task = ns.MazeTaskSampler(n=n, allow_loops=True, crowd_ratio=0.35,
                                              food_density=0.15 if n < 21 else 0.05, food_interval=6, goal_reward=1.0)
                    rng = np.random.RandomState(800 + k)
                    max_steps = (150 if kind == 2 else 45) if k % 3 == 0 else 1000
                    T = 300 if kind == 2 else 90                 # a continuous step moves at most 0.1 (cell size 2)
                    env, rec = record(ns, kind, tt, task, S, T, [0, 1, T // 3, T], max_steps, rng)
                    for kk, v in task_arrays(task).items():
                        out["%s.task.%s" % (name, kk)] = v
                    for kk, v in rec.items():
                        out["%s.%s" % (name, kk)] = v
                    out["%s.meta" % name] = np.array([kind, 0 if tt == "SURVIVAL" else 1, n, S, max_steps],
                                                     dtype=np.int32)
                    if kind == 0 and tt == "SURVIVAL" and n == 9 and S == 480:
                        for kk, v in record_additional(env, S).items():
                            out["%s.%s" % (name, kk)] = v
                    names.append(name)
                    k += 1
                    tr = rec["traj"][rec["traj_off"][-2]:]
                    print(name, "frames", rec["frames"].tolist(), "done", int(rec["done"]), "path", len(tr),
                          "distinct cells", len(set(map(tuple, tr.tolist()))))
    out["cases"] = np.array(names)
    path = os.path.join(HERE, "maze_trajectory_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
