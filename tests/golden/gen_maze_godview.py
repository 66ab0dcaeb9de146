"""Generate tests/golden/maze_godview_golden.npz by RUNNING THE UNMODIFIED REFERENCE (build container only).

    python tests/golden/gen_maze_godview.py

The reference draws its god view with pygame, which is not installed: this script adds recording stand-ins for the pygame
calls of render_init / render_update (draw.rect / line / circle, Color, Surface.fill / blit, display.*, font.SysFont,
transform.scale, event.get, key.get_pressed, image.save) to the stub module _refload installs, without changing what
_refload itself provides, so every other generator writes the same fixtures as before.  For each case (three kinds x
SURVIVAL / ESCAPE x n in {9, 15, 21}, view sizes 480 and 500) one episode is stepped through the reference env and, at
several steps, the god-panel primitives of render_init + render_update are recorded together with the agent state, the
live food values and _agent_trajectory.
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
from gen_maze import task_arrays  # noqa: E402
from metagym_b200.textures import synthetic_textures  # noqa: E402
from oracle import maze_godview as gv  # noqa: E402

NAMED = {"white": (255, 255, 255), "black": (0, 0, 0), "green": (0, 255, 0), "red": (255, 0, 0), "blue": (0, 0, 255)}


class RecSurface(object):
    """A pygame Surface that logs what is drawn on it."""

    def __init__(self, size=(0, 0)):
        self.size = tuple(size) if isinstance(size, (tuple, list)) else (0, 0)
        self.log = []

    def fill(self, colour):
        self.log.append(("fill", tuple(colour), (), 0))

    def blit(self, src, pos):
        self.log.append(("blit", src, tuple(pos), 0))

    def get_width(self):
        return self.size[0]

    def get_height(self):
        return self.size[1]


def _colour(*args):
    if len(args) == 1 and isinstance(args[0], str):
        return NAMED[args[0]]
    return tuple(int(v) for v in args[:3])


def install_recording_pygame():
    pygame = sys.modules["pygame"]
    draw = types.ModuleType("pygame.draw")
    draw.rect = lambda s, c, r, width=0: s.log.append(("rect", tuple(c), tuple(float(v) for v in r), width))
    draw.circle = lambda s, c, p, r, width=0: s.log.append(("circle", tuple(c), (float(p[0]), float(p[1]), float(r)),
                                                             width))
    draw.line = lambda s, c, a, b, width=1: s.log.append(("line", tuple(c), (float(a[0]), float(a[1]), float(b[0]),
                                                                              float(b[1])), width))
    display = types.ModuleType("pygame.display")
    display.set_mode = lambda size: RecSurface(size)
    display.set_caption = lambda *a: None
    display.update = lambda *a: None
    font = sys.modules["pygame.font"]
    font.SysFont = lambda *a: types.SimpleNamespace(render=lambda *a: RecSurface((60, 18)))
    transform = types.ModuleType("pygame.transform")
    transform.scale = lambda surf, size: RecSurface(size)
    event = types.ModuleType("pygame.event")
    event.get = lambda: []
    key = types.ModuleType("pygame.key")
    key.get_pressed = lambda: {}
    pygame.image.save = lambda surf, name: None
    pygame.draw, pygame.display, pygame.transform, pygame.event, pygame.key = draw, display, transform, event, key
    pygame.Color, pygame.Surface, pygame.QUIT = _colour, RecSurface, 256
    sys.modules.update({"pygame.draw": draw, "pygame.display": display, "pygame.transform": transform,
                        "pygame.event": event, "pygame.key": key})


def god_panel(core, S):
    """render_init's panel surface, then the primitives render_update draws on the screen inside the panel (x >= S)."""
    core._screen.log = []
    core.render_update()
    prims = [(op, "god", c, co, w) for op, c, co, w in core._surf_god.log if op != "blit"]
    blits = [b for b in core._screen.log if b[0] == "blit" and b[1] is core._surf_god]
    assert len(blits) == 1 and blits[0][2] == (S, 0)
    prims += [(op, "screen", c, co, w) for op, c, co, w in core._screen.log if op != "blit" and co[0] >= S]
    return prims


def record(ns, kind, task_type, task, S, n_steps, frames, rng):
    kw = dict(enable_render=False, max_steps=1000, task_type=task_type)
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
    acts, rows, offs, state, food, traj, traj_off = [], [], [0], [], [], [], [0]
    for t in range(n_steps + 1):
        if t in frames:
            prims = god_panel(core, S)
            rows.append(gv.encode(prims))
            offs.append(offs[-1] + len(prims))
            loc, ori = core._agent_loc, core._agent_ori
            state.append([core._agent_grid[0], core._agent_grid[1], core.steps, float(loc[0]), float(loc[1]),
                          isinstance(loc, np.ndarray) and loc.dtype == np.float32, float(ori),
                          isinstance(ori, np.float32), getattr(core, "_agent_ori_index", 0)])
            food.append(np.array(core._cur_food_rewards, np.float64) if task_type == "SURVIVAL"
                        else np.zeros(np.shape(task.cell_walls)))
            tr = np.array(core._agent_trajectory)
            traj.append(tr)
            traj_off.append(traj_off[-1] + len(tr))
        if t == n_steps:
            break
        a = (np.array([rng.uniform(-1, 1), rng.uniform(-0.3, 1)], dtype=np.float32) if kind == 2
             else int(rng.randint(4)))
        acts.append(a)
        _, _, done, _ = env.step(a)
        if done:
            raise RuntimeError("episode ended before the last recorded step; pick other seeds")
    return dict(act=np.asarray(acts), prims=np.concatenate(rows), prim_off=np.asarray(offs, np.int64),
                state=np.asarray(state, np.float64), food_now=np.asarray(food), frames=np.asarray(frames, np.int32),
                traj=np.concatenate(traj).astype(np.int32), traj_off=np.asarray(traj_off, np.int64))


def main():
    ns = _refload.load_reference()
    install_recording_pygame()
    grounds, ceil = synthetic_textures(seed=0)
    ns.MAZE_TASK_MANAGER.grounds = grounds.astype(np.float32)
    ns.MAZE_TASK_MANAGER.ceil = ceil.astype(np.uint8)
    out = {}
    names = []
    k = 0
    for kind in (0, 1, 2):
        for tt in ("SURVIVAL", "ESCAPE"):
            for n in (9, 15, 21):
                S = (480, 500)[(k + n // 3) % 2]
                name = "k%d_%s_n%d_s%d" % (kind, tt[:4].lower(), n, S)
                random.seed(300 + k)
                np.random.seed(300 + k)
                task = ns.MazeTaskSampler(n=n, allow_loops=True, crowd_ratio=0.35, food_density=0.15 if n < 21 else 0.05,
                                          food_interval=6, goal_reward=1.0)
                rng = np.random.RandomState(400 + k)
                n_steps = 40
                rec = record(ns, kind, tt, task, S, n_steps, [0, 1, 5, 13, 26, 40], rng)
                for kk, v in task_arrays(task).items():
                    out["%s.task.%s" % (name, kk)] = v
                for kk, v in rec.items():
                    out["%s.%s" % (name, kk)] = v
                out["%s.meta" % name] = np.array([kind, 0 if tt == "SURVIVAL" else 1, n, S], dtype=np.int32)
                names.append(name)
                k += 1
                print(name, "primitives", len(rec["prims"]), "cells visited", len(set(map(tuple, rec["traj"].tolist()))))
    out["cases"] = np.array(names)
    path = os.path.join(HERE, "maze_godview_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
