"""The trajectory picture of the MetaMaze envs in numpy, on top of oracle/maze_godview.py: (a) the ordered drawing
primitives of MazeBase.render_trajectory (maze_base.py:159-189) with additional=None, (b) a rasteriser that adds the
width-3 line rule of DESIGN.md "God view" to oracle.maze_godview.rasterise.

(a) restates render_trajectory with the reference's own numpy typing, so every coordinate is the float the reference passes
to pygame; tests/test_maze_trajectory_oracle.py checks the lists against calls recorded from the unmodified reference
(tests/golden/maze_trajectory_golden.npz).  (b) is the project's pixel rule, which metagym_b200/csrc/maze.cu
(maze_god_view_kernel in trajectory mode, then maze_god_path_kernel) implements identically.  Primitives are those of
oracle.maze_godview; every one of them is drawn on the trajectory screen at offset 0 (surface "god").
"""
import numpy as np

from oracle import maze_godview as gv

RED = gv.COLOURS["red"]


def trajectory_primitives(task_type, walls, goal, view_size, grid, trajectory, food=None):
    """render_trajectory(file_name) after render_init(view_size): traj_screen.fill(white); blit of the god surface (its
    fill, wall rects and ESCAPE goal, nditer order); the red agent rect at _agent_grid; SURVIVAL food at offset (0, 0)
    (food: _cur_food_rewards [n, n]); a red width-3 line per consecutive pair of _agent_trajectory."""
    walls = np.asarray(walls)
    n = walls.shape[0]
    rcs = view_size / n
    out = [("fill", "god", gv.COLOURS["white"], (), 0), ("fill", "god", gv.COLOURS["white"], (), 0)]
    for x in range(n):                                          # render_init, numpy.nditer order: x outer, y inner
        for y in range(n):
            if walls[x, y] > 0:
                out.append(("rect", "god", gv.COLOURS["black"], (x * rcs, view_size - (y + 1) * rcs, rcs, rcs), 0))
            if task_type == "ESCAPE" and x == goal[0] and y == goal[1]:
                out.append(("rect", "god", gv.COLOURS["green"], (x * rcs, view_size - (y + 1) * rcs, rcs, rcs), 0))
    out.append(("rect", "god", RED, (grid[0] * rcs, view_size - (grid[1] + 1) * rcs, rcs, rcs), 0))
    if task_type == "SURVIVAL":                                 # draw_food(traj_screen, (0, 0))
        for x in range(n):
            for y in range(n):
                if food[x, y] > 1.0e-2:
                    f = int(255 - 255 * food[x, y])
                    out.append(("rect", "god", (f, 255, f), (x * rcs + 0, 0 + view_size - (y + 1) * rcs, rcs, rcs), 0))
    for i in range(len(trajectory) - 1):
        p, q = trajectory[i], trajectory[i + 1]
        p = [(p[0] + 0.5) * rcs, view_size - (p[1] + 0.5) * rcs]
        q = [(q[0] + 0.5) * rcs, view_size - (q[1] + 0.5) * rcs]
        out.append(("line", "god", RED, (p[0], p[1], q[0], q[1]), 3))
    return out


def wide_line(x0, y0, x1, y1):
    """Pixels of a width-3 line between integer end points: every pixel of the width-1 line widened into a 3-pixel span
    across the minor axis, along x when |dx| <= |dy| and along y otherwise (pygame 2's draw_line_width); a zero-length
    segment is one span along x."""
    span_x = abs(x1 - x0) <= abs(y1 - y0)
    out = []
    for px, py in gv._bresenham(x0, y0, x1, y1):
        out += [(px + k, py) if span_x else (px, py + k) for k in (-1, 0, 1)]
    return out


def rasterise(prims, view_size):
    """oracle.maze_godview.rasterise with width-3 lines: the primitives before the first width-3 line are rasterised by
    it, then the width-3 lines (which render_trajectory draws last) on top."""
    S = int(view_size)
    first = next((i for i, p in enumerate(prims) if p[0] == "line" and p[4] == 3), len(prims))
    img = gv.rasterise(prims[:first], S)
    for op, surf, colour, c, width in prims[first:]:
        assert op == "line" and width == 3 and surf == "god", "render_trajectory draws its path lines last"
        tr = gv._trunc
        for px, py in wide_line(tr(c[0]), tr(c[1]), tr(c[2]), tr(c[3])):
            if 0 <= px < S and 0 <= py < S:
                img[py, px] = colour
    return img
