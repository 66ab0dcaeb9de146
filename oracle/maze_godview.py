"""God view of the MetaMaze envs in numpy: (a) the ordered drawing primitives the reference emits for the god panel,
(b) a rasteriser for them with the pixel rules of DESIGN.md "God view".

(a) restates MazeBase.render_init + render_update (maze_base.py:100-157) and the agent markers of maze_2d.py:73-75,
maze_discrete_3d.py:83-99 and maze_continuous_3d.py:58-74 with the reference's own numpy typing, so that every
coordinate is the float the reference passes to pygame.  tests/test_maze_godview_oracle.py checks the lists against
calls recorded from the unmodified reference (tests/golden/maze_godview_golden.npz).  (b) is the project's pixel rule,
which metagym_b200/csrc/maze.cu (maze_god_view_kernel) implements identically.

A primitive is (op, surface, colour, coords, width):
  op       "fill" | "rect" | "circle" | "line"
  surface  "god" (the panel surface of render_init) or "screen" (the window; the panel starts at x = view_size)
  coords   fill: (); rect: (x, y, w, h); circle: (cx, cy, radius); line: (x0, y0, x1, y1)
"""
import numpy as np

PI = 3.1415926                      # metagym/metamaze/envs/dynamics.py:6
COLOURS = {"white": (255, 255, 255), "black": (0, 0, 0), "green": (0, 255, 0), "red": (255, 0, 0)}


def reference_pose(kind, grid, ori_index, steps, pos, ori, cell_size):
    """(_agent_loc, _agent_ori) with the reference's types for the state a batched env reports.
    kind 1 (discrete 3-D): the cell centre as python floats (maze_discrete_3d.py:67) and the float32 heading table entry
    (:46-48), except right after a reset, where MazeBase.reset has overwritten the heading with 0.0 (maze_base.py:50).
    kind 2 (continuous): right after a reset the cell centre as python floats and heading 0.0 (maze_base.py:42,50); after
    a step the float32 position array and the float64 heading (dynamics.py:71-92)."""
    centre = [grid[0] * cell_size + 0.5 * cell_size, grid[1] * cell_size + 0.5 * cell_size]
    if kind == 1 and steps == 0:
        return centre, 0.0
    if kind == 1:
        return centre, (np.asarray([0.0, 0.5, 1.0, 1.5], dtype="float32") * PI)[int(ori_index)]
    if kind == 2:
        if steps == 0:
            return centre, 0.0
        return np.asarray(pos, dtype=np.float32), float(ori)
    return None, None


def live_primitives(kind, task_type, walls, goal, view_size, cell_size=None, food=None, grid=None, loc=None, ori=None):
    """God-panel primitives of render_init(view_size) followed by render_update().  food: the current food values [n, n]
    (_cur_food_rewards; SURVIVAL only); grid: _agent_grid; loc / ori: _agent_loc / _agent_ori typed as reference_pose
    returns them (3-D only)."""
    walls = np.asarray(walls)
    n = walls.shape[0]
    rcs = view_size / n
    out = [("fill", "god", COLOURS["white"], (), 0)]
    for x in range(n):                                          # numpy.nditer order: x outer, y inner
        for y in range(n):
            if walls[x, y] > 0:
                out.append(("rect", "god", COLOURS["black"], (x * rcs, view_size - (y + 1) * rcs, rcs, rcs), 0))
            if task_type == "ESCAPE" and x == goal[0] and y == goal[1]:
                out.append(("rect", "god", COLOURS["green"], (x * rcs, view_size - (y + 1) * rcs, rcs, rcs), 0))
    if task_type == "SURVIVAL":                                 # draw_food(screen, (view_size, 0))
        for x in range(n):
            for y in range(n):
                if food[x, y] > 1.0e-2:
                    f = int(255 - 255 * food[x, y])
                    out.append(("rect", "screen", (f, 255, f),
                                (x * rcs + view_size, 0 + view_size - (y + 1) * rcs, rcs, rcs), 0))
    if kind == 0:                                               # maze_2d.py:73-75
        out.append(("rect", "screen", COLOURS["red"],
                    (grid[0] * rcs + view_size, view_size - (grid[1] + 1) * rcs, rcs, rcs), 0))
    else:                                                       # maze_discrete_3d.py:94-99 / maze_continuous_3d.py:69-74
        pos_conversion = rcs / cell_size
        ori_size = 0.60 * pos_conversion
        agent_pos = np.array(loc) * pos_conversion
        dx = ori_size * np.cos(ori)
        dy = ori_size * np.sin(ori)
        centre = (agent_pos[0] + view_size, view_size - agent_pos[1])
        out.append(("circle", "screen", COLOURS["green"], centre + (0.15 * pos_conversion,), 0))
        out.append(("line", "screen", COLOURS["green"],
                    centre + (agent_pos[0] + view_size + dx, view_size - agent_pos[1] - dy), 1))
    return out


def _bresenham(x0, y0, x1, y1):
    """Pixels of a width-1 line between integer end points: the major axis steps by one from the start point; at step i
    the minor offset is i * d_minor / d_major rounded half up (a tie moves toward the end point)."""
    dx, dy = abs(x1 - x0), abs(y1 - y0)
    sx, sy = (1 if x1 >= x0 else -1), (1 if y1 >= y0 else -1)
    if dx >= dy:
        if dx == 0:
            return [(x0, y0)]
        return [(x0 + sx * i, y0 + sy * ((2 * i * dy + dx) // (2 * dx))) for i in range(dx + 1)]
    return [(x0 + sx * ((2 * i * dx + dy) // (2 * dy)), y0 + sy * i) for i in range(dy + 1)]


def _trunc(v):
    return int(max(-1.0e9, min(1.0e9, float(v))))


def rasterise(prims, view_size):
    """Primitives -> uint8 [S, S, 3], image rows top to bottom (img[y, x] = pygame pixel (x, y) of the panel).
    Rules: a rect covers the pixels whose centre (p + 0.5) lies in [x, x + w) x [y, y + h), in the coordinates of its
    surface; a circle covers (px - cx)^2 + (py - cy)^2 <= r^2 with cx, cy, r truncated to integers (nothing when r < 1); a
    line covers the Bresenham pixels between its truncated end points.  Screen primitives are shifted left by view_size,
    after truncation for circles and lines.  A food colour outside [0, 255] is clamped."""
    S = int(view_size)
    img = np.zeros((S, S, 3), np.uint8)
    centres = np.arange(S) + 0.5
    for op, surf, colour, c, width in prims:
        off = S if surf == "screen" else 0
        col = np.clip(np.asarray(colour, dtype=np.int64), 0, 255).astype(np.uint8)
        if op == "fill":
            img[:, :] = col
        elif op == "rect":
            x, y, w, h = c
            cx = centres + off
            mx = (x <= cx) & (cx < x + w)
            my = (y <= centres) & (centres < y + h)
            img[np.ix_(my, mx)] = col
        elif op == "circle":
            cx, cy, r = _trunc(c[0]) - off, _trunc(c[1]), _trunc(c[2])
            if r >= 1:
                py, px = np.mgrid[0:S, 0:S]
                img[(px - cx) ** 2 + (py - cy) ** 2 <= r * r] = col
        elif op == "line":
            assert width == 1, "only width-1 lines are drawn by the god panel"
            for px, py in _bresenham(_trunc(c[0]) - off, _trunc(c[1]), _trunc(c[2]) - off, _trunc(c[3])):
                if 0 <= px < S and 0 <= py < S:
                    img[py, px] = col
        else:
            raise ValueError(op)
    return img


# ---- the fixture's encoding of primitive lists: one float64 row per primitive -------------------------------------
_OPS = ("fill", "rect", "circle", "line")
_SURF = ("god", "screen")


def encode(prims):
    """-> float64 [P, 10]: op, surface, r, g, b, four coordinates (zero-padded), width."""
    rows = []
    for op, surf, colour, c, width in prims:
        cc = [float(v) for v in c] + [0.0] * (4 - len(c))
        rows.append([_OPS.index(op), _SURF.index(surf)] + [float(v) for v in colour] + cc + [float(width)])
    return np.asarray(rows, dtype=np.float64).reshape(-1, 10)


def decode(rows):
    ncoord = {"fill": 0, "rect": 4, "circle": 3, "line": 4}
    out = []
    for r in np.asarray(rows):
        op = _OPS[int(r[0])]
        out.append((op, _SURF[int(r[1])], tuple(int(v) for v in r[2:5]), tuple(float(v) for v in r[5:5 + ncoord[op]]),
                    int(r[9])))
    return out
