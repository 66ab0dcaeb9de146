"""CPU: the god-view oracle (oracle/maze_godview.py) against primitives recorded from the unmodified reference
(tests/golden/maze_godview_golden.npz, written by tests/golden/gen_maze_godview.py), and unit cases of its rasteriser."""
import os

import numpy as np
import pytest

from oracle import maze_godview as gv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "maze_godview_golden.npz")


def load_cases():
    g = np.load(GOLDEN, allow_pickle=False)
    cases = []
    for name in g["cases"]:
        pre = str(name) + "."
        d = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
        d["name"] = str(name)
        cases.append(d)
    return cases


CASES = load_cases()


def frame_inputs(d, f):
    """Arguments of gv.live_primitives for frame f of a case, typed like the recorded reference state."""
    kind, tt, n, S = (int(v) for v in d["meta"])
    gx, gy, steps, lx, ly, loc_f32, ori, ori_f32, ori_idx = d["state"][f]
    loc = np.asarray([lx, ly], np.float32) if loc_f32 else [float(lx), float(ly)]
    ori = np.float32(ori) if ori_f32 else float(ori)
    return dict(kind=kind, task_type=("SURVIVAL", "ESCAPE")[tt], walls=d["task.walls"],
                goal=(int(d["task.scalars"][2]), int(d["task.scalars"][3])), view_size=S,
                cell_size=float(d["task.scalars"][4]), food=d["food_now"][f], grid=(int(gx), int(gy)), loc=loc, ori=ori)


def recorded(d, f):
    o = d["prim_off"]
    return gv.decode(d["prims"][o[f]:o[f + 1]])


def test_fixture_covers_every_kind_task_size_and_view():
    metas = {tuple(int(v) for v in d["meta"]) for d in CASES}
    assert {m[0] for m in metas} == {0, 1, 2} and {m[1] for m in metas} == {0, 1}
    assert {m[2] for m in metas} == {9, 15, 21} and {m[3] for m in metas} == {480, 500}
    assert len({m[:3] for m in metas}) == 18
    for S in (480, 500):                           # both view sizes for every kind
        assert {m[0] for m in metas if m[3] == S} == {0, 1, 2}


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_oracle_primitives_equal_the_reference_calls(d):
    """Every primitive, in order, with its colour and every float coordinate bit for bit."""
    for f in range(len(d["frames"])):
        assert gv.live_primitives(**frame_inputs(d, f)) == recorded(d, f), (d["name"], int(d["frames"][f]))


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_reference_pose_restates_the_recorded_types(d):
    """reference_pose() (what the GPU tests build from a batched env's state) gives the reference's own position and
    heading values and types at every recorded frame of the 3-D envs."""
    kind = int(d["meta"][0])
    if kind == 0:
        pytest.skip("2-D: no pose")
    for f in range(len(d["frames"])):
        gx, gy, steps, lx, ly, loc_f32, ori, ori_f32, ori_idx = d["state"][f]
        loc, o = gv.reference_pose(kind, (int(gx), int(gy)), int(ori_idx), int(steps), (lx, ly), ori,
                                   float(d["task.scalars"][4]))
        want = frame_inputs(d, f)
        assert type(o) is type(want["ori"]) and o == want["ori"]
        if loc_f32:
            assert loc.dtype == np.float32 and np.array_equal(loc, want["loc"])
        else:
            assert isinstance(loc, list) and loc == want["loc"]


@pytest.mark.parametrize("d", CASES, ids=[d["name"] for d in CASES])
def test_recorded_paths_are_the_agent_cells(d):
    """_agent_trajectory recorded with each frame: start cell, one cell per step, ending at the agent's cell, and a
    prefix of the next frame's path."""
    tr, off, frames = d["traj"], d["traj_off"], d["frames"]
    prev = None
    for f in range(len(frames)):
        p = tr[off[f]:off[f + 1]]
        assert len(p) == int(frames[f]) + 1
        assert tuple(p[0]) == (int(d["task.scalars"][0]), int(d["task.scalars"][1]))
        assert tuple(p[-1]) == tuple(int(v) for v in d["state"][f][:2])
        if prev is not None:
            assert np.array_equal(p[:len(prev)], prev)
        prev = p


def test_food_colours_and_eaten_food_appear_in_the_fixture():
    """The SURVIVAL cases draw graded food colours, and some food is eaten (drawn at one frame, gone at a later one)."""
    greens, eaten = set(), 0
    for d in CASES:
        if int(d["meta"][1]) != 0:
            continue
        fn = d["food_now"]
        eaten += int(((fn[0] > 1e-2) & (fn[1:] <= 1e-2)).sum())
        for f in range(len(d["frames"])):
            greens |= {p[2] for p in recorded(d, f) if p[0] == "rect" and p[1] == "screen" and p[2][1] == 255}
    assert len(greens) > 5 and eaten > 0


@pytest.mark.parametrize("S,n", [(500, 15), (480, 21), (480, 9), (500, 9), (500, 21), (37, 9)])
def test_cell_rects_tile_the_panel(S, n):
    """Every pixel is covered by exactly one cell rect, also when S / n is not an integer."""
    rcs = S / n
    count = np.zeros((S, S), np.int32)
    for x in range(n):
        for y in range(n):
            img = gv.rasterise([("rect", "god", (255, 255, 255), (x * rcs, S - (y + 1) * rcs, rcs, rcs), 0)], S)
            count += img[:, :, 0] > 0
    assert (count == 1).all()
    # the same for the screen-space rects of draw_food and the 2-D agent
    count[:] = 0
    for x in range(n):
        for y in range(n):
            img = gv.rasterise([("rect", "screen", (255, 255, 255), (x * rcs + S, 0 + S - (y + 1) * rcs, rcs, rcs), 0)],
                               S)
            count += img[:, :, 0] > 0
    assert (count == 1).all()


def test_y_axis_points_up():
    """Cell (0, 0) is the bottom-left block of the image, cell (n-1, n-1) the top-right one."""
    S, n = 90, 9
    img = gv.live_primitives(0, "ESCAPE", np.zeros((n, n), np.int32), (n - 1, n - 1), S, grid=(0, 0))
    ras = gv.rasterise(img, S)
    assert tuple(ras[S - 1, 0]) == (255, 0, 0) and tuple(ras[S - 10, 9]) == (255, 0, 0)
    assert tuple(ras[S - 11, 0]) == (255, 255, 255) and tuple(ras[0, S - 1]) == (0, 255, 0)
    assert tuple(ras[9, S - 10]) == (0, 255, 0) and tuple(ras[10, S - 10]) == (255, 255, 255)


def test_food_colour():
    S, n = 45, 9
    food = np.zeros((n, n))
    food[2, 3] = 0.3
    food[4, 4] = 0.01            # not above the 1e-2 threshold: not drawn
    food[5, 5] = 1.5             # would make pygame.Color raise: clamped
    walls = np.zeros((n, n), np.int32)
    ras = gv.rasterise(gv.live_primitives(0, "SURVIVAL", walls, (7, 7), S, food=food, grid=(1, 1)), S)
    assert tuple(ras[S - 5 * 3 - 2, 2 * 5 + 2]) == (int(255 - 255 * 0.3), 255, int(255 - 255 * 0.3))
    assert tuple(ras[S - 5 * 4 - 2, 4 * 5 + 2]) == (255, 255, 255)
    assert tuple(ras[S - 5 * 5 - 2, 5 * 5 + 2]) == (0, 255, 0)


def test_lines_and_discs():
    S = 20
    g = lambda prims: gv.rasterise([("fill", "god", (0, 0, 0), (), 0)] + prims, S)[:, :, 1] > 0   # noqa: E731
    # zero-length segment: one pixel at the truncated point
    m = g([("line", "god", (0, 255, 0), (5.9, 7.2, 5.1, 7.99), 1)])
    assert m.sum() == 1 and m[7, 5]
    # shallow line: one pixel per column, minor coordinate rounded half up
    m = g([("line", "god", (0, 255, 0), (2.0, 3.0, 6.0, 5.0), 1)])
    assert [tuple(p) for p in np.argwhere(m.T)] == [(2, 3), (3, 4), (4, 4), (5, 5), (6, 5)]
    # steep line, drawn backwards
    m = g([("line", "god", (0, 255, 0), (4.0, 9.0, 3.0, 5.0), 1)])
    assert sorted(tuple(p) for p in np.argwhere(m.T)) == [(3, 5), (3, 6), (3, 7), (4, 8), (4, 9)]
    # screen coordinates: shifted by view_size after truncation
    assert np.array_equal(g([("line", "screen", (0, 255, 0), (S + 2.5, 3.0, S + 6.2, 5.0), 1)]),
                          g([("line", "god", (0, 255, 0), (2.0, 3.0, 6.0, 5.0), 1)]))
    # disc: truncated centre and radius; radius < 1 draws nothing
    m = g([("circle", "god", (0, 255, 0), (10.7, 10.2, 2.9), 0)])
    assert m.sum() == 13 and m[10, 10] and m[8, 10] and m[10, 12] and not m[8, 9]
    assert g([("circle", "god", (0, 255, 0), (10.7, 10.2, 0.9), 0)]).sum() == 0
