"""Shared comparison helpers for the parity tests."""
import numpy as np

# state row = p3 v3 w3 prop4 R9
STATE_GROUPS = [(0, 3), (3, 6), (6, 9), (9, 13), (13, 22)]
# obs row = b_v3 b_p3 acc3 gyro3 (pitch roll yaw) z [target3]
# third entry = scale floor of the group: angles are compared against 1 rad, the barometer z = p_z + z_offset against the
# 5 m offset it contains (near the floor z -> 0 by cancellation while p_z itself is ~5)
OBS_GROUPS = [(0, 3), (3, 6), (6, 9), (9, 12), (12, 15, 1.0), (15, 16, 5.0)]
TASK_NAMES = {0: "no_collision", 1: "hovering_control", 2: "velocity_control"}


def group_rel_err(a, ref, groups, floor=1e-3):
    """max over entries of |a-ref| / max(group inf-norm of ref, floor): the '1e-5 relative fp32' metric of the
    north star, taken per physical vector (a 1e-15 m position component is compared against the vector's size)."""
    a = np.asarray(a, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    a = a.reshape(-1, a.shape[-1])
    ref = ref.reshape(-1, ref.shape[-1])
    worst = 0.0
    for grp in groups:
        lo, hi = grp[0], grp[1]
        gfloor = grp[2] if len(grp) > 2 else floor
        scale = np.maximum(np.abs(ref[:, lo:hi]).max(axis=1, keepdims=True), gfloor)
        err = np.abs(a[:, lo:hi] - ref[:, lo:hi]) / scale
        if err.size:
            worst = max(worst, float(np.nanmax(err)))
        assert not np.isnan(a[:, lo:hi]).any()
    return worst


def group_rel_err_rows(a, ref, groups, floor=1e-3):
    """group_rel_err of every row on its own: [n]."""
    a = np.asarray(a, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    a = a.reshape(-1, a.shape[-1])
    ref = ref.reshape(-1, ref.shape[-1])
    worst = np.zeros(a.shape[0])
    for grp in groups:
        lo, hi = grp[0], grp[1]
        gfloor = grp[2] if len(grp) > 2 else floor
        scale = np.maximum(np.abs(ref[:, lo:hi]).max(axis=1, keepdims=True), gfloor)
        worst = np.maximum(worst, (np.abs(a[:, lo:hi] - ref[:, lo:hi]) / scale).max(axis=1))
        assert not np.isnan(a[:, lo:hi]).any()
    return worst


def scalar_rel_err(a, ref, floor=1.0):
    a = np.asarray(a, dtype=np.float64).reshape(-1)
    ref = np.asarray(ref, dtype=np.float64).reshape(-1)
    return float((np.abs(a - ref) / np.maximum(np.abs(ref), floor)).max()) if a.size else 0.0


def golden_run(g, name):
    """dict view of one recorded run of tests/golden/quadrotor_golden.npz."""
    pre = name + "."
    d = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    task, dt, nt, seed = d["meta"]
    d["task"], d["dt"], d["nt"], d["seed"] = TASK_NAMES[int(task)], float(dt), int(nt), int(seed)
    return d


QUAD_RUNS = ["hover_a", "hover_b", "hover_fall", "nocol_fall", "nocol_a", "vel_a", "vel_b", "vel_c"]
QUAD_MAP_RUNS = ["map_hover", "map_nocol"]      # recorded with the obstacle map stored as "map_obst"


# ---------------------------------------------------------------------------------------------------------------
# maze fixtures
# ---------------------------------------------------------------------------------------------------------------
from collections import namedtuple  # noqa: E402

MazeTask = namedtuple("MazeTask", ["start", "goal", "cell_walls", "cell_texts", "cell_size", "wall_height",
                                   "agent_height", "initial_life", "max_life", "step_reward", "goal_reward",
                                   "food_rewards", "food_interval"])
MAZE_CASES = ["m2d_surv", "m2d_surv_g2", "m2d_esc", "m3d_surv", "m3d_esc", "m3d_big"]
# tests/golden/maze_optics_golden.npz (gen_maze_optics.py): non-default vision range / field of view, odd, tall and
# degenerate screens, and an arena with more transparent crossings per column than any sampled task
OPTICS_CASES = ["o3d_near", "o3d_wide", "o3d_esc", "o3d_tall", "o3d_dot1", "o3d_dot3", "xings"]
OPTICS_CONT_CASES = ["oc3d", "xings_c"]


def task_from_arrays(walls, texts, food, interval, scalars):
    s = scalars
    return MazeTask(start=(int(s[0]), int(s[1])), goal=(int(s[2]), int(s[3])), cell_walls=np.asarray(walls),
                    cell_texts=np.asarray(texts), cell_size=float(s[4]), wall_height=float(s[5]),
                    agent_height=float(s[6]), initial_life=float(s[7]), max_life=float(s[8]),
                    step_reward=float(s[9]), goal_reward=float(s[10]), food_rewards=np.asarray(food),
                    food_interval=np.asarray(interval))


def maze_case(g, name):
    pre = name + "."
    d = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    kind, tt, max_steps, view_grid, rh, rv = [int(x) for x in d["meta"]]
    d["kind"] = "2D" if kind == 0 else "3D"
    d["task_type"] = "SURVIVAL" if tt == 0 else "ESCAPE"
    d["max_steps"], d["view_grid"], d["resolution"] = max_steps, view_grid, (rh, rv)
    d["task"] = task_from_arrays(d["task.walls"], d["task.texts"], d["task.food"], d["task.interval"],
                                 d["task.scalars"])
    return d


def optics_kw(c):
    """OracleMaze keyword arguments of a case's optics (the reference defaults when the fixture has none)."""
    return {} if "optics" not in c else dict(max_vision=float(c["optics"][0]), fov=float(c["optics"][1]))


def cont_case(g, name):
    pre = name + "."
    d = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    tt, max_steps, rh, rv = [int(x) for x in d["meta"]]
    d["task_type"] = "SURVIVAL" if tt == 0 else "ESCAPE"
    d["max_steps"], d["resolution"] = max_steps, (rh, rv)
    d["task"] = task_from_arrays(d["task.walls"], d["task.texts"], d["task.food"], d["task.interval"], d["task.scalars"])
    return d


# ---------------------------------------------------------------------------------------------------------------
# outputs past 32-bit offsets (tests/test_large_index_gpu.py, checked on the CPU by tests/test_large_index_layout.py)
# ---------------------------------------------------------------------------------------------------------------
B31, B32, E31 = "byte 2^31", "byte 2^32", "element 2^31"


def layout_bytes(T, n, row_bytes):
    """Bytes of a [T, n, row_bytes] output (T None: [n, row_bytes])."""
    return (1 if T is None else int(T)) * int(n) * int(row_bytes)


def crossings(T, n, row_bytes, elem_bytes):
    """The boundaries among B31, B32 and E31 (element index 2^31, elements of elem_bytes) that lie inside the output:
    the offset of its last byte / element is at least the boundary, so a 32-bit offset of that kind wraps there."""
    total = layout_bytes(T, n, row_bytes)
    out = set()
    if total > 1 << 31:
        out.add(B31)
    if total > 1 << 32:
        out.add(B32)
    if total // elem_bytes > 1 << 31:
        out.add(E31)
    return out


def straddle_rows(T, n, row_bytes, elem_bytes, seed=0, n_random=12):
    """(t, env) rows of a [T, n, row_bytes] output (t = 0 throughout when T is None) worth comparing env for env: the row
    holding each boundary of crossings() and the rows on either side of it, envs 0, 1, n - 2 and n - 1 at the first and
    the last t, and n_random seeded random rows.  Returns (sorted list of distinct (t, env), {boundary: (t, env) of the
    row holding it})."""
    TT, n = (1 if T is None else int(T)), int(n)
    rows = TT * n
    held = {}
    pick = set()
    for name in sorted(crossings(T, n, row_bytes, elem_bytes)):
        byte = (1 << 31) * (elem_bytes if name == E31 else 1) if name != B32 else 1 << 32
        r = byte // row_bytes
        held[name] = (r // n, r % n)
        pick.update(q for q in (r - 1, r, r + 1) if 0 <= q < rows)
    for t in {0, TT - 1}:
        pick.update(t * n + e for e in (0, 1, n - 2, n - 1) if 0 <= e < n)
    rs = np.random.RandomState(seed)
    pick.update(int(r) for r in rs.randint(0, rows, n_random))
    return sorted((r // n, r % n) for r in pick), held


def twin_bases(envs, n, width=3):
    """env_index_base of the width-env twins that hold every env of `envs` (one twin per env not yet covered; a twin
    starts one env before the env it is built for, clamped into [0, n - width])."""
    bases = []
    for e in sorted(set(int(e) for e in envs)):
        if any(b <= e < b + width for b in bases):
            continue
        bases.append(min(max(e - 1, 0), n - width))
    return bases


# name -> outputs (name, T, n, row_bytes, elem_bytes, boundaries the test exists to cross).  Row sizes: quadrotor
# velocity_control obs 19 float32; state planes 6 float4 per env of n padded to 128; MetaMaze 3-D 128 x 128 RGB frames
# (uint8 or int32 words); 2-D view_grid 5 windows of 11 x 11 float32; god views 480 x 480 RGB; the path record
# [max_steps + 1][n padded to 128] char2.
QUAD_BIG_N = (1 << 25) + 37
QUAD_BENCH_N = 4194304
FRAME_U8, FRAME_I32 = 128 * 128 * 3, 128 * 128 * 3 * 4
PATH_N = 2200000
LARGE_SHAPES = {
    "quad_step_stream": [("obs", None, QUAD_BIG_N, 76, 4, {B31}), ("final_obs", None, QUAD_BIG_N, 76, 4, {B31}),
                         ("planes", None, (QUAD_BIG_N + 127) // 128 * 128, 96, 16, {B31})],
    "quad_step_bench": [("obs", None, QUAD_BENCH_N, 76, 4, set())],
    "quad_rollout": [("obs", 28, QUAD_BENCH_N, 76, 4, {B31, B32, E31}), ("act", 28, QUAD_BENCH_N, 16, 4, set())],
    "quad_rollout_final": [("obs", 14, QUAD_BENCH_N, 76, 4, {B31, B32}),
                           ("final_obs", 14, QUAD_BENCH_N, 76, 4, {B31, B32})],
    "maze3d_step_u8": [("obs", None, 90000, FRAME_U8, 1, {B31, B32, E31}),
                       ("final_obs", None, 90000, FRAME_U8, 1, {B31, B32, E31})],
    "maze3d_rollout_u8": [("obs", 12, 8192, FRAME_U8, 1, {B31, B32, E31}),
                          ("final_obs", 12, 8192, FRAME_U8, 1, {B31, B32, E31})],
    "maze3d_rollout_i32": [("obs", 6, 8192, FRAME_I32, 4, {B31, B32, E31})],
    "mazec3d_rollout_u8": [("obs", 12, 8192, FRAME_U8, 1, {B31, B32, E31})],
    "maze2d_rollout": [("obs", 280, 65536, 11 * 11 * 4, 4, {B31, B32, E31})],
    "god_view": [("views", None, 6300, 480 * 480 * 3, 1, {B31, B32, E31})],
    "path": [("path", 1001, (PATH_N + 127) // 128 * 128, 2, 2, {B31, B32, E31})],
}
