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
