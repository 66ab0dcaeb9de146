"""CPU: pin the maze oracle (oracle/maze_oracle.c) against golden vectors recorded from the unmodified reference.
Everything here is integer / exact: grid state, done flags, float64 rewards and life, float32 2-D observations and the
int32 raycast images must match bit for bit."""
import numpy as np
import pytest

from oracle.maze_oracle import OracleMaze
from metagym_b200.textures import synthetic_textures
from util import MAZE_CASES, OPTICS_CASES, OPTICS_CONT_CASES, maze_case, optics_kw


def replay(case, make_env):
    env = make_env()
    env.set_task(case["task"])
    obs0 = env.reset()
    yield ("reset", -1, obs0, None, None, None)
    kept = {int(t): k for k, t in enumerate(case["obs_idx"])}
    for t, a in enumerate(case["act"]):
        obs, rew, done, info = env.step(int(a))
        yield ("step", t, obs, rew, done, (env.agent, env.life, kept.get(t)))
        if done:
            env.reset()


@pytest.fixture(scope="module")
def geom_golden():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maze_geom_golden.npz"))


@pytest.fixture(scope="module")
def optics_golden():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maze_optics_golden.npz"))


GEOM_CASES = ["g3d_surv", "g3d_esc"]      # non-default cell / wall / eye heights (tests/golden/gen_maze_geom.py)


@pytest.mark.parametrize("name", MAZE_CASES + GEOM_CASES + OPTICS_CASES)
def test_oracle_matches_reference_episode(maze_golden, geom_golden, optics_golden, name):
    c = maze_case(geom_golden if name in GEOM_CASES else optics_golden if name in OPTICS_CASES else maze_golden, name)
    tex = synthetic_textures(seed=0)

    def make():
        return OracleMaze(c["kind"], c["task_type"], c["max_steps"], c["view_grid"], c["resolution"], textures=tex,
                          **optics_kw(c))

    n_frames = 0
    for what, t, obs, rew, done, extra in replay(c, make):
        if what == "reset":
            assert np.array_equal(np.asarray(obs), c["reset_obs"].astype(obs.dtype))
            assert obs.dtype == (np.float32 if c["kind"] == "2D" else np.int32)
            continue
        agent, life, k = extra
        assert rew == c["rew"][t], (t, rew, c["rew"][t])
        assert done == bool(c["done"][t]), t
        assert tuple(agent) == tuple(int(x) for x in c["agent"][t]), t
        if c["task_type"] == "SURVIVAL":
            assert life == c["life"][t], t
        if k is not None:
            ref = c["obs"][k]
            if c["kind"] == "2D":
                assert obs.dtype == np.float32 and np.array_equal(obs, ref), t
            else:
                assert np.array_equal(obs, ref.astype(np.int32)), (t, int((obs != ref).sum()))
            n_frames += 1
    assert n_frames == len(c["obs_idx"])
    if name in OPTICS_CASES and c["task_type"] == "SURVIVAL":
        assert (c["done"] & (c["life"] < 0)).any()        # a death: the terminal frame of a dead agent is pinned


def test_values_can_exceed_uint8(maze_golden):
    """Near-floor pixels are lit with v_screen / l_focal > 1 (ray_caster_utils.py:99,114): with a bright ground texture
    the reference's int32 image exceeds 255, which is why the engine offers an exact int32 mode next to the clamped
    uint8 one (MGB_OBS_I32 / MGB_OBS_U8)."""
    c = maze_case(maze_golden, "m3d_big")
    grounds, ceil = synthetic_textures(seed=0)
    grounds = grounds.copy()
    grounds[0] = 255
    env = OracleMaze("3D", "ESCAPE", 200, 1, (128, 128), textures=(grounds, ceil))
    env.set_task(c["task"])
    obs = env.reset()
    assert 300 < int(obs.max()) < 400


@pytest.mark.parametrize("name", ["c3d_surv", "c3d_esc", "gc3d"] + OPTICS_CONT_CASES)
def test_continuous_maze_oracle_matches_reference(cont_golden, geom_golden, optics_golden, name):
    """MetaMazeContinuous3D (SURVEY.md 8f row 2): float32 positions, float64 headings, rewards, dones and every
    recorded frame of the reference episodes, bit for bit (numba/numpy typing of dynamics.py reproduced in C)."""
    from util import cont_case
    c = cont_case(geom_golden if name == "gc3d" else optics_golden if name in OPTICS_CONT_CASES else cont_golden, name)
    tex = synthetic_textures(seed=0)
    env = OracleMaze("C3D", c["task_type"], c["max_steps"], 1, c["resolution"], textures=tex, **optics_kw(c))
    env.set_task(c["task"])
    assert np.array_equal(env.reset(), c["reset_obs"].astype(np.int32))
    kept = {int(t): k for k, t in enumerate(c["obs_idx"])}
    for t, a in enumerate(c["act"]):
        obs, rew, done, info = env.step(a)
        pos, ori = env.pose
        assert np.array_equal(pos, c["pos"][t]) and ori == c["ori"][t], t
        assert rew == c["rew"][t] and done == bool(c["done"][t]) and info["steps"] == int(c["steps"][t]), t
        assert tuple(env.agent[:2]) == tuple(int(x) for x in c["grid"][t])
        if c["task_type"] == "SURVIVAL":
            assert env.life == c["life"][t]
        if t in kept:
            assert np.array_equal(obs, c["obs"][kept[t]].astype(np.int32)), t
        if done:
            env.reset()
    assert c["done"].sum() >= 1 and (c["rew"] > 0).sum() >= 1


def test_oracle_vs_reference_real_textures():
    """The reference renderer with its own PNG textures (decoded into the fixture) vs the oracle: one 60-step episode
    recorded by tests/golden/gen_maze_real_textures.py; every frame bit for bit (reset frame pixel for pixel, step frames
    by the SHA-256 of their int32 bytes), rewards and dones exactly."""
    import hashlib
    import os
    from util import task_from_arrays
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maze_real_textures_golden.npz"))
    task = task_from_arrays(g["task.walls"], g["task.texts"], g["task.food"], g["task.interval"], g["task.scalars"])
    ora = OracleMaze("3D", "SURVIVAL", 500, 1, (128, 128), textures=(g["grounds"], g["ceil"]))
    ora.set_task(task)
    o0 = ora.reset()
    assert np.array_equal(o0, g["reset_obs"].astype(np.int32)), int((o0 != g["reset_obs"]).sum())
    for t, a in enumerate(g["act"]):
        o2, r2, d2, _ = ora.step(int(a))
        digest = hashlib.sha256(np.ascontiguousarray(o2, dtype=np.int32).tobytes()).digest()
        assert digest == g["sha256"][t].tobytes(), t
        assert r2 == g["rew"][t] and d2 == bool(g["done"][t]), t


def dda_crossings(pos, n, cell_size, cos_ori, sin_ori, walls, transp, max_vision):
    """DDA_2D (ray_caster_utils.py:11-62) in plain numpy scalars -> (transparent crossings it lists, whether the column is
    painted at all, i.e. the ray meets a wall within max_vision: :162-163)."""
    i, j = int(pos[0] / cell_size), int(pos[1] / cell_size)
    ddx = 1.0e+6 if abs(cos_ori) < 1.0e-6 else abs(cell_size / cos_ori)
    ddy = 1.0e+6 if abs(sin_ori) < 1.0e-6 else abs(cell_size / sin_ori)
    d_x = ((i + 1) * cell_size - pos[0]) if cos_ori > 0 else (i * cell_size - pos[0])
    d_y = ((j + 1) * cell_size - pos[1]) if sin_ori > 0 else (j * cell_size - pos[1])
    sx = 1.0e+6 if abs(cos_ori) < 1.0e-6 else d_x / cos_ori
    sy = 1.0e+6 if abs(sin_ori) < 1.0e-6 else d_y / sin_ori
    di, dj = (1 if cos_ori > 0 else -1), (1 if sin_ori > 0 else -1)
    count = 1 if transp[i, j] > 0.01 else 0
    dist = 0.0
    while dist < max_vision:
        if sx < sy:
            i += di
            sy -= sx
            dist += sx
            sx = ddx
        else:
            j += dj
            sx -= sy
            dist += sy
            sy = ddy
        if not (0 <= i < n and 0 <= j < n):
            if not (0 <= i < n) and not (0 <= j < n):
                return count, False
            continue
        count += transp[i, j] > 0.01
        if walls[i, j] > 0:
            break
    return count, dist <= max_vision


def column_crossings(task, pos, ori, res_h, max_vision, fov, l_focal=0.20):
    """Crossings per screen column for the agent at `pos` / `ori` with every food present (the column tables of
    maze_view, ray_caster_utils.py:68-92, stored as float32 like the reference's arrays)."""
    walls, transp = np.asarray(task.cell_walls), np.asarray(task.food_rewards)
    n = walls.shape[0]
    pixel_factor = 2.0 * np.tan(fov / 2) * l_focal / res_h / l_focal
    s_ori, c_ori = np.sin(ori), np.cos(ori)
    tan_hp = (-0.5 - res_h / 2) * pixel_factor
    out = []
    for _ in range(res_h):
        tan_hp += pixel_factor
        cos_hp = np.sqrt(1.0 / (1.0 + tan_hp ** 2))
        sin_hp = tan_hp * cos_hp
        sin_abs = float(np.float32(sin_hp * c_ori + cos_hp * s_ori))
        cos_abs = float(np.float32(cos_hp * c_ori - sin_hp * s_ori))
        cnt, painted = dda_crossings(pos, n, task.cell_size, cos_abs, sin_abs, walls, transp, max_vision)
        out.append(cnt if painted else 0)
    return np.array(out)


@pytest.mark.parametrize("name", ["xings", "xings_c"])
def test_xings_fixture_has_columns_past_48_crossings(optics_golden, name):
    """The xings arena's start frame (recorded as reset_obs, every food present) has painted columns listing more than 48
    transparent crossings -- more than the renderer once kept per column -- and never more than a ray can enter cells of
    an n x n grid (2 n - 1), the bound the renderer's lists are sized by."""
    from util import cont_case
    c = (maze_case if name == "xings" else cont_case)(optics_golden, name)
    t = c["task"]
    n = np.shape(t.cell_walls)[0]
    pos = [t.start[0] * t.cell_size + 0.5 * t.cell_size, t.start[1] * t.cell_size + 0.5 * t.cell_size]
    counts = column_crossings(t, pos, 0.0, c["resolution"][0], *optics_kw(c).values())
    assert 48 < counts.max() <= 2 * n - 1, counts.max()
    assert (counts > 48).sum() >= 2, counts
