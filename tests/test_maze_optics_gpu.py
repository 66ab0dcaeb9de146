"""GPU tests of the 3-D MetaMaze renderers at non-default optics and screen shapes (tests/golden/maze_optics_golden.npz,
recorded from the unmodified reference by gen_maze_optics.py): every discrete step path, the continuous step and the
fused rollouts, against the reference episodes and against the CPU oracle (oracle/maze_oracle.c), bit for bit.

The optics (max_vision_range, fol_angle) size the crossing lists, the fog tables and the screen / column tables; the
screen shape selects the pose-cache paths (4-pixel groups, baked and variant frames, the 16-pixel compose loop, the fused
uint8 step).  Case `xings` has columns with more than 48 transparent crossings, every one of which the reference
blends."""
import os

import numpy as np
import pytest

from util import OPTICS_CASES, OPTICS_CONT_CASES, cont_case, maze_case, optics_kw

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


@pytest.fixture(scope="module")
def optics_golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "maze_optics_golden.npz"))


def env_optics(c):
    return dict(max_vision_range=float(c["optics"][0]), fol_angle=float(c["optics"][1]))


def as_dtype(frame, dtype):
    """A reference / oracle int32 frame in an obs dtype (uint8 = min(value, 255))."""
    frame = np.asarray(frame).astype(np.int32)
    if dtype == "uint8":
        return np.minimum(frame, 255).astype(np.uint8)
    return frame.astype(np.float32) if dtype == "float32" else frame


def packed_cache_holds(c, textures):
    """The pose cache packs a pixel into 10 bits per channel.  Floor and ceiling texels are lit by v_screen / l_focal
    (ray_caster_utils.py:99,132), up to tan(fov / 2) * (res_v - 1) / res_h: on tall screens that can exceed 1023, and
    those render directly."""
    res_h, res_v = c["resolution"]
    brightest = max(int(textures[0].max()), int(textures[1].max()))
    return np.tan(float(c["optics"][1]) / 2) * (res_v - 1) / res_h * brightest < 1024.0


# path id -> (obs dtype, constructor kwargs, environment)
PATHS = {
    "cache_i32": ("int32", {}, {}),
    "cache_u8": ("uint8", {}, {}),
    "cache_u8_unfused": ("uint8", {}, {"MGB_MAZE_FUSED_STEP": "0"}),
    "cache_f32": ("float32", {}, {}),
    "direct_i32": ("int32", {"cache": False}, {}),
    "direct_u8": ("uint8", {"cache": False}, {}),
}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("name", OPTICS_CASES)
def test_optics_reference_episode(torch_mod, optics_golden, textures, monkeypatch, name, n, path):
    """Replay the recorded reference episode on n identical envs (manual reset after done, like the reference user):
    rewards, dones, agent state, life and every recorded frame bit for bit, on the path the parameters select."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    if path == "cache_u8_unfused" and name not in ("o3d_wide", "xings"):
        pytest.skip("the fused uint8 step takes 16-row, 128-pixel screens: o3d_wide and xings")
    c = maze_case(optics_golden, name)
    dtype, kw, envvars = PATHS[path]
    monkeypatch.setenv("MGB_MAZE_FUSED_STEP", "1")
    for k, v in envvars.items():
        monkeypatch.setenv(k, v)
    env = BatchedMetaMazeDiscrete3D(resolution=c["resolution"], max_steps=c["max_steps"], task_type=c["task_type"],
                                    num_envs=n, squeeze=False, textures=textures, obs_dtype=dtype, **env_optics(c), **kw)
    env.set_task(c["task"])
    obs0 = env.reset().cpu().numpy()
    for k in range(n):
        assert np.array_equal(obs0[k], as_dtype(c["reset_obs"], dtype)), (k, int((obs0[k] != c["reset_obs"]).sum()))
    info = env.cache_info()
    assert info["in_use"] == (path.startswith("cache") and packed_cache_holds(c, textures)), info
    if name == "xings" and path.startswith("direct"):
        assert info["hits_in_global"]          # 61 crossings x 128 columns per record set: lists in global scratch
    kept = {int(t): k for k, t in enumerate(c["obs_idx"])}
    for t, a in enumerate(c["act"]):
        obs, rew, done, _ = env.step(torch.full((n,), int(a), dtype=torch.int32, device="cuda"))
        ag, life = env.agent_state()
        ag, life, rew_h, done_h = ag.cpu().numpy(), life.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        for k in range(n):
            assert rew_h[k] == c["rew"][t] and bool(done_h[k]) == bool(c["done"][t]), (t, k)
            assert tuple(ag[k]) == tuple(int(x) for x in c["agent"][t]), (t, ag[k], c["agent"][t])
            if c["task_type"] == "SURVIVAL":
                assert life[k] == c["life"][t], t
        if t in kept:
            o, ref = obs.cpu().numpy(), as_dtype(c["obs"][kept[t]], dtype)
            for k in range(n):
                assert np.array_equal(o[k], ref), (t, k, int((o[k] != ref).any(-1).sum()))
        if c["done"][t]:
            env.reset()
    env.close()


@pytest.mark.parametrize("name", OPTICS_CONT_CASES)
def test_optics_continuous_reference_episode(torch_mod, optics_golden, textures, name):
    """MetaMazeContinuous3D with the case's optics: float32 positions, float64 headings, rewards, dones, life and every
    recorded frame bit for bit."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D
    c = cont_case(optics_golden, name)
    n = 3
    env = BatchedMetaMazeContinuous3D(resolution=c["resolution"], max_steps=c["max_steps"], task_type=c["task_type"],
                                      num_envs=n, squeeze=False, textures=textures, **env_optics(c))
    env.set_task(c["task"])
    obs0 = env.reset().cpu().numpy()
    assert np.array_equal(obs0[n - 1], c["reset_obs"].astype(np.int32))
    kept = {int(t): k for k, t in enumerate(c["obs_idx"])}
    for t, a in enumerate(c["act"]):
        obs, rew, done, _ = env.step(torch.as_tensor(np.tile(a, (n, 1))).cuda())
        pos, ori = env.pose()
        _, life = env.agent_state()
        pos, ori, life = pos.cpu().numpy(), ori.cpu().numpy(), life.cpu().numpy()
        for k in range(n):
            assert np.array_equal(pos[k], c["pos"][t]) and ori[k] == c["ori"][t], (t, k)
            assert float(rew[k]) == c["rew"][t] and bool(done[k]) == bool(c["done"][t]), (t, k)
            assert life[k] == c["life"][t], (t, k)
        if t in kept:
            o, ref = obs.cpu().numpy(), c["obs"][kept[t]].astype(np.int32)
            for k in range(n):
                assert np.array_equal(o[k], ref), (t, k, int((o[k] != ref).any(-1).sum()))
        if c["done"][t]:
            env.reset()
    env.close()


def batch_tasks(c, task_type):
    """Four tasks for a random batch: three sampled 9x9 mazes and one with the 1.5 / 2.5 / 0.9 geometry (xings: its own
    arena four times).  SURVIVAL: step rewards that end episodes by death (tasks 0, 2) and by the step limit (1, 3).
    ESCAPE: the goal of tasks 0 and 2 is next to the start, so that random walks reach it."""
    from metagym_b200 import MazeTaskSampler
    if c["task"].cell_size == 0.25:
        tasks = [c["task"]] * 4
    else:
        rs = np.random.RandomState(int(c["resolution"][0] * 1000 + c["resolution"][1]))
        tasks = [MazeTaskSampler(n=9, allow_loops=True, crowd_ratio=0.3, food_density=0.08, food_interval=5, rng=rs)
                 for _ in range(3)]
        tasks.append(MazeTaskSampler(n=9, allow_loops=True, crowd_ratio=0.3, food_density=0.08, food_interval=5,
                                     cell_size=1.5, wall_height=2.5, agent_height=0.9, rng=rs))
    out = []
    for k, t in enumerate(tasks):
        if task_type == "SURVIVAL":
            t = t._replace(step_reward=(-0.15, -0.01, -0.15, -0.01)[k])
        elif k % 2 == 0:
            sx, sy = t.start
            w = np.asarray(t.cell_walls)
            t = t._replace(goal=[(sx + dx, sy + dy) for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1))
                                 if w[sx + dx, sy + dy] == 0][0])
        out.append(t)
    return out


BATCH_CASES = ["o3d_near", "o3d_wide", "o3d_esc", "o3d_tall", "o3d_dot1", "o3d_dot3", "xings", "oc3d"]


@pytest.mark.parametrize("name", BATCH_CASES)
def test_optics_random_batch_vs_oracle(torch_mod, optics_golden, textures, name):
    """40 envs over four tasks with the case's optics and screen, random actions, auto_reset and final_obs: every
    frame, reward and done, the terminal frame of every finished env and its truncated flag equal each env's own oracle."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    from oracle.maze_oracle import OracleMaze
    cont = name in OPTICS_CONT_CASES
    c = (cont_case if cont else maze_case)(optics_golden, name)
    task_type, res = c["task_type"], c["resolution"]
    tasks = batch_tasks(c, task_type)
    n, T, max_steps = 40, (30 if name == "xings" else 40), 14
    cls = BatchedMetaMazeContinuous3D if cont else BatchedMetaMazeDiscrete3D
    env = cls(resolution=res, max_steps=max_steps, task_type=task_type, num_envs=n, squeeze=False, auto_reset=True,
              final_obs=True, textures=textures, **env_optics(c))
    env.set_task(tasks)
    oracles = []
    for e in range(n):
        o = OracleMaze("C3D" if cont else "3D", task_type, max_steps, 1, res, textures=textures, **optics_kw(c))
        o.set_task(tasks[e % 4])
        oracles.append(o)
    obs = env.reset().cpu().numpy()
    for e in range(n):
        assert np.array_equal(obs[e], oracles[e].reset()), e
    rng = np.random.RandomState(5)
    ends = {"death": 0, "goal": 0, "limit": 0}
    for t in range(T):
        act = rng.uniform(-1.3, 1.3, (n, 2)).astype(np.float32) if cont else rng.randint(0, 4, n).astype(np.int32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        obs, rew, done = obs.cpu().numpy(), rew.cpu().numpy(), done.cpu().numpy()
        fin, trunc = env.final_observation.cpu().numpy(), env.truncated.cpu().numpy()
        for e in range(n):
            o = oracles[e]
            o2, r2, d2, _ = o.step(act[e])
            assert rew[e] == r2 and bool(done[e]) == d2, (t, e)
            if not d2:
                assert not trunc[e] and np.array_equal(obs[e], o2), (t, e)
                continue
            if task_type == "SURVIVAL":
                ended = o.life < 0
            else:
                ended = (o.env.gx, o.env.gy) == tuple(tasks[e % 4].goal)
            over = o.env.steps > max_steps - 1
            assert bool(trunc[e]) == (over and not ended), (t, e)
            ends["limit" if not ended else ("death" if task_type == "SURVIVAL" else "goal")] += 1
            assert np.array_equal(fin[e], o2), (t, e, int((fin[e] != o2).any(-1).sum()))
            assert np.array_equal(obs[e], o.reset()), (t, e)
    assert ends["limit"] > 0 and ends["death" if task_type == "SURVIVAL" else "goal"] > 0, ends
    env.close()


@pytest.mark.parametrize("name,obs_dtype", [("o3d_wide", "uint8"), ("o3d_near", "int32"), ("o3d_esc", "uint8"),
                                            ("o3d_dot3", "uint8"), ("xings", "uint8"), ("oc3d", "int32"),
                                            ("xings_c", "uint8")])
def test_optics_rollout_equals_steps(torch_mod, optics_golden, textures, name, obs_dtype):
    """rollout(T, final_obs=True) -- the discrete pose-cache rollout, rollout_continuous for the continuous env -- equals
    the stream of T step() calls with the same actions: frames, rewards, dones, terminal frames and truncated flags."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    cont = name in OPTICS_CONT_CASES
    c = (cont_case if cont else maze_case)(optics_golden, name)
    tasks = batch_tasks(c, c["task_type"])
    n, T = 24, 30
    cls = BatchedMetaMazeContinuous3D if cont else BatchedMetaMazeDiscrete3D

    def fresh():
        env = cls(resolution=c["resolution"], max_steps=12, task_type=c["task_type"], num_envs=n, squeeze=False,
                  auto_reset=True, final_obs=True, obs_dtype=obs_dtype, textures=textures, **env_optics(c))
        env.set_task(tasks)
        env.reset()
        return env

    a_env, b_env = fresh(), fresh()
    rng = np.random.RandomState(9)
    if cont:
        act = torch.as_tensor(rng.uniform(-1.3, 1.3, (T, n, 2)).astype(np.float32)).cuda()
    else:
        act = torch.as_tensor(rng.randint(0, 4, (T, n)), dtype=torch.int32).cuda()
    out = a_env.rollout(T, actions=act, final_obs=True)
    n_done = 0
    for t in range(T):
        obs, rew, done, _ = b_env.step(act[t])
        assert torch.equal(out["obs"][t], obs), (t, int((out["obs"][t] != obs).sum()))
        assert torch.equal(out["rew"][t], rew) and torch.equal(out["done"][t].bool(), done.bool()), t
        assert torch.equal(out["truncated"][t].bool(), b_env.truncated), t
        d = done.bool()
        assert torch.equal(out["final_obs"][t][d], b_env.final_observation[d]), t
        n_done += int(d.sum())
    assert n_done > 0
    if not cont:
        assert a_env.cache_info()["in_use"]
    sa, sb = a_env.agent_state(), b_env.agent_state()
    assert torch.equal(sa[0], sb[0]) and torch.equal(sa[1], sb[1])
    a_env.close()
    b_env.close()
