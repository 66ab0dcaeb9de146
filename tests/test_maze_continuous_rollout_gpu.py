"""GPU tests of the fused continuous-maze rollout (mgb_maze_rollout, maze3d_kernel<false, true>): T steps in one
launch equal T step() calls bit for bit, device-drawn actions equal their NumPy restatement, every env equals its own CPU
oracle, sharding does not change a trajectory, and misuse is refused."""
import itertools

import numpy as np
import pytest

from maze_continuous_draws import maze_continuous_rollout_actions
from util import cont_case, task_from_arrays

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def dense_tasks(g):
    """Four 15x15 tasks of maze_golden.npz with food on every free cell within 4 cells of the start (the start cell
    included) and a food interval of 3, so that random walks eat food every few steps; task 0's goal is its start
    cell, so ESCAPE envs on it finish (with the goal reward) on every step."""
    tasks = []
    for k in range(4):
        t = task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                             g["tasks15.interval"][k], g["tasks15.scalars"][k])
        walls = np.asarray(t.cell_walls)
        i, j = np.indices(walls.shape)
        near = (walls == 0) & (np.abs(i - t.start[0]) + np.abs(j - t.start[1]) <= 4)
        food = np.where(near, 0.2 + 0.05 * ((i + j) % 5), 0.0)
        t = t._replace(food_rewards=food, food_interval=np.where(near, 3, 0).astype(np.int32))
        tasks.append(t._replace(goal=t.start) if k == 0 else t)
    return tasks


def make(textures, tasks, n, res, task_type="SURVIVAL", obs_dtype="uint8", auto_reset=True, max_steps=10,
         env_index_base=0):
    from metagym_b200 import BatchedMetaMazeContinuous3D
    env = BatchedMetaMazeContinuous3D(resolution=res, max_steps=max_steps, task_type=task_type, num_envs=n,
                                      squeeze=False, auto_reset=auto_reset, obs_dtype=obs_dtype, textures=textures,
                                      env_index_base=env_index_base)
    env.set_task(tasks)
    env.reset()
    return env


def assert_same_state(torch, a_env, b_env):
    pa, pb = a_env.pose(), b_env.pose()
    sa, sb = a_env.agent_state(), b_env.agent_state()
    assert torch.equal(pa[0], pb[0]) and torch.equal(pa[1], pb[1])
    assert torch.equal(sa[0], sb[0]) and torch.equal(sa[1], sb[1])


# task type x obs dtype x auto_reset x MGB_MAZE_RENDER_PIPE, each with one of the nine (screen, envs) shapes in turn so that
# every shape runs: ragged and non-square screens, and envs below and above the SM count (a CTA owning several envs)
SHAPES = list(itertools.product([(40, 24), (64, 48), (128, 128)], [9, 37, 300]))
CASES = [combo + SHAPES[k % len(SHAPES)] for k, combo in
         enumerate(itertools.product(["SURVIVAL", "ESCAPE"], ["uint8", "int32", "float32"], [True, False], ["1", "0"]))]


@pytest.mark.parametrize("task_type,obs_dtype,auto_reset,pipe,res,n", CASES)
def test_rollout_equals_single_steps(torch_mod, maze_golden, textures, monkeypatch, task_type, obs_dtype, auto_reset,
                                     pipe, res, n):
    """rollout(T, actions) on one handle == T step(actions[t]) on an identical one: every frame, reward and done, then
    the final pose and agent state, then one more step() on both.  Episodes end and food is eaten inside the chunk."""
    torch = torch_mod
    monkeypatch.setenv("MGB_MAZE_RENDER_PIPE", pipe)       # read when the handle is created
    tasks = dense_tasks(maze_golden)
    a_env = make(textures, tasks, n, res, task_type, obs_dtype, auto_reset)
    b_env = make(textures, tasks, n, res, task_type, obs_dtype, auto_reset)
    T = 24
    rng = np.random.RandomState(n + res[0])
    act = torch.as_tensor(rng.uniform(-1.3, 1.3, (T, n, 2)).astype(np.float32)).cuda()   # clipped by the kernel
    out = a_env.rollout(T, actions=act)
    assert out["obs"].dtype == b_env._obs.dtype and out["obs"].shape == (T, n) + res + (3,) and out["act"] is None
    n_done = n_food = 0
    for t in range(T):
        obs, rew, done, _ = b_env.step(act[t])
        assert torch.equal(out["obs"][t], obs), (t, int((out["obs"][t] != obs).sum()))
        assert torch.equal(out["rew"][t], rew) and torch.equal(out["done"][t].bool(), done), t
        n_done += int(done.sum())
        n_food += int((rew > 0).sum())
    assert n_done > 0 and n_food > 0
    assert_same_state(torch, a_env, b_env)
    last = torch.as_tensor(rng.uniform(-1.0, 1.0, (n, 2)).astype(np.float32)).cuda()
    ra, rb = a_env.step(last), b_env.step(last)
    assert torch.equal(ra[0], rb[0]) and torch.equal(ra[1], rb[1]) and torch.equal(ra[2], rb[2])
    a_env.close(); b_env.close()


@pytest.mark.parametrize("pipe", ["1", "0"])
def test_drawn_actions_restated_and_replayed(torch_mod, maze_golden, textures, monkeypatch, pipe):
    """Two consecutive drawn chunks after a given-action chunk: the drawn actions equal
    maze_continuous_rollout_actions(seed, genv, t_base + t) bit for bit (the given chunk advanced t_base too),
    and replaying them through step() on a twin handle reproduces every frame, reward and done."""
    torch = torch_mod
    monkeypatch.setenv("MGB_MAZE_RENDER_PIPE", pipe)
    tasks = dense_tasks(maze_golden)
    n, res, T0 = 150, (64, 48), 5
    a_env = make(textures, tasks, n, res, env_index_base=1000)
    b_env = make(textures, tasks, n, res, env_index_base=1000)
    given = torch.as_tensor(np.random.RandomState(5).uniform(-1, 1, (T0, n, 2)).astype(np.float32)).cuda()
    a_env.rollout(T0, actions=given.reshape(T0, -1))          # any shape that reshapes to [T, N, 2]
    for t in range(T0):
        b_env.step(given[t])
    o1 = a_env.rollout(11, act_seed=2 ** 40 + 9, want_actions=True)
    o2 = a_env.rollout(8, act_seed=2 ** 40 + 9, want_actions=True)
    drawn = torch.cat([o1["act"], o2["act"]])
    assert drawn.dtype == torch.float32 and drawn.shape == (19, n, 2)
    genv = 1000 + np.arange(n)
    for t in range(19):
        assert np.array_equal(drawn[t].cpu().numpy(), maze_continuous_rollout_actions(2 ** 40 + 9, genv, T0 + t)), t
    assert float(drawn.min()) >= -1.0 and float(drawn.max()) < 1.0
    obs_r, rew_r, done_r = (torch.cat([o1[k], o2[k]]) for k in ("obs", "rew", "done"))
    for t in range(19):
        obs, rew, done, _ = b_env.step(drawn[t])
        assert torch.equal(obs_r[t], obs) and torch.equal(rew_r[t], rew) and torch.equal(done_r[t].bool(), done), t
    assert_same_state(torch, a_env, b_env)
    a_env.close(); b_env.close()


def test_rollout_vs_oracle(torch_mod, maze_golden, textures):
    """64 envs over 4 tasks (the tasks of test_continuous_maze_random_batch_vs_oracle), drawn actions, auto-reset, two
    chunks: every env's frames, rewards, dones and final pose equal its own CPU oracle instance stepped with the
    restated draws."""
    from oracle.maze_oracle import OracleMaze
    g = maze_golden
    tasks = [task_from_arrays(g["tasks15.walls"][k], g["tasks15.texts"][k], g["tasks15.food"][k],
                              g["tasks15.interval"][k] // 10, g["tasks15.scalars"][k]) for k in range(4)]
    n, max_steps, res, seed = 64, 25, (40, 24), 123
    env = make(textures, tasks, n, res, obs_dtype="int32", max_steps=max_steps)
    oracles = []
    for e in range(n):
        o = OracleMaze("C3D", "SURVIVAL", max_steps, 1, res, textures=textures)
        o.set_task(tasks[e % 4])
        o.reset()
        oracles.append(o)
    t_base = 0
    for T in (35, 25):
        out = env.rollout(T, act_seed=seed)
        obs, rew, done = out["obs"].cpu().numpy(), out["rew"].cpu().numpy(), out["done"].cpu().numpy()
        for t in range(T):
            act = maze_continuous_rollout_actions(seed, np.arange(n), t_base + t)
            for e in range(n):
                o2, r2, d2, _ = oracles[e].step(act[e])
                assert rew[t, e] == r2 and bool(done[t, e]) == d2, (t_base + t, e)
                if d2:
                    o2 = oracles[e].reset()
                assert np.array_equal(obs[t, e], o2), (t_base + t, e, int((obs[t, e] != o2).sum()))
        t_base += T
    pos, ori = env.pose()
    pos, ori = pos.cpu().numpy(), ori.cpu().numpy()
    for e in range(n):
        p2, a2 = oracles[e].pose
        assert np.array_equal(pos[e], p2) and ori[e] == a2, e
    env.close()


def test_rollout_vs_oracle_non_default_geometry(torch_mod, geom_golden, textures):
    """The continuous task of maze_geom_golden.npz (cell 3.0 / wall 4.0 / eye 2.2: the renderer's division paths),
    drawn actions, auto-reset: every env equals its oracle instance bit for bit."""
    from oracle.maze_oracle import OracleMaze
    c = cont_case(geom_golden, "gc3d")
    n, T, seed = 6, 40, 77
    env = make(textures, c["task"], n, c["resolution"], c["task_type"], "int32", max_steps=c["max_steps"])
    out = env.rollout(T, act_seed=seed)
    obs, rew, done = out["obs"].cpu().numpy(), out["rew"].cpu().numpy(), out["done"].cpu().numpy()
    for e in range(n):
        o = OracleMaze("C3D", c["task_type"], c["max_steps"], 1, c["resolution"], textures=textures)
        o.set_task(c["task"])
        o.reset()
        for t in range(T):
            o2, r2, d2, _ = o.step(maze_continuous_rollout_actions(seed, [e], t)[0])
            assert rew[t, e] == r2 and bool(done[t, e]) == d2, (t, e)
            if d2:
                o2 = o.reset()
            assert np.array_equal(obs[t, e], o2), (t, e, int((obs[t, e] != o2).sum()))
    env.close()


def test_sharding_invariance(torch_mod, maze_golden, textures):
    """Handles with env_index_base 0 and n/2, each over its half, produce the same drawn-action rollout as one handle
    over all n envs: frames, rewards, dones, actions and final poses."""
    torch = torch_mod
    tasks = dense_tasks(maze_golden)
    n, res, T = 40, (40, 24), 20
    full = make(textures, tasks, n, res)
    halves = [make(textures, tasks, n // 2, res, env_index_base=b) for b in (0, n // 2)]
    ref = full.rollout(T, act_seed=31, want_actions=True)
    parts = [h.rollout(T, act_seed=31, want_actions=True) for h in halves]
    for k in ("obs", "rew", "done", "act"):
        assert torch.equal(ref[k], torch.cat([p[k] for p in parts], dim=1)), k
    pos, ori = full.pose()
    assert torch.equal(pos, torch.cat([h.pose()[0] for h in halves])) and torch.equal(ori, torch.cat([h.pose()[1] for h in halves]))
    full.close()
    for h in halves:
        h.close()


def test_rollout_errors(torch_mod, maze_golden, textures):
    """T = 0, a rollout before reset(), output mirrors or multicast switched on, and a handle without a task are refused
    with a message; the rollout works again afterwards, through Python and through the C call."""
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeContinuous3D, MgbError, _lib
    tasks = dense_tasks(maze_golden)
    n, res = 4, (40, 24)
    env = BatchedMetaMazeContinuous3D(resolution=res, max_steps=10, num_envs=n, squeeze=False, textures=textures)
    env.set_task(tasks)
    with pytest.raises(Exception, match="Must \"reset\" before doing any actions"):
        env.rollout(3)
    env.reset()
    with pytest.raises(MgbError, match="T must be positive"):
        env.rollout(0)
    delta = np.array([1 << 20], dtype=np.int64)
    _lib.check(env._lib.mgb_maze_set_mirrors(env._h, 1, delta.ctypes.data))
    with pytest.raises(MgbError, match="mirrors are not implemented for the 3-D rollouts"):
        env.rollout(3)
    _lib.check(env._lib.mgb_maze_set_multicast(env._h, 1 << 20))
    with pytest.raises(MgbError, match="mirrors are not implemented for the 3-D rollouts"):
        env.rollout(3)
    _lib.check(env._lib.mgb_maze_set_mirrors(env._h, 0, None))
    out = env.rollout(3)
    _lib.check(env._lib.mgb_maze_rollout(env._h, 3, None, 0, None, out["obs"].data_ptr(), out["rew"].data_ptr(),
                                         out["done"].data_ptr(), None, None, None, 0, env._stream()))
    torch.cuda.synchronize()
    env.close()
    bare = BatchedMetaMazeContinuous3D(resolution=res, max_steps=10, num_envs=n, squeeze=False, textures=textures)
    bare._create(15)                                          # a handle with textures but no task table
    with pytest.raises(MgbError, match="set_task"):
        _lib.check(bare._lib.mgb_maze_rollout(bare._h, 3, None, 0, None, out["obs"].data_ptr(), out["rew"].data_ptr(),
                                              out["done"].data_ptr(), None, None, None, 0, bare._stream()))
    bare.close()
