"""CPU tests of the expert restatement (tests/expert_ref.py): the backward search against a forward search on tasks
the reference's sampler draws, the tables against the C oracle's own steps, and the draws' rules."""
import numpy as np
import pytest

from metagym_b200.metamaze import MazeTaskSampler
from oracle.maze_oracle import OracleMaze
import expert_ref as xr

# (n, allow_loops, crowd_ratio, sampler seed)
TASKS = [(7, False, 0.0, 1), (9, True, 0.35, 2), (15, False, 0.0, 3), (15, True, 0.0, 4), (15, True, 0.6, 5),
         (31, False, 0.0, 6), (31, True, 0.35, 7)]


def sampled(n, loops, crowd, seed):
    return MazeTaskSampler(n=n, allow_loops=loops, crowd_ratio=crowd, seed=seed)


def walled_off(n=9):
    """A task with a sealed room (unreachable cells) and the start outside it."""
    walls = np.ones((n, n), np.int32)
    walls[1:-1, 1:-1] = 0
    walls[5, 1:-1] = 1                                 # row 5 seals rows 6..7 off
    return walls, (1, 1), (3, 6)


def all_states(P, n):
    return [(ori, gx, gy) for ori in range(P) for gx in range(n) for gy in range(n)]


@pytest.mark.parametrize("kind", ["2D", "3D"])
@pytest.mark.parametrize("case", TASKS, ids=lambda c: "n%d_loops%d_crowd%.2f" % c[:3])
def test_backward_search_equals_forward_search(kind, case):
    task = sampled(*case)
    walls, goal = np.asarray(task.cell_walls), tuple(task.goal)
    dist, mask = xr.tables(walls, goal, kind)
    n, P = walls.shape[0], xr.planes(kind)
    states = all_states(P, n)
    rng = np.random.RandomState(case[3])
    pick = states if len(states) <= 400 else [states[i] for i in rng.choice(len(states), 400, replace=False)]
    pick.append((0, int(task.start[0]), int(task.start[1])))
    for ori, gx, gy in pick:
        assert dist[ori, gx, gy] == xr.forward_dist(walls, goal, kind, gx, gy, ori), (ori, gx, gy)
    assert dist[0, task.start[0], task.start[1]] < xr.FAR
    # the mask is exactly the set of actions one step closer
    for ori, gx, gy in pick:
        d = int(dist[ori, gx, gy])
        want = 0
        if 0 < d < xr.FAR:
            for a in range(4):
                x, y, o = xr.step_rule(walls, kind, gx, gy, ori, a)
                want |= (int(dist[o, x, y]) == d - 1) << a
        assert mask[ori, gx, gy] == want


@pytest.mark.parametrize("kind", ["2D", "3D"])
def test_unreachable_states(kind):
    walls, start, goal = walled_off()
    dist, mask = xr.tables(walls, goal, kind)
    assert (dist[:, 6:8, 1:-1] == xr.FAR).all() and (mask[:, 6:8, 1:-1] == 0).all()
    assert (dist[:, goal[0], goal[1]] == 0).all() and (mask[:, goal[0], goal[1]] == 0).all()
    free = walls == 0
    free[6:8] = False
    assert (dist[:, free] < xr.FAR).all() and (mask[:, free & (np.arange(9)[:, None] * 9 + np.arange(9) != goal[0] * 9 + goal[1])] != 0).all()


@pytest.mark.parametrize("kind", ["2D", "3D"])
@pytest.mark.parametrize("case", TASKS, ids=lambda c: "n%d_loops%d_crowd%.2f" % c[:3])
def test_expert_reaches_goal_in_dist_steps_on_the_oracle(kind, case):
    """From any free state at distance d, every optimal action keeps the oracle one step closer: the episode ends on
    the goal after exactly d steps and not before."""
    task = sampled(*case)
    walls, goal = np.asarray(task.cell_walls), tuple(task.goal)
    dist, mask = xr.tables(walls, goal, kind)
    n, P = walls.shape[0], xr.planes(kind)
    rng = np.random.RandomState(case[3] + 100)
    free = [s for s in all_states(P, n) if walls[s[1], s[2]] == 0 and 0 < dist[s] < xr.FAR]
    textures = None
    if kind == "3D":
        from metagym_b200.textures import synthetic_textures
        textures = synthetic_textures(seed=0)
    o = OracleMaze(kind, "ESCAPE", max_steps=100000, textures=textures, resolution=(4, 4))
    o.set_task(task)
    o.reset()
    for k in rng.choice(len(free), min(24, len(free)), replace=False):
        ori, gx, gy = free[k]
        o.env.gx, o.env.gy, o.env.ori, o.env.steps = gx, gy, ori, 0
        d = int(dist[ori, gx, gy])
        for step in range(d):
            m = int(mask[o.env.ori if P == 4 else 0, o.env.gx, o.env.gy])
            assert m != 0
            bits = [a for a in range(4) if (m >> a) & 1]
            _, rew, done, _ = o.step(bits[rng.randint(len(bits))], render=False)
            assert done == (step == d - 1), (free[k], step)
        assert (o.env.gx, o.env.gy) == goal and rew == task.step_reward + task.goal_reward


def test_draws():
    rng = np.random.RandomState(0)
    N = 4096
    genv = np.arange(N, dtype=np.int64) + (2 ** 32 - 100)
    mask = rng.randint(0, 16, N).astype(np.uint8)
    seed, t = (0xabc << 32) | 9, 77
    a0 = xr.expert_actions(seed, genv, t, mask, 0.0)
    assert all(((m >> a) & 1) or m == 0 for a, m in zip(a0, mask))
    a1 = xr.expert_actions(seed, genv, t, mask, 1.0)
    assert np.bincount(a1, minlength=4).min() > N // 4 - 200
    mean = xr.expert_actions(seed, genv, t, mask, 0.3, mean=True)
    low = np.array([(int(m) & -int(m)).bit_length() - 1 if m else 0 for m in mask])
    assert np.array_equal(mean, low)
    # the rules written out on the words: uniform choice in the choice set, exploration below eps
    r = xr.expert_words(seed, genv, t).astype(np.uint64)
    u = (r[:, 0] >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    a3 = xr.expert_actions(seed, genv, t, mask, 0.3)
    for i in range(N):
        c = 15 if (u[i] < np.float32(0.3) or mask[i] == 0) else int(mask[i])
        bits = [a for a in range(4) if (c >> a) & 1]
        assert a3[i] == bits[(int(r[i, 1]) * len(bits)) >> 32]
    explored = u < np.float32(0.3)
    assert 0.27 < explored.mean() < 0.33
