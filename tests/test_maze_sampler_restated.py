"""CPU checks of maze_sampler_draws, the NumPy restatement of the device task sampler (maze_sample_tasks_kernel):
its counters against hand-built Philox counters, its vectorised phases against a one-env-at-a-time transcription of the
kernel, the structural invariants of what it draws over thousands of tasks, and its distribution against the host
sampler MazeTaskSampler(rng=...)."""
import math

import numpy as np
import pytest

from oracle import philox

import maze_sampler_draws as msd
from maze_sampler_draws import restated_tasks, same_task

SEED = (0x9e3779b9 << 32) | 0x7f4a7c15          # high word set
GENV = 2 ** 32 + 12345                           # genv >= 2^32: the high word enters the fourth counter word


def _philox(ctr, seed):
    return philox.philox4x32_10([ctr], [seed & 0xFFFFFFFF, seed >> 32])[0]


def test_streams_match_hand_built_counters():
    """The first words of every stream equal Philox4x32-10 at counters built here by hand: lane 0's stream (genv lo, ep,
    z, 0x300 + genv hi) in word order x, y, z, w across blocks, and the per-cell purposes texture 0x310, value 0x320 and
    keep 0x1300 + round // 4."""
    lo, hi = GENV & 0xFFFFFFFF, GENV >> 32
    for ep in (1, 7, 2 ** 32 - 1):
        w = msd.lane0_words(SEED, [GENV], ep, 10)[0]
        hand = np.concatenate([_philox([lo, ep, z, 0x300 + hi], SEED) for z in range(3)])[:10]
        assert w.dtype == np.uint32 and np.array_equal(w, hand)
        for cell in (0, 1, 480, 960):
            for purpose in (0x310, 0x320, 0x1300, 0x1300 + 5):
                got = msd.cell_words(SEED, [GENV], ep, [cell], purpose)[0, 0]
                assert np.array_equal(got, _philox([lo, ep, cell, purpose + hi], SEED)), (ep, cell, hex(purpose))
    # the fourth word wraps: genv hi + purpose is taken modulo 2^32
    g = (0xFFFFFFF0 << 32) | 3
    got = msd.cell_words(SEED, [g], 1, [2], 0x320)[0, 0]
    assert np.array_equal(got, _philox([3, 1, 2, (0x320 + 0xFFFFFFF0) & 0xFFFFFFFF], SEED))


def test_below_and_value_rules():
    """below(k) = (word * k) >> 32; food values clip(u * food_reward, 0.10, food_reward) with np.clip's order, so a
    food_reward under 0.10 is the value of every food cell."""
    words = np.array([0, 1, 2 ** 31, 2 ** 32 - 1], dtype=np.uint32)
    assert msd._below(words, 7).tolist() == [0, 0, 3, 6]
    u24 = np.array([0, 1, 2 ** 23, 2 ** 24 - 1], dtype=np.uint32)
    assert msd.food_value(u24, 0.5).tolist() == [0.10, 0.10, 0.25, (2 ** 24 - 1) / 2 ** 24 * 0.5]
    assert msd.food_value(u24, 0.05).tolist() == [0.05] * 4
    assert np.array_equal(msd.food_value(u24, 0.05), np.clip(u24 / 2.0 ** 24 * 0.05, 0.10, 0.05))


def test_warp_total_order():
    """Lane partial sums in ascending cell order, then the xor butterfly: differs from np.sum where rounding does."""
    rs = np.random.RandomState(0)
    v = rs.rand(64, 225) * 10.0 ** rs.randint(-8, 3, size=(64, 225))
    got = msd.warp_total(v)
    for e in range(64):
        lane = [0.0] * 32
        for k in range(225):
            lane[k % 32] += v[e, k]
        for o in (16, 8, 4, 2, 1):
            lane = [lane[i] + lane[i ^ o] for i in range(32)]
        assert got[e] == lane[0]
    assert (got != v.sum(axis=1)).any()


# ---------------------------------------------------------------------------------------------------------------
# one env at a time, line for line as maze_sample_tasks_kernel runs (scalar Python, no vectorisation)
# ---------------------------------------------------------------------------------------------------------------
class _Stream(object):
    def __init__(self, seed, genv, ep):
        self.seed, self.ctr, self.buf = seed, [genv & 0xFFFFFFFF, ep, 0, (0x300 + (genv >> 32)) & 0xFFFFFFFF], []

    def next(self):
        if not self.buf:
            self.buf = [int(x) for x in _philox(self.ctr, self.seed)]
            self.ctr[2] += 1
        return self.buf.pop(0)

    def below(self, k):
        return (self.next() * k) >> 32


def _kernel_one_env(seed, genv, ep, n, f_max, allow_loops, crowd_ratio, food_reward, food_density, food_interval,
                    n_texts):
    m, nn = (n - 1) // 2, n * n
    walls = [0 if (i & 1) and (j & 1) else 1 for i in range(n) for j in range(n)]
    parent = list(range(m * m))
    rng = _Stream(seed, genv, ep)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    order = []
    for ra in range(m):
        for rb in range(m):
            if ra + 1 < m:
                order.append(2 * (ra * m + rb))
            if rb + 1 < m:
                order.append(2 * (ra * m + rb) + 1)
    for k in range(len(order) - 1, 0, -1):
        j = rng.below(k + 1)
        order[k], order[j] = order[j], order[k]
    for e in order:
        room, d = e >> 1, e & 1
        ra, rb = room // m, room % m
        x, y = find(room), find((ra + 1) * m + rb if d == 0 else ra * m + rb + 1)
        if x != y:
            parent[x] = y
            walls[(2 * ra + 2) * n + 2 * rb + 1 if d == 0 else (2 * ra + 1) * n + 2 * rb + 2] = 0
    if allow_loops:
        cand = [i * n + j for i in range(1, n - 1) for j in range(1, n - 1) if walls[i * n + j]]
        standing = len(cand)
        budget = float((n - 2) * (n - 2)) * crowd_ratio
        for k in range(len(cand) - 1, 0, -1):
            j = rng.below(k + 1)
            cand[k], cand[j] = cand[j], cand[k]
        for c in cand:
            if not standing > budget:
                break
            if not walls[c - n] or not walls[c + n] or not walls[c - 1] or not walls[c + 1]:
                walls[c] = 0
                standing -= 1
    sx, sy = rng.below(m) * 2 + 1, rng.below(m) * 2 + 1
    gx = gy = n - 2
    for _ in range(m * m):
        ex, ey = rng.below(m) * 2 + 1, rng.below(m) * 2 + 1
        if math.sqrt(float(ex - sx) ** 2 + float(ey - sy) ** 2) > 0.45 * n:
            gx, gy = ex, ey
            break
    hi, lo = genv >> 32, genv & 0xFFFFFFFF

    def draw(k, purpose):
        return [int(x) for x in _philox([lo, ep, k, (purpose + hi) & 0xFFFFFFFF], seed)]

    def value_of(u24):
        return min(max(u24 / 16777216.0 * food_reward, 0.10), food_reward)

    texts = [1 + ((draw(k, 0x310)[0] * (n_texts - 1)) >> 32) if walls[k] else 0 for k in range(nn)]
    val = [draw(k, 0x320)[0] >> 8 for k in range(nn)]
    alive = [not walls[k] for k in range(nn)]

    def totals():
        lane = [0.0] * 32
        for k in range(nn):
            if alive[k]:
                lane[k % 32] += value_of(val[k])
        for o in (16, 8, 4, 2, 1):
            lane = [lane[i] + lane[i ^ o] for i in range(32)]
        return lane[0], sum(alive)

    total, cnt = totals()
    expected = float((n - 1) * (n - 1)) * food_density
    r = 0
    while total > expected or cnt > f_max:
        for k in range(nn):
            if alive[k] and not (draw(k, 0x1300 + r // 4)[r % 4] >> 8) / 16777216.0 < 0.90:
                alive[k] = False
        total, cnt = totals()
        r += 1
    food = [value_of(val[k]) if alive[k] else 0.0 for k in range(nn)]
    itv = [food_interval if alive[k] and food[k] > 1e-3 else 0 for k in range(nn)]
    return (sx, sy), (gx, gy), walls, texts, food, itv


@pytest.mark.parametrize("n,allow_loops,crowd_ratio,food_reward,food_density,f_max", [
    (7, False, 0.0, 0.5, 0.2, 127), (9, True, 0.35, 0.05, 0.01, 127), (15, True, 0.0, 0.5, 0.01, 3),
    (15, True, 1.0, 0.0005, 0.2, 0), (21, False, 0.0, 0.5, 0.0, 127), (31, True, 0.35, 0.5, 0.05, 1)])
def test_vectorised_restatement_equals_the_kernel_transcribed(n, allow_loops, crowd_ratio, food_reward, food_density,
                                                              f_max):
    """restated_tasks, vectorised over envs, equals the kernel's steps written out for one env, for three envs with
    different resample counts (one with genv >= 2^32)."""
    genv = [5, 2 ** 32 + 9, 1027]
    ep = [1, 3, 2]
    kw = dict(allow_loops=allow_loops, crowd_ratio=crowd_ratio, food_reward=food_reward, food_density=food_density,
              food_interval=17, n_texts=5)
    got = restated_tasks(SEED, genv, ep, n, f_max, **kw)
    for e in range(3):
        start, goal, walls, texts, food, itv = _kernel_one_env(SEED, genv[e], ep[e], n, f_max, **kw)
        t = got[e]
        assert t.start == start and t.goal == goal
        assert t.cell_walls.ravel().tolist() == walls and t.cell_texts.ravel().tolist() == texts
        assert t.food_rewards.ravel().tolist() == food and t.food_interval.ravel().tolist() == itv


# ---------------------------------------------------------------------------------------------------------------
# structural invariants, thousands of tasks
# ---------------------------------------------------------------------------------------------------------------
def _reachable(walls, start):
    n = walls.shape[0]
    seen = np.zeros_like(walls, dtype=bool)
    seen[start] = True
    todo = [start]
    while todo:
        i, j = todo.pop()
        for a, b in ((i - 1, j), (i + 1, j), (i, j - 1), (i, j + 1)):
            if 0 <= a < n and 0 <= b < n and walls[a, b] == 0 and not seen[a, b]:
                seen[a, b] = True
                todo.append((a, b))
    return seen


STRUCT = [(7, False, 0.0, 800), (7, True, 0.35, 800), (9, True, 0.0, 800), (9, False, 0.0, 800),
          (15, True, 0.35, 600), (15, False, 0.0, 600), (21, True, 1.0, 300), (21, True, 0.2, 300),
          (31, True, 0.35, 200), (31, False, 0.0, 200)]


@pytest.mark.parametrize("n,allow_loops,crowd_ratio,count", STRUCT)
def test_restated_tasks_structure(n, allow_loops, crowd_ratio, count):
    """Closed border, rooms on odd cells, every free cell reachable from the start; without loops exactly a spanning tree
    (2 m^2 - 1 free interior cells), with loops never fewer interior walls than the crowd budget allows; textures
    1..n_texts-1 on walls only; start a room, goal a room farther than 0.45 n or the corner room; food on free cells only,
    each value in [min(0.10, food_reward), food_reward], the total within (n-1)^2 food_density and the count within
    f_max; intervals exactly where the value is above 1e-3."""
    m = (n - 1) // 2
    for food_reward, food_density, f_max, n_texts in ((0.5, 0.01, 127, 7), (0.05, 0.2, 6, 2), (0.0005, 0.1, 127, 4)):
        tasks = restated_tasks(SEED + n, np.arange(count) + 2 ** 32 - count // 2, 1, n, f_max, allow_loops=allow_loops,
                               crowd_ratio=crowd_ratio, food_reward=food_reward, food_density=food_density,
                               food_interval=9, n_texts=n_texts, goal_reward=None)
        for t in tasks:
            w = t.cell_walls
            assert w[0].all() and w[-1].all() and w[:, 0].all() and w[:, -1].all()
            assert (w[1:n:2, 1:n:2] == 0).all()
            sx, sy = t.start
            gx, gy = t.goal
            assert sx % 2 == 1 and sy % 2 == 1 and gx % 2 == 1 and gy % 2 == 1
            assert 1 <= min(sx, sy, gx, gy) and max(sx, sy, gx, gy) <= n - 2
            assert _reachable(w, (sx, sy)).sum() == (w == 0).sum()
            inner = w[1:-1, 1:-1]
            tree_walls = (n - 2) ** 2 - (2 * m * m - 1)
            if not allow_loops:
                assert inner.sum() == tree_walls
            else:      # one pass over the candidates, stopping as soon as the budget is met: never below it
                assert inner.sum() <= tree_walls
                assert inner.sum() == tree_walls or inner.sum() > (n - 2) ** 2 * crowd_ratio - 1
            tx = t.cell_texts
            assert (tx[w == 0] == 0).all() and (tx[w > 0] >= 1).all() and (tx[w > 0] <= n_texts - 1).all()
            assert (gx, gy) == (n - 2, n - 2) or math.sqrt((gx - sx) ** 2 + (gy - sy) ** 2) > 0.45 * n
            f = t.food_rewards
            assert (f[w > 0] == 0).all()
            assert ((f == 0) | ((f >= min(0.10, food_reward)) & (f <= food_reward))).all()
            assert f.sum() <= (n - 1) ** 2 * food_density + 1e-9 and (f > 0).sum() <= f_max
            assert np.array_equal(t.food_interval, np.where(f > 1e-3, 9, 0))
            assert t.goal_reward == -np.sqrt(n) * n * -0.01
        if n > 7 and (crowd_ratio > 0 or not allow_loops):     # (crowd_ratio 0 knocks nearly every interior wall out)
            assert len({t.cell_walls.tobytes() for t in tasks}) > 0.9 * count


def test_resample_counts_and_seeds_give_new_tasks():
    """Another resample count, seed or env gives another maze; the same arguments give the same tasks."""
    kw = dict(crowd_ratio=0.35)
    base = restated_tasks(SEED, np.arange(200), 1, 15, 127, **kw)
    again = restated_tasks(SEED, np.arange(200), 1, 15, 127, **kw)
    assert all(same_task(a, b) for a, b in zip(base, again))
    for other in (restated_tasks(SEED, np.arange(200), 2, 15, 127, **kw),
                  restated_tasks(SEED + 1, np.arange(200), 1, 15, 127, **kw),
                  restated_tasks(SEED, np.arange(200) + 200, 1, 15, 127, **kw)):
        assert sum(np.array_equal(a.cell_walls, b.cell_walls) for a, b in zip(base, other)) < 5
    shifted = restated_tasks(SEED, np.arange(100, 200), 1, 15, 127, **kw)
    assert all(same_task(a, b) for a, b in zip(base[100:], shifted))


# ---------------------------------------------------------------------------------------------------------------
# distribution: the host sampler of the same family
# ---------------------------------------------------------------------------------------------------------------
DIST = [dict(n=15, allow_loops=True, crowd_ratio=0.35, food_density=0.01, food_reward=0.5),
        dict(n=15, allow_loops=True, crowd_ratio=0.0, food_density=0.02, food_reward=0.05),
        dict(n=9, allow_loops=False, crowd_ratio=0.0, food_density=0.02, food_reward=0.5)]


@pytest.mark.parametrize("kw", DIST, ids=["loops035", "reward005", "tree9"])
def test_restated_distribution_matches_the_host_sampler(kw):
    """2000 restated tasks against 2000 of MazeTaskSampler(rng=RandomState): mean interior wall density, food count,
    total food and start-goal distance agree within 4 standard errors of the difference.  f_max = 127 leaves the
    thinning to the food total alone, as in the host sampler."""
    from metagym_b200 import MazeTaskSampler
    N = 2000
    dev = restated_tasks(20261017, np.arange(N), 1, f_max=127, **kw)
    rs = np.random.RandomState(5)
    host = [MazeTaskSampler(rng=rs, **kw) for _ in range(N)]

    def stats(tasks):
        return np.array([[t.cell_walls[1:-1, 1:-1].mean(), (t.food_rewards > 0).sum(), t.food_rewards.sum(),
                          math.sqrt((t.goal[0] - t.start[0]) ** 2 + (t.goal[1] - t.start[1]) ** 2)] for t in tasks])

    a, b = stats(dev), stats(host)
    diff = a.mean(axis=0) - b.mean(axis=0)
    se = np.sqrt(a.var(axis=0, ddof=1) / N + b.var(axis=0, ddof=1) / N)
    assert (np.abs(diff) <= 4 * se).all(), (diff, se)
    if kw["food_reward"] < 0.10:
        assert (np.concatenate([t.food_rewards[t.food_rewards > 0] for t in dev]) == kw["food_reward"]).all()
