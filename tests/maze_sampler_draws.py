"""The device task sampler (maze_sample_tasks_kernel, metagym_b200/csrc/maze.cu) restated in NumPy, on top of
oracle.philox's Philox4x32-10 and vectorised over envs, so that a few thousand 31x31 tasks restate in seconds.

Every draw of the kernel is counter-based, keyed by the 64-bit seed (key = (lo, hi)) and counted by the env's GLOBAL
index genv = env_index_base + local index and its resample count ep (the count after the increment that precedes the
draw, so the first resample of an env has ep = 1):

  * lane 0's sequential stream, counter (genv lo, ep, z, 0x300 + genv hi) for z = 0, 1, ..., words x, y, z, w in that
    order, leftover words carried from one phase to the next: the Fisher-Yates shuffle of the room-lattice edges, the
    shuffle of the loop candidates (allow_loops only), the start room, then up to m^2 goal tries of two words each;
  * per-cell draws, counter (genv lo, ep, cell, purpose + genv hi): texture 0x310 (word x), food value 0x320 (word x)
    and the keep draw of thinning round r, 0x1300 + r // 4, word r % 4.

restated_tasks() returns one TaskConfig per env, field for field what BatchedMetaMaze*.get_tasks returns for the env's
slot: the same dtypes, and float64 values equal to the device's, not merely close.  Food values follow the host sampler
MazeTaskSampler(rng=...): clip(U * food_reward, 0.10, food_reward) in np.clip's order (min(max(v, 0.10), food_reward)),
and a food cell gets food_interval only where its value is above 1e-3.
"""
import numpy as np

from metagym_b200.metamaze import TaskConfig
from oracle import philox

STREAM_SAMPLER = 0x300          # lane 0's sequential stream (MGB_STREAM_SAMPLER)
PURPOSE_TEXTURE = 0x310
PURPOSE_VALUE = 0x320
PURPOSE_KEEP = 0x1300           # + round // 4

_M32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def _key(seed):
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, s >> 32


def _genv(genv):
    g = np.asarray(genv).reshape(-1)
    if g.dtype.kind == "i":
        g = g.astype(np.int64)                   # two's complement, like (uint64_t)genv
    return g.astype(np.uint64)


def _ep(ep, size):
    return np.broadcast_to(np.asarray(ep, dtype=np.int64).astype(np.uint64) & _M32, (size,)).copy()


def _draw(key, g, ep, third, purpose):
    """Philox blocks at counters (g lo, ep, third, purpose + g hi), all arrays flat and of one length -> [len, 4]."""
    c = np.empty((g.size, 4), dtype=np.uint64)
    c[:, 0] = g & _M32
    c[:, 1] = ep
    c[:, 2] = np.asarray(third, dtype=np.uint64) & _M32
    c[:, 3] = (np.uint64(purpose) + (g >> _S32)) & _M32
    return philox.philox4x32_10(c, key)


def lane0_words(seed, genv, ep, count):
    """The first `count` words of every env's sequential stream -> uint32 [E, count]."""
    g = _genv(genv)
    e = _ep(ep, g.size)
    blocks = (count + 3) // 4
    z = np.tile(np.arange(blocks, dtype=np.uint64), g.size)
    r = _draw(_key(seed), np.repeat(g, blocks), np.repeat(e, blocks), z, STREAM_SAMPLER)
    return r.reshape(g.size, blocks * 4)[:, :count]


def cell_words(seed, genv, ep, cells, purpose):
    """Philox blocks of per-cell purpose `purpose` for every env and each of `cells` -> uint32 [E, len(cells), 4]."""
    g = _genv(genv)
    e = _ep(ep, g.size)
    cells = np.asarray(cells, dtype=np.uint64).reshape(-1)
    k = cells.size
    r = _draw(_key(seed), np.repeat(g, k), np.repeat(e, k), np.tile(cells, g.size), purpose)
    return r.reshape(g.size, k, 4)


def _below(word, k):
    """Uniform integer in [0, k): (word * k) >> 32."""
    return ((word.astype(np.uint64) * np.uint64(k)) >> _S32).astype(np.int64)


def _shuffle(order, words):
    """Fisher-Yates from the last element down, one word per swap, every row of `order` at once."""
    ar = np.arange(order.shape[0])
    for i, k in enumerate(range(order.shape[1] - 1, 0, -1)):
        j = _below(words[:, i], k + 1)
        t = order[:, k].copy()
        order[:, k] = order[ar, j]
        order[ar, j] = t


def warp_total(values):
    """The kernel's float64 total over the cells of each env: lane L adds the cells L, L + 32, ... in ascending order,
    then the 32 partial sums meet in the xor butterfly 16, 8, 4, 2, 1.  values [E, nn] -> [E]."""
    E, nn = values.shape
    P = (nn + 31) // 32
    v = np.zeros((E, P * 32), dtype=np.float64)
    v[:, :nn] = values
    v = v.reshape(E, P, 32)
    part = np.zeros((E, 32), dtype=np.float64)
    for p in range(P):                       # sequential, not np.sum's pairwise order
        part = part + v[:, p, :]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        part = part + part[:, lanes ^ o]
    return part[:, 0]


def food_value(u24, food_reward):
    """Food value of a 24-bit draw: clip(u24 * 2^-24 * food_reward, 0.10, food_reward) in np.clip's order, so
    food_reward < 0.10 gives food_reward."""
    v = np.asarray(u24).astype(np.float64) * (1.0 / 16777216.0) * food_reward
    return np.minimum(np.maximum(v, 0.10), food_reward)


def restated_tasks(seed, genv, ep, n, f_max, allow_loops=True, cell_size=2.0, wall_height=3.2, agent_height=1.6,
                   step_reward=-0.01, goal_reward=None, food_reward=0.50, initial_life=1.0, max_life=2.0,
                   food_density=0.010, food_interval=100, crowd_ratio=0.0, n_texts=7):
    """The tasks resample_tasks(seed=seed, **sampler_kw) writes for global envs `genv` at resample counts `ep` (scalar
    or one per env) on an n x n handle whose set_task table has at most f_max food cells per task -> [TaskConfig]."""
    g = _genv(genv)
    E = g.size
    epv = _ep(ep, E)
    ar = np.arange(E)
    m = (n - 1) // 2
    nn = n * n
    walls = np.ones((E, nn), dtype=np.int32)
    walls.reshape(E, n, n)[:, 1:n:2, 1:n:2] = 0
    # ---- lane 0's stream: every phase before the goal tries takes the same number of words in every env
    edges = []
    for ra in range(m):
        for rb in range(m):
            if ra + 1 < m:
                edges.append(2 * (ra * m + rb))
            if rb + 1 < m:
                edges.append(2 * (ra * m + rb) + 1)
    ne = len(edges)
    nc = (n - 2) ** 2 - m * m - (m * m - 1)          # interior walls a spanning tree leaves standing
    n_loop = max(nc - 1, 0) if allow_loops else 0
    words = lane0_words(seed, g, epv, (ne - 1) + n_loop + 2 + 2 * m * m)
    pos = 0
    # random spanning tree: Kruskal over the shuffled edges (edge id = 2 * room + dir)
    order = np.tile(np.array(edges, dtype=np.int64), (E, 1))
    _shuffle(order, words[:, pos:pos + ne - 1])
    pos += ne - 1
    label = np.tile(np.arange(m * m, dtype=np.int64), (E, 1))
    for k in range(ne):
        room, d = order[:, k] >> 1, order[:, k] & 1
        ra, rb = room // m, room % m
        other = np.where(d == 0, room + m, room + 1)
        lu, lv = label[ar, room], label[ar, other]
        join = lu != lv
        cell = np.where(d == 0, (2 * ra + 2) * n + 2 * rb + 1, (2 * ra + 1) * n + 2 * rb + 2)
        walls[ar[join], cell[join]] = 0
        label = np.where((label == lu[:, None]) & join[:, None], lv[:, None], label)
    # loops: standing interior walls in row-major order, shuffled, knocked out next to a free cell down to crowd_ratio
    if allow_loops:
        inner = walls.reshape(E, n, n)[:, 1:n - 1, 1:n - 1].reshape(E, -1) != 0
        assert (inner.sum(axis=1) == nc).all()
        f = np.nonzero(inner)[1].reshape(E, nc)
        cand = (f // (n - 2) + 1) * n + f % (n - 2) + 1
        _shuffle(cand, words[:, pos:pos + n_loop])
        pos += n_loop
        standing = np.full(E, nc, dtype=np.int64)
        budget = float((n - 2) * (n - 2)) * crowd_ratio
        for k in range(nc):
            c = cand[:, k]
            free = (walls[ar, c - n] == 0) | (walls[ar, c + n] == 0) | (walls[ar, c - 1] == 0) | (walls[ar, c + 1] == 0)
            hit = (standing.astype(np.float64) > budget) & free
            walls[ar[hit], c[hit]] = 0
            standing -= hit
    # start room, then the first of up to m^2 tries far enough from it (else the corner room)
    sx = _below(words[:, pos], m) * 2 + 1
    sy = _below(words[:, pos + 1], m) * 2 + 1
    pos += 2
    gx, gy = np.full(E, n - 2, dtype=np.int64), np.full(E, n - 2, dtype=np.int64)
    found = np.zeros(E, dtype=bool)
    for _ in range(m * m):
        ex = _below(words[:, pos], m) * 2 + 1
        ey = _below(words[:, pos + 1], m) * 2 + 1
        pos += 2
        dx, dy = (ex - sx).astype(np.float64), (ey - sy).astype(np.float64)
        ok = ~found & (np.sqrt(dx * dx + dy * dy) > 0.45 * n)
        gx[ok], gy[ok] = ex[ok], ey[ok]
        found |= ok
    # ---- per-cell draws: textures on walls, a food value on every free cell
    cells = np.arange(nn)
    tx = 1 + ((cell_words(seed, g, epv, cells, PURPOSE_TEXTURE)[:, :, 0].astype(np.uint64) * np.uint64(n_texts - 1))
              >> _S32).astype(np.int64)
    texts = np.where(walls != 0, tx, 0)
    value = food_value(cell_words(seed, g, epv, cells, PURPOSE_VALUE)[:, :, 0] >> np.uint32(8), food_reward)
    alive = walls == 0
    total = warp_total(np.where(alive, value, 0.0))
    # ---- thinning: every live food survives a round with probability 0.90 until the total and the count fit
    expected = float((n - 1) * (n - 1)) * food_density
    active = (total > expected) | (alive.sum(axis=1) > f_max)
    keep_words = np.zeros((E, nn, 4), dtype=np.uint32)
    r = 0
    while active.any():
        if r % 4 == 0:            # one block per 4 rounds; only cells still alive at its start can draw from it
            ei, ci = np.nonzero(alive & active[:, None])
            keep_words[ei, ci] = _draw(_key(seed), g[ei], epv[ei], ci, PURPOSE_KEEP + r // 4)
        x = keep_words[:, :, r % 4]
        keep = (x >> np.uint32(8)).astype(np.float64) * (1.0 / 16777216.0) < 0.90
        alive = np.where(active[:, None], alive & keep, alive)
        total = warp_total(np.where(alive, value, 0.0))
        active &= (total > expected) | (alive.sum(axis=1) > f_max)
        r += 1
    food = np.where(alive, value, 0.0)
    interval = np.where(alive & (value > 1.0e-3), food_interval, 0).astype(np.int32)
    gr = -np.sqrt(n) * n * step_reward if goal_reward is None else goal_reward
    return [TaskConfig(start=(int(sx[e]), int(sy[e])), goal=(int(gx[e]), int(gy[e])),
                       cell_walls=walls[e].reshape(n, n).astype(np.int32), cell_texts=texts[e].reshape(n, n).astype(np.int64),
                       cell_size=float(cell_size), step_reward=float(step_reward), goal_reward=float(gr),
                       wall_height=float(wall_height), agent_height=float(agent_height), initial_life=float(initial_life),
                       max_life=float(max_life), food_rewards=food[e].reshape(n, n),
                       food_interval=interval[e].reshape(n, n)) for e in range(E)]


def same_task(a, b):
    """Field for field equality of two TaskConfigs: arrays by dtype, shape and value, scalars by ==."""
    for name in TaskConfig._fields:
        x, y = getattr(a, name), getattr(b, name)
        if isinstance(x, np.ndarray) or isinstance(y, np.ndarray):
            if not (isinstance(x, np.ndarray) and isinstance(y, np.ndarray) and x.dtype == y.dtype
                    and x.shape == y.shape and np.array_equal(x, y)):
                return False
        elif isinstance(x, tuple) or isinstance(y, tuple):
            if tuple(x) != tuple(y):
                return False
        elif x != y:
            return False
    return True
