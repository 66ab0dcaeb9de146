"""TEST INFRASTRUCTURE -- the ESCAPE expert of include/mgb200.h ("Expert") restated in NumPy.

A state is s = (ori n + gx) n + gy; MetaMaze2D has one heading plane (ori = 0), MetaMazeDiscrete3D four.  `step_rule`
restates the move of one action as the reference writes it (maze_2d.py:21-34 with numpy's negative index, which the
border walls make unreachable; maze_discrete_3d.py:51-81: turn, then move); `tables` is the backward breadth-first
search from the goal; `forward_dist` a plain forward search from one state, used to pin `tables`.  `expert_actions`
restates the per-step draws.
"""
from collections import deque

import numpy as np

from oracle import philox

STREAM_EXPERT = 0x800    # MGB_STREAM_EXPERT
FAR = 0xFFFF


def planes(kind):
    return 1 if kind == "2D" else 4


def step_rule(walls, kind, gx, gy, ori, a):
    """(gx, gy, ori) after action a."""
    n = walls.shape[0]
    if kind == "2D":
        dx, dy = ((-1, 0), (1, 0), (0, -1), (0, 1))[a]
        tx, ty = gx + dx, gy + dy
        if tx < 0:
            tx += n
        if ty < 0:
            ty += n
        if tx < n and ty < n and walls[tx, ty] < 1:
            gx, gy = tx, ty
        return gx, gy, ori
    turn, mv = ((-1, 0), (1, 0), (0, -1), (0, 1))[a]
    ori = (ori + turn + 4) % 4
    dx, dy = ((1, 0), (0, 1), (-1, 0), (0, -1))[ori]
    tx, ty = gx + mv * dx, gy + mv * dy
    if 0 <= tx < n and 0 <= ty < n and walls[tx, ty] == 0:
        gx, gy = tx, ty
    return gx, gy, ori


def successors(walls, kind):
    """[S, 4] int64: the state every action leads to."""
    n, P = walls.shape[0], planes(kind)
    nxt = np.empty((P * n * n, 4), np.int64)
    for ori in range(P):
        for gx in range(n):
            for gy in range(n):
                for a in range(4):
                    x, y, o = step_rule(walls, kind, gx, gy, ori, a)
                    nxt[(ori * n + gx) * n + gy, a] = (o * n + x) * n + y
    return nxt


def tables(walls, goal, kind):
    """(dist uint16 [P, n, n], mask uint8 [P, n, n]) of one task."""
    walls = np.asarray(walls)
    n, P = walls.shape[0], planes(kind)
    nxt = successors(walls, kind)
    cell = np.arange(P * n * n) % (n * n)
    dist = np.where(cell == goal[0] * n + goal[1], 0, FAR).astype(np.int64)
    lev = 1
    while True:
        grow = (dist == FAR) & (dist[nxt] == lev - 1).any(axis=1)
        if not grow.any():
            break
        dist[grow] = lev
        lev += 1
    opt = dist[nxt] == (dist - 1)[:, None]
    live = (dist != 0) & (dist != FAR)
    mask = np.where(live, (opt * (1 << np.arange(4))).sum(axis=1), 0)
    return dist.astype(np.uint16).reshape(P, n, n), mask.astype(np.uint8).reshape(P, n, n)


def forward_dist(walls, goal, kind, gx, gy, ori):
    """The fewest actions from (gx, gy, ori) to the goal cell by forward search (FAR: never)."""
    walls = np.asarray(walls)
    start = (gx, gy, ori)
    if (gx, gy) == tuple(goal):
        return 0
    seen, q = {start: 0}, deque([start])
    while q:
        s = q.popleft()
        for a in range(4):
            t = step_rule(walls, kind, *s, a)
            if t in seen:
                continue
            if (t[0], t[1]) == tuple(goal):
                return seen[s] + 1
            seen[t] = seen[s] + 1
            q.append(t)
    return FAR


def expert_words(seed, genv, t):
    """[n, 4] uint32 Philox words of the expert stream at step counter t."""
    return philox.philox4x32_10(philox._counters(genv, t, STREAM_EXPERT), philox._seed_key(seed))


def expert_actions(seed, genv, t, mask, eps, mean=False):
    """[n] int32 actions of the expert at step counter t on states with masks `mask` [n] uint8."""
    mask = np.asarray(mask, dtype=np.int64)
    full = np.where(mask == 0, 15, mask)
    if mean:
        choice, j = full, np.zeros_like(mask)
    else:
        r = expert_words(seed, genv, t).astype(np.uint64)
        explore = philox.u01(r[:, 0].astype(np.uint32)) < np.float32(eps)
        choice = np.where(explore, 15, full)
        k = np.array([bin(int(c)).count("1") for c in choice], dtype=np.uint64)
        j = ((r[:, 1] * k) >> np.uint64(32)).astype(np.int64)
    out = np.empty(mask.shape, np.int32)
    for i, (c, jj) in enumerate(zip(choice, j)):
        bits = [a for a in range(4) if (int(c) >> a) & 1]
        out[i] = bits[int(jj)]
    return out
