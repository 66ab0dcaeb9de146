"""Float64 restatement of the episode split of whole-episode evaluation (mgb_quad_evaluate, mgb_maze_evaluate; DESIGN.md
"Whole-episode evaluation"), from a rollout's per-step rew / done / truncated."""
import numpy as np


def split_episodes(rew, done, truncated, episodes):
    """rew [T, N] (float32 or float64), done and truncated [T, N] of a rollout long enough for every env to reach its
    `episodes`-th done.  Returns (ret [episodes, N] float64, length [episodes, N] int32, trunc [episodes, N] uint8,
    steps [N] int64): episode j of env e is the steps after its done number j - 1 up to and including done number j
    (episode 0 starts at t = 0); ret sums its rewards in step order, each widened to float64 on its own; trunc is
    truncated at the done that ends it; steps is the step count L_e at which the env stops."""
    rew, done, truncated = np.asarray(rew), np.asarray(done) != 0, np.asarray(truncated)
    T, N = done.shape
    ret = np.zeros((episodes, N), np.float64)
    length = np.zeros((episodes, N), np.int32)
    trunc = np.zeros((episodes, N), np.uint8)
    steps = np.zeros(N, np.int64)
    acc = np.zeros(N, np.float64)           # every env's running sum, episode index and length; all envs step together
    j = np.zeros(N, np.int64)
    n = np.zeros(N, np.int64)
    for t in range(T):
        live = j < episodes
        if not live.any():
            break
        acc = np.where(live, acc + rew[t].astype(np.float64), acc)
        n += live
        end = np.nonzero(live & done[t])[0]
        ret[j[end], end], length[j[end], end], trunc[j[end], end] = acc[end], n[end], truncated[t, end] != 0
        acc[end], n[end] = 0.0, 0
        j[end] += 1
        steps[end[j[end] == episodes]] = t + 1
    if (j < episodes).any():
        e = int(np.nonzero(j < episodes)[0][0])
        raise ValueError("env %d finished %d of %d episodes in %d steps" % (e, j[e], episodes, T))
    return ret, length, trunc, steps
