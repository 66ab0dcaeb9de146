"""The continuous-maze rollout's device-drawn actions restated in NumPy, on top of oracle.philox's Philox4x32-10."""
import numpy as np

from oracle import philox


def maze_continuous_rollout_actions(act_seed, genv, t):
    """Device-drawn continuous-maze rollout action of step counter t (t_base + step): [n,2] float32 (turn_rate,
    walk_speed) = 2 u01 - 1 of words x and y of counter (genv lo, genv hi, t, STREAM_ACTION) keyed by the 64-bit seed,
    in float32 arithmetic (exact for every 24-bit u01), uniform on [-1, 1)."""
    g = np.asarray(genv, dtype=np.int64).reshape(-1).astype(np.uint64)     # two's complement, like (uint64_t)genv
    ctr = np.stack([g & np.uint64(0xFFFFFFFF), g >> np.uint64(32),
                    np.full(g.size, int(t) & 0xFFFFFFFF, dtype=np.uint64),
                    np.full(g.size, philox.STREAM_ACTION, dtype=np.uint64)], axis=1)
    s = int(act_seed) & 0xFFFFFFFFFFFFFFFF
    r = philox.philox4x32_10(ctr, (s & 0xFFFFFFFF, s >> 32))
    return np.float32(2.0) * philox.u01(r[:, :2]) - np.float32(1.0)
