"""TEST INFRASTRUCTURE -- the engine's counter-based random draws restated in NumPy.

Philox4x32-10 as mgb_philox4x32_10 computes it (metagym_b200/csrc/mgb_common.cuh), vectorised over envs with uint64
arithmetic, and the three places the engine draws from it with their counter layouts.  Every env owns a stream keyed
by the 64-bit seed (key = (lo, hi)) and counted by its GLOBAL index `genv` = env_index_base + local index, so these
functions reproduce the device's draws bit for bit without a GPU.
"""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_S32 = np.uint64(32)

STREAM_RESET = 0x100     # + j, j = 0..2: the twelve reset draws (MGB_STREAM_RESET)
STREAM_ACTION = 0x200    # rollout actions (MGB_STREAM_ACTION)


def philox4x32_10(ctr, key):
    """ctr [n,4] (or [4]) 32-bit words x,y,z,w; key (k0, k1).  Returns [n,4] uint32."""
    c = np.asarray(ctr, dtype=np.uint64).reshape(-1, 4) & _MASK
    x, y, z, w = (c[:, i].copy() for i in range(4))
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = _M0 * x, _M1 * z                   # < 2^64: exact in uint64
        x, y, z, w = (p1 >> _S32) ^ y ^ k0, p1 & _MASK, (p0 >> _S32) ^ w ^ k1, p0 & _MASK
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return np.stack([x, y, z, w], axis=1).astype(np.uint32)


def u01(x):
    """mgb_u01: the top 24 bits as a float32 in [0, 1)."""
    return (np.asarray(x, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def _seed_key(seed):
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, s >> 32


def _counters(genv, third, w):
    g = np.asarray(genv, dtype=np.int64).reshape(-1).astype(np.uint64)     # two's complement, like (uint64_t)genv
    n = g.size
    c = np.empty((n, 4), dtype=np.uint64)
    c[:, 0] = g & _MASK
    c[:, 1] = g >> _S32
    c[:, 2] = np.broadcast_to(np.asarray(third, dtype=np.int64).astype(np.uint64), (n,)) & _MASK
    c[:, 3] = w
    return c


def quad_reset_draws(seed, genv, ep):
    """philox_reset_draws (quad.cu): [n,12] float64, u[4j..4j+3] = words x,y,z,w of ctr (genv lo, genv hi, ep,
    0x100 + j).  `ep` is the episode count after the increment that precedes the draw."""
    key = _seed_key(seed)
    out = [u01(philox4x32_10(_counters(genv, ep, STREAM_RESET + j), key)) for j in range(3)]
    return np.concatenate(out, axis=1).astype(np.float64)


def quad_rollout_actions(act_seed, genv, t, vmin, vmax):
    """Device-drawn quadrotor rollout action of step counter t (t_base + step): [n,4] float32,
    fmaf(vmax - vmin, u01, vmin) with both bounds float32.  The float64 product span * u01 is exact and is rounded
    once to float32 after the addition; for the default voltage range this equals fmaf for every u01 value."""
    u = u01(philox4x32_10(_counters(genv, t, STREAM_ACTION), _seed_key(act_seed))).astype(np.float64)
    lo, hi = np.float32(vmin), np.float32(vmax)
    span = np.float64(np.float32(hi - lo))
    return (span * u + np.float64(lo)).astype(np.float32)


def maze_rollout_actions(act_seed, genv, t):
    """Device-drawn maze rollout action of step counter t: the top two bits of word x, uniform over {0,1,2,3}."""
    r = philox4x32_10(_counters(genv, t, STREAM_ACTION), _seed_key(act_seed))
    return (r[:, 0] >> np.uint32(30)).astype(np.int32)
