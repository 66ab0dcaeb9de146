"""TEST INFRASTRUCTURE -- the random draws of the policy-driven rollouts restated in NumPy.

The counter of env `genv` at step counter t (t_base + step) is (genv lo, genv hi, t, STREAM_POLICY) with key = seed,
as for the other streams of oracle/philox.py.
"""
import numpy as np

from oracle import philox

STREAM_POLICY = 0x400    # MGB_STREAM_POLICY


def policy_words(seed, genv, t):
    """[n,4] uint32 Philox words of the policy stream."""
    return philox.philox4x32_10(philox._counters(genv, t, STREAM_POLICY), philox._seed_key(seed))


def quad_policy_normals(seed, genv, t):
    """[n,4] float64 standard normals z0..z3 of mgb_gaussian_action: Box-Muller on the word pairs (x, y), (z, w) with
    u1 = ((x >> 8) + 1) 2^-24 in (0, 1] and u2 = (y >> 8) 2^-24."""
    r = policy_words(seed, genv, t).astype(np.uint64)
    z = np.empty(r.shape, dtype=np.float64)
    for p in range(2):
        u1 = ((r[:, 2 * p] >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24
        u2 = (r[:, 2 * p + 1] >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
        rad = np.sqrt(-2.0 * np.log(u1))
        z[:, 2 * p] = rad * np.cos(2.0 * np.pi * u2)
        z[:, 2 * p + 1] = rad * np.sin(2.0 * np.pi * u2)
    return z


def maze_policy_uniforms(seed, genv, t):
    """[n] float32 uniforms u = (x >> 8) 2^-24 of mgb_categorical_action (the first Philox word)."""
    from oracle.philox import u01
    return u01(policy_words(seed, genv, t)[:, 0])
