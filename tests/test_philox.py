"""CPU checks of oracle/philox.py, the NumPy restatement of the engine's counter-based draws."""
import numpy as np

from oracle import philox


def test_philox4x32_10_known_answers():
    """Random123's known-answer vectors for Philox4x32-10 (kat_vectors: ctr, key -> output)."""
    cases = [
        ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
        ([0xffffffff] * 4, [0xffffffff, 0xffffffff], [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
        ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
         [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
    ]
    for ctr, key, want in cases:
        got = philox.philox4x32_10(np.array([ctr]), key)
        assert got.dtype == np.uint32
        assert got[0].tolist() == want, [hex(v) for v in got[0]]
    # vectorised rows are independent: the batch equals its rows one by one
    ctrs = np.array([c for c, _, _ in cases[:2]], dtype=np.uint64)
    assert np.array_equal(philox.philox4x32_10(ctrs, [7, 9])[1], philox.philox4x32_10(ctrs[1:], [7, 9])[0])


def test_u01_edges():
    u = philox.u01(np.array([0, 0xff, 0x100, 0xffffffff], dtype=np.uint32))
    assert u.dtype == np.float32
    assert u[0] == 0.0 and u[1] == 0.0 and u[2] == np.float32(2.0 ** -24)
    assert u[3] == np.float32(1.0 - 2.0 ** -24) and u[3] < 1.0


def test_counter_layout():
    """The global env index splits into counter words (lo, hi) and the seed into key (lo, hi)."""
    seed = (0x12345678 << 32) | 0x9abcdef0
    genv = np.array([5, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 7], dtype=np.int64)
    u = philox.quad_reset_draws(seed, genv, np.array([1, 2, 3, 4]))
    assert u.shape == (4, 12) and u.dtype == np.float64
    for i, g in enumerate(genv.tolist()):
        for j in range(3):
            r = philox.philox4x32_10([[g & 0xffffffff, g >> 32, i + 1, 0x100 + j]], [0x9abcdef0, 0x12345678])
            assert np.array_equal(u[i, 4 * j:4 * j + 4], philox.u01(r[0]).astype(np.float64))
    a = philox.quad_rollout_actions(seed, genv, 9, 0.1, 15.0)
    assert a.dtype == np.float32 and a.shape == (4, 4)
    assert (a >= np.float32(0.1)).all() and (a < np.float32(15.0)).all()
    m = philox.maze_rollout_actions(seed, genv, 9)
    r = philox.philox4x32_10(np.stack([genv & 0xffffffff, genv >> 32, np.full(4, 9), np.full(4, 0x200)], 1),
                             [0x9abcdef0, 0x12345678])
    assert np.array_equal(m, (r[:, 0] >> 30).astype(np.int32))
