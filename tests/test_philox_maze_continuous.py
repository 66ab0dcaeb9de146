"""CPU checks of maze_continuous_draws.maze_continuous_rollout_actions, the restated action draw of the continuous-maze
rollout."""
import numpy as np

from oracle import philox

from maze_continuous_draws import maze_continuous_rollout_actions


def test_maze_continuous_rollout_actions_match_a_hand_computation():
    """turn_rate, walk_speed = 2 u01(x) - 1, 2 u01(y) - 1 of the Philox words of counter (genv lo, genv hi, t, 0x200),
    computed here as (x >> 8) / 2^23 - 1 in float64 (exact) and compared bit for bit."""
    seed = (0x0badf00d << 32) | 0x12345678
    genv = np.array([0, 3, 2 ** 32 - 1, 2 ** 32 + 5], dtype=np.int64)
    for t in (0, 1, 77, 2 ** 32 - 1):
        a = maze_continuous_rollout_actions(seed, genv, t)
        assert a.dtype == np.float32 and a.shape == (4, 2)
        assert (a >= -1.0).all() and (a < 1.0).all()
        for i, g in enumerate(genv.tolist()):
            r = philox.philox4x32_10([[g & 0xffffffff, g >> 32, t, 0x200]], [0x12345678, 0x0badf00d])[0]
            for k in range(2):
                assert a[i, k] == np.float32((int(r[k]) >> 8) / 2.0 ** 23 - 1.0), (t, g, k)


def test_maze_continuous_rollout_actions_edges(monkeypatch):
    """u01 = 0 gives exactly -1 and the largest u01 (1 - 2^-24) gives 1 - 2^-23: the draw covers [-1, 1) in steps of
    2^-23 with no rounding at either end.  Words z and w do not take part."""
    words = np.array([[0x000000ff, 0xffffffff, 0x12345678, 0x9abcdef0],
                      [0xffffff00, 0x00000100, 0, 0],
                      [0x80000000, 0x7fffffff, 0xffffffff, 0xffffffff]], dtype=np.uint32)
    monkeypatch.setattr(philox, "philox4x32_10", lambda ctr, key: words)
    a = maze_continuous_rollout_actions(1, np.arange(3), 0)
    top = np.float32(1.0 - 2.0 ** -23)
    assert a[0].tolist() == [-1.0, top]
    assert a[1].tolist() == [top, np.float32(-1.0 + 2.0 ** -23)]
    assert a[2].tolist() == [0.0, np.float32(-2.0 ** -23)]
