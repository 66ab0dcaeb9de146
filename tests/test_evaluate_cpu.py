"""The float64 episode split that the whole-episode evaluation tests compare against (tests/episode_ref.py), pinned on
synthetic rew / done / truncated arrays."""
import numpy as np
import pytest

from episode_ref import split_episodes


def test_partial_first_episode_back_to_back_and_last_step_done():
    # env 0: a done at t = 1 ends the (partial) first episode; dones at t = 2 and t = 3 back to back
    # env 1: its only done is at the last step
    # env 2: a done at t = 0, then one at t = 4
    rew = np.array([[1.0, 0.5, 2.0],
                    [2.0, 0.25, 3.0],
                    [4.0, 0.125, 5.0],
                    [8.0, 0.0625, 6.0],
                    [16.0, 1.0, 7.0]], np.float32)
    done = np.array([[0, 0, 1],
                     [1, 0, 0],
                     [1, 0, 0],
                     [1, 0, 0],
                     [0, 1, 1]], np.uint8)
    trunc = np.array([[0, 0, 1],
                      [0, 0, 0],
                      [1, 0, 0],
                      [0, 0, 0],
                      [0, 1, 0]], np.uint8)
    ret, length, tr, steps = split_episodes(rew, done, trunc, 1)
    assert ret.dtype == np.float64 and length.dtype == np.int32 and tr.dtype == np.uint8
    np.testing.assert_array_equal(ret, [[3.0, 1.9375, 2.0]])
    np.testing.assert_array_equal(length, [[2, 5, 1]])
    np.testing.assert_array_equal(tr, [[0, 1, 1]])
    np.testing.assert_array_equal(steps, [2, 5, 1])
    ret, length, tr, steps = split_episodes(rew[:, [0, 2]], done[:, [0, 2]], trunc[:, [0, 2]], 2)
    np.testing.assert_array_equal(ret, [[3.0, 2.0], [4.0, 3.0 + 5.0 + 6.0 + 7.0]])
    np.testing.assert_array_equal(length, [[2, 1], [1, 4]])
    np.testing.assert_array_equal(tr, [[0, 1], [1, 0]])
    np.testing.assert_array_equal(steps, [3, 5])
    ret, length, tr, steps = split_episodes(rew[:, :1], done[:, :1], trunc[:, :1], 3)
    np.testing.assert_array_equal(ret[:, 0], [3.0, 4.0, 8.0])
    np.testing.assert_array_equal(length[:, 0], [2, 1, 1])
    np.testing.assert_array_equal(tr[:, 0], [0, 1, 0])
    assert steps[0] == 4      # the last step is never taken: the env stops at its third done


def test_sums_widen_each_float32_reward_in_step_order():
    # float32 rewards whose float64 sum differs from the float32 sum and from a reordered float64 sum
    rew = np.array([[1e8], [np.float32(1.0 / 3.0)], [-1e8], [np.float32(1e-3)]], np.float32)
    done = np.array([[0], [0], [0], [1]], np.uint8)
    ret, length, _, _ = split_episodes(rew, done, np.zeros_like(done), 1)
    want = ((np.float64(rew[0, 0]) + np.float64(rew[1, 0])) + np.float64(rew[2, 0])) + np.float64(rew[3, 0])
    assert ret[0, 0] == want and length[0, 0] == 4
    assert ret[0, 0] != np.float64(rew[:, 0].sum(dtype=np.float32))
    # float64 rewards (the maze's) are summed as they are
    r64 = np.array([[0.1], [0.2], [0.3]], np.float64)
    ret, _, _, _ = split_episodes(r64, np.array([[0], [0], [1]]), np.zeros((3, 1)), 1)
    assert ret[0, 0] == (0.1 + 0.2) + 0.3


def test_unfinished_env_is_an_error():
    with pytest.raises(ValueError, match="finished 1 of 2"):
        split_episodes(np.ones((3, 1)), np.array([[1], [0], [0]]), np.zeros((3, 1)), 2)
