"""CPU: metagym_b200.metamaze.new_tasks(out) -- where a rollout's envs drew a new maze -- against a brute-force scan."""
import numpy as np
import pytest
import torch

from metagym_b200.metamaze import new_tasks


def brute_force(done, count0, k, resampled, trial):
    T, N = done.shape
    want = np.zeros((T, N), bool)
    if not resampled:
        return want
    for e in range(N):
        c = int(count0[e]) if trial else 0
        for t in range(T):
            if not done[t, e]:
                continue
            if not trial:
                want[t, e] = True
                continue
            c += 1
            if c >= k:
                want[t, e] = True
                c = 0
    return want


@pytest.mark.parametrize("k", [1, 2, 3, 7])
@pytest.mark.parametrize("resampled", [False, True])
@pytest.mark.parametrize("seed", range(3))
def test_new_tasks_equals_a_brute_force_scan(k, resampled, seed):
    rng = np.random.RandomState(seed * 10 + k)
    T, N = 17, 301
    done = rng.rand(T, N) < rng.uniform(0.05, 0.6)
    count0 = rng.randint(0, k + 2, N)            # counts at and past k too: the rule holds for any start count
    out = {"done": torch.as_tensor(done.astype(np.uint8)), "resampled": resampled,
           "task_episodes0": torch.as_tensor(count0.astype(np.int32)), "episodes_per_task": k}
    got = new_tasks(out)
    assert got.dtype == torch.bool and got.shape == (T, N)
    assert np.array_equal(got.numpy(), brute_force(done, count0, k, resampled, True))


@pytest.mark.parametrize("resampled", [False, True])
def test_new_tasks_without_trials(resampled):
    """A rollout dict of a handle without trials: done where the launch resampled, else nothing; a dict without the
    "resampled" entry (an open-loop rollout of such a handle) counts as not resampled."""
    rng = np.random.RandomState(4)
    done = rng.rand(9, 40) < 0.3
    out = {"done": torch.as_tensor(done.astype(np.uint8)), "resampled": resampled}
    assert np.array_equal(new_tasks(out).numpy(), brute_force(done, None, None, resampled, False))
    del out["resampled"]
    assert not new_tasks(out).any()
