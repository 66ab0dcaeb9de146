"""Velocity-target rows on every quadrotor step path when envs do NOT move in lockstep: tasks scattered over the envs
(7 tasks, a random env -> task map) and a random step counter per env, so that the lanes of a warp read rows of
different tasks at different times.  The handle keeps its own time-major copy of the [n_tasks][nt][3] table; these
tests check that each reader picks the right row of it: the step kernels (tile, one-CTA-per-SM, packed), the fused
rollout, the reset kernel and the auto-reset observation.  Observation columns 16..18 are copies of table rows and
are compared bit for bit."""
import numpy as np
import pytest

from util import OBS_GROUPS, group_rel_err, scalar_rel_err

pytestmark = pytest.mark.gpu

N_TASKS, NT, DT = 7, 40, 0.005


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def _env(n, rng, auto_reset=False):
    from metagym_b200 import BatchedQuadrotor
    env = BatchedQuadrotor(task="velocity_control", dt=DT, nt=NT, seed=list(range(N_TASKS)), num_envs=n, device=0,
                           squeeze=False, auto_reset=auto_reset)
    env.set_velocity_tasks(list(range(N_TASKS)), env2task=rng.randint(0, N_TASKS, n))
    return env


def _scatter_ct(env, ct):
    """Load per-env step counters, keeping the state the last reset left."""
    import torch
    sd = env.state_dict()
    env.load_state_dict({"state": sd["state"], "ct": torch.as_tensor(np.asarray(ct, np.int32))})


def _path_size(path, sms):
    return {"tile": 301, "wide": sms * 100 + 3, "packed": 301}[path]


@pytest.mark.parametrize("path", ["tile", "wide", "packed"])
def test_scattered_rows_vs_oracle(torch_mod, monkeypatch, path):
    torch = torch_mod
    from oracle import quad_oracle as qo
    if path == "packed":
        monkeypatch.setenv("MGB_PACKED", "1")
    n = _path_size(path, torch.cuda.get_device_properties(0).multi_processor_count)
    rng = np.random.RandomState(31 + n)
    env = _env(n, rng)
    kname = env.step_kernel_name()
    want = {"tile": "quad_step_kernel", "wide": "quad_step_wide_kernel", "packed": "quad_step2_kernel"}[path]
    assert kname.startswith(want), kname
    noise = rng.random_sample((n, 12))
    env.reset(noise=noise)
    state = qo.reset_state(None, noise)
    ct = rng.randint(0, NT, n).astype(np.int32)
    ct[:5] = NT - 1                                   # these end their episode on the first step
    _scatter_ct(env, ct)
    tg, e2t = env.velocity_targets.cpu().numpy(), env.env2task.cpu().numpy()
    cfg = qo.make_cfg()
    for t in range(3):
        act = rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)
        obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
        o_ref, r_ref, d_ref, _, _ = qo.env_step(cfg, state, ct, act, "velocity_control", DT, NT, targets=tg,
                                                env2task=e2t, mode="mix")
        o = obs.cpu().numpy()
        assert np.array_equal(o[:, 16:], o_ref[:, 16:]), t
        assert group_rel_err(o[:, :16], o_ref[:, :16], OBS_GROUPS) < 1e-5, t
        assert scalar_rel_err(rew.cpu().numpy(), r_ref) < 1e-5, t
        assert np.array_equal(done.cpu().numpy(), d_ref.astype(bool)), t
    assert np.array_equal(env.state_dict()["ct"].cpu().numpy(), ct)
    env.close()


def test_scattered_rows_rollout_equals_steps(torch_mod):
    torch = torch_mod
    n, T = 301, 4
    outs = []
    for mode in ("step", "rollout"):
        rng = np.random.RandomState(5)
        env = _env(n, rng, auto_reset=True)
        env.reset(noise=rng.random_sample((n, 12)))
        _scatter_ct(env, rng.randint(0, NT, n))
        acts = torch.as_tensor(rng.uniform(0.1, 15.0, (T, n, 4)).astype(np.float32)).cuda()
        if mode == "step":
            rows = [[x.clone() for x in env.step(acts[t])[:3]] for t in range(T)]
            outs.append([torch.stack([r[k] for r in rows]).cpu().numpy() for k in range(3)])
        else:
            r = env.rollout(T, actions=acts)
            outs.append([r["obs"].cpu().numpy(), r["rew"].cpu().numpy(), r["done"].cpu().numpy()])
        env.close()
    assert outs[0][2].any()                            # some envs crossed an episode end inside the rollout
    for a, b in zip(outs[0], outs[1]):
        assert np.array_equal(a.astype(b.dtype), b)


def test_reset_and_auto_reset_rows(torch_mod):
    torch = torch_mod
    n = 301
    rng = np.random.RandomState(9)
    env = _env(n, rng, auto_reset=True)
    tg, e2t = env.velocity_targets.cpu().numpy(), env.env2task.cpu().numpy()
    obs = env.reset(noise=rng.random_sample((n, 12))).cpu().numpy()
    assert np.array_equal(obs[:, 16:], tg[e2t, 0])                       # reset kernel: ct = 0
    ct = rng.randint(0, NT, n).astype(np.int32)
    ct[::3] = NT - 1                                                       # every third env finishes on this step
    _scatter_ct(env, ct)
    obs, _, done, _ = env.step(torch.as_tensor(rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)).cuda())
    obs, done = obs.cpu().numpy(), done.cpu().numpy().astype(bool)
    assert done[::3].all()
    new_ct = np.where(done, 0, ct + 1)
    assert np.array_equal(env.state_dict()["ct"].cpu().numpy(), new_ct)
    # a replaced env shows the first row of its next episode, the others the row after the step
    assert np.array_equal(obs[:, 16:], tg[e2t, np.minimum(new_ct, NT - 1)])
    env.close()
