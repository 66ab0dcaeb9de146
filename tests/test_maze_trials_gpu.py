"""GPU tests of trial handles (episodes_per_task=k, mgb_maze_set_episodes_per_task): each env counts the episodes it
finishes on its current maze, and a resampling rollout gives a finished env a new maze only at its k-th episode there.

k = 1 against a handle without trials, bit for bit; k = 2 and 3 against the host loop step + resample_tasks(m) +
reset(mask=m) with m = done & (task_episodes >= k) on all three maze kinds; the counting and zeroing of every path; the
recurrent "task" wipes against new_tasks(out); snapshot / restore / clone; refusals and CUDA-graph capture."""
import numpy as np
import pytest
import torch
from torch import nn

from test_maze2d_resample_rollout_gpu import CFG, slot_table
import test_lstm_policy_rollout_maze_gpu as lstm_tests
import test_policy_rollout_maze_gpu as mlp_tests
import test_rnn_policy_rollout_maze_gpu as gru_tests

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
BASE_HI = 2 ** 32 - 70                   # env_index_base: the batch straddles genv = 2^32
SEED = (0xfeed << 32) | 21


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    pass


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def make_2d(N, n=7, k=None, **kw):
    from metagym_b200 import BatchedMetaMaze2D
    table, fc = slot_table(n, N)
    kw = dict(dict(num_envs=N, squeeze=False, auto_reset=True, max_steps=5, view_grid=1), **kw)
    env = BatchedMetaMaze2D(episodes_per_task=k, **kw)
    env.set_task(table, env2task=np.arange(N))
    env.reset()
    return env, fc


def make_3d(kind, N, n, textures, k=None, **kw):
    from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    table, fc = slot_table(n, N)
    cls = BatchedMetaMazeContinuous3D if kind == "C3D" else BatchedMetaMazeDiscrete3D
    kw = dict(dict(num_envs=N, squeeze=False, auto_reset=True, max_steps=5, resolution=(24, 16), obs_dtype="int32",
                   textures=textures, cache=False), **kw)
    env = cls(episodes_per_task=k, **kw)
    env.set_task(table, env2task=np.arange(N))
    env.reset()
    return env, fc


def records(env):
    snap = env.snapshot()
    snap["records"].zero_()
    return env.snapshot(out=snap)["records"]


def count_off(fc):
    """Byte offset of a trial record's count block: behind the 48-byte head and the food stamps."""
    return 48 + (fc + 3) // 4 * 16


def strip_count(rec, fc):
    off = count_off(fc)
    return torch.cat([rec[:, :off], rec[:, off + 16:]], 1)


def record_counts(env, fc):
    return records(env)[:, count_off(fc):count_off(fc) + 4].contiguous().view(torch.int32)[:, 0]


def policy_for(kind, env, reset="task"):
    if kind == "mlp":
        return mlp_tests.make_policy(env, (16,), nn.Tanh, seed=2)[1]
    if kind == "gru":
        return gru_tests.make_policy(env, 17, 8, nn.Tanh, True, reset, seed=4)
    return lstm_tests.make_policy(env, 16, 0, nn.Tanh, True, reset, seed=5)


# ---------------------------------------------------------------------------------------------------------------------
# 1. k = 1 changes nothing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["open", "mlp", "gru", "lstm"])
@pytest.mark.parametrize("final,record", [(False, False), (True, True)], ids=["plain", "fin+path"])
def test_one_episode_per_task_equals_no_trials(kind, final, record):
    """A k = 1 handle and a handle without trials run the same resampling rollouts (two launches): every output, the
    carried state, the agent state and the snapshot records with the count block removed are bit for bit equal, and the
    counts stay 0 (every finished env draws)."""
    N, T = 150, 20
    kw = dict(final_obs=final, record_path=record, task_type="SURVIVAL", env_index_base=BASE_HI)
    trial, fc = make_2d(N, k=1, **kw)
    plain, _ = make_2d(N, **kw)
    pol = None if kind == "open" else policy_for(kind, plain)
    states = [pol.initial_state(N) if kind in ("gru", "lstm") else None for _ in range(2)]
    for launch in range(2):
        outs = []
        for env, st in zip((trial, plain), states):
            if pol is None:
                o = env.rollout(T, act_seed=3, want_actions=True, resample=dict(seed=SEED, **CFG))
            else:
                o = env.rollout(T, policy=pol, state=st, act_seed=3, resample=dict(seed=SEED, **CFG),
                                want_hidden=kind != "mlp")
            outs.append(o)
        a, b = outs
        assert a["episodes_per_task"] == 1 and a["resampled"] is True and "task_episodes0" not in b
        assert int(a["task_episodes0"].abs().sum()) == 0
        d = b["done"].bool()
        for key, v in b.items():
            if key == "final_obs":                     # rows with done = 0 are not written
                assert torch.equal(a[key][d], v[d]), launch
            elif isinstance(v, torch.Tensor):
                assert torch.equal(a[key], v), (launch, key)
        assert int(a["done"].sum()) > 0
        if states[0] is not None:
            assert torch.equal(states[0], states[1])
        assert int(trial.task_episodes.abs().sum()) == 0
    assert torch.equal(strip_count(records(trial), fc), records(plain))
    for x, y in zip(trial.agent_state(), plain.agent_state()):
        assert torch.equal(x, y)
    if record:
        for x, y in zip(trial.trajectory(), plain.trajectory()):
            assert torch.equal(x, y)
    trial.close(); plain.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. k in {2, 3} = the host loop step + resample_tasks(m) + reset(mask=m), m = done & (task_episodes >= k)
# ---------------------------------------------------------------------------------------------------------------------
TRIALS = [("2D", "SURVIVAL", 2, 7, 5, True), ("2D", "ESCAPE", 3, 7, BASE_HI, False),
          ("2D", "ESCAPE", 2, 15, BASE_HI, True), ("D3D", "SURVIVAL", 2, 9, BASE_HI, True),
          ("D3D", "ESCAPE", 3, 9, 7, False), ("C3D", "SURVIVAL", 3, 9, 7, True), ("C3D", "ESCAPE", 2, 9, BASE_HI, False)]


@pytest.mark.parametrize("kind,task_type,k,n,base,final", TRIALS)
def test_trials_equal_the_host_loop(textures, kind, task_type, k, n, base, final):
    """Three consecutive resampling rollouts of a trial handle (trials span launches) against a twin that runs, per
    step, step(act[t]), m = done & (task_episodes >= k), resample_tasks(m, seed, **CFG), obs_t = reset(mask=m): obs,
    rew, done, final_obs and truncated per step, the counts after every launch, and at the end the snapshot records
    byte for byte (counts, resample counts and tasks included) and the agent state."""
    N, T = (150, 12) if kind == "2D" else (40, 10)
    kw = dict(task_type=task_type, env_index_base=base)
    if kind == "2D":
        roll, fc = make_2d(N, n, k=k, final_obs=final, **kw)
        twin, _ = make_2d(N, n, k=k, final_obs=True, **kw)
    else:
        roll, fc = make_3d(kind, N, n, textures, k=k, **kw)
        twin, _ = make_3d(kind, N, n, textures, k=k, final_obs=True, **kw)
    rng = np.random.RandomState(n + k)
    drew_any = kept_any = False
    for launch in range(3):
        if kind == "C3D":
            acts = torch.as_tensor(rng.uniform(-1.3, 1.3, (T, N, 2)).astype(np.float32)).cuda()
        else:
            acts = torch.as_tensor(rng.randint(0, 4, (T, N)).astype(np.int32)).cuda()
        if kind == "2D":
            out = roll.rollout(T, actions=acts, resample=dict(seed=SEED, **CFG))
        else:
            out = roll.rollout(T, actions=acts, final_obs=final, resample=dict(seed=SEED, **CFG))
        assert torch.equal(out["task_episodes0"], twin.task_episodes), launch
        from metagym_b200.metamaze import new_tasks
        drew = new_tasks(out)
        for t in range(T):
            _, r, d, _ = twin.step(acts[t])
            assert torch.equal(out["rew"][t], r) and torch.equal(out["done"][t].bool(), d), (launch, t)
            if final:
                assert torch.equal(out["truncated"][t].bool(), twin.truncated), (launch, t)
                assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), (launch, t)
            m = d & (twin.task_episodes >= k)
            assert torch.equal(drew[t], m), (launch, t)
            drew_any |= bool(m.any())
            kept_any |= bool((d & ~m).any())
            twin.resample_tasks(m, seed=SEED, **CFG)
            o = twin.reset(mask=m)
            assert torch.equal(out["obs"][t], o), (launch, t, int((out["obs"][t] != o).sum()))
        assert torch.equal(roll.task_episodes, twin.task_episodes), launch
    assert drew_any and kept_any
    assert torch.equal(records(roll), records(twin))
    assert torch.equal(record_counts(roll, fc), roll.task_episodes)
    for x, y in zip(roll.agent_state(), twin.agent_state()):
        assert torch.equal(x, y)
    roll.close(); twin.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. counting and zeroing
# ---------------------------------------------------------------------------------------------------------------------
def test_counting_and_zeroing():
    """step() (device and host actions), open-loop and policy rollouts without resampling add their done totals;
    reset() leaves the counts; resample_tasks(mask) zeroes the masked envs, update_tasks the envs of the replaced
    slots, set_task every env."""
    N, T = 96, 16
    env, _ = make_2d(N, k=3)
    want = torch.zeros(N, dtype=torch.int64, device="cuda")
    assert torch.equal(env.task_episodes.long(), want)
    rng = np.random.RandomState(0)
    for t in range(7):
        a = rng.randint(0, 4, N).astype(np.int32)
        _, _, d, _ = env.step(torch.as_tensor(a).cuda() if t % 2 else a)
        want += d.long()
    assert int(want.max()) >= 1
    assert torch.equal(env.task_episodes.long(), want)
    out = env.rollout(T, act_seed=1)
    assert torch.equal(out["task_episodes0"].long(), want) and out["resampled"] is False
    assert not new_tasks_any(out)
    want += out["done"].long().sum(0)
    assert torch.equal(env.task_episodes.long(), want)
    pol = policy_for("gru", env)
    st = pol.initial_state(N)
    out = env.rollout(T, policy=pol, state=st, act_seed=2)
    want += out["done"].long().sum(0)
    assert torch.equal(env.task_episodes.long(), want)
    out = env.rollout(T, policy=policy_for("mlp", env), act_seed=2)
    want += out["done"].long().sum(0)
    assert torch.equal(env.task_episodes.long(), want)
    env.reset()
    env.reset(mask=torch.ones(N, dtype=torch.bool, device="cuda"))
    assert torch.equal(env.task_episodes.long(), want)
    mask = torch.as_tensor(rng.rand(N) < 0.3).cuda()
    env.resample_tasks(mask, seed=5, **CFG)
    want[mask] = 0
    assert torch.equal(env.task_episodes.long(), want)
    slots = [3, 17, 40]
    env.update_tasks(slots, [env.tasks[0]] * 3)
    want[slots] = 0
    assert torch.equal(env.task_episodes.long(), want)
    assert int(want.max()) > 0
    env.set_task(env.tasks, env2task=np.arange(N))
    assert int(env.task_episodes.abs().sum()) == 0
    env.close()


def new_tasks_any(out):
    from metagym_b200.metamaze import new_tasks
    return bool(new_tasks(out).any())


def test_three_d_step_and_rollout_count(textures):
    """The 3-D step, the pose-cache rollout and the direct rollout without resampling add their done totals."""
    for kind, cache in (("D3D", True), ("D3D", False), ("C3D", False)):
        env, _ = make_3d(kind, 24, 9, textures, k=2, cache=cache)
        want = torch.zeros(24, dtype=torch.int64, device="cuda")
        for t in range(6):
            a = torch.zeros((24, 2), dtype=torch.float32, device="cuda") if kind == "C3D" else \
                torch.full((24,), t % 4, dtype=torch.int32, device="cuda")
            _, _, d, _ = env.step(a)
            want += d.long()
        out = env.rollout(9, act_seed=4)
        want += out["done"].long().sum(0)
        assert int(want.sum()) > 0, kind
        assert torch.equal(env.task_episodes.long(), want), kind
        env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. recurrent wipes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cell", ["gru", "lstm"])
def test_task_rule_wipes_where_new_tasks(cell):
    """Under "task" on a k = 2 handle, launches of T = 1 leave a state row zero exactly where new_tasks(out) is true
    (feedback on: a kept row holds a one-hot action); a T = 24 launch's logp is reproduced by policy.unroll(out)."""
    N = 200
    env, _ = make_2d(N, k=2, max_steps=3)
    pol = policy_for(cell, env, "task")
    st = pol.initial_state(N)
    wiped = kept = 0
    for launch in range(12):
        out = env.rollout(1, policy=pol, state=st, act_seed=7, resample=dict(seed=SEED, **CFG))
        from metagym_b200.metamaze import new_tasks
        drew = new_tasks(out)[0]
        zero = (st == 0).all(1)
        assert torch.equal(zero, drew), launch
        wiped += int(drew.sum())
        kept += int((out["done"][0].bool() & ~drew).sum())
    assert wiped > 0 and kept > 0
    out = env.rollout(24, policy=pol, state=st, act_seed=9, resample=dict(seed=SEED, **CFG))
    assert bool(new_tasks_any(out)) and bool((out["done"].bool() & ~new_tasks_from(out)).any())
    _, logp = pol.unroll(out)
    assert float((logp.detach() - out["logp"].cpu()).abs().max()) < 1e-4
    env.close()


def new_tasks_from(out):
    from metagym_b200.metamaze import new_tasks
    return new_tasks(out)


# ---------------------------------------------------------------------------------------------------------------------
# 5. snapshot, restore, clone
# ---------------------------------------------------------------------------------------------------------------------
def test_snapshot_restore_clone_carry_the_counts():
    """A mid-trial snapshot restored after more launches continues bit for bit (outputs and counts); restore with a
    mask and clone_envs carry the counts; a trial snapshot is refused by a handle without trials and by one with
    another k."""
    N, T = 130, 9
    env, fc = make_2d(N, k=3)
    env.rollout(T, act_seed=1, resample=dict(seed=SEED, **CFG))
    snap = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in env.snapshot().items()}
    counts = env.task_episodes
    assert int(counts.max()) > 0
    assert torch.equal(record_counts(env, fc), counts)
    first = env.rollout(T, act_seed=1, resample=dict(seed=SEED, **CFG))
    first = {k: v.clone() for k, v in first.items() if isinstance(v, torch.Tensor)}
    after = env.task_episodes
    env.rollout(T, act_seed=1, resample=dict(seed=SEED, **CFG))
    env.restore(snap)
    assert torch.equal(env.task_episodes, counts)
    again = env.rollout(T, act_seed=1, resample=dict(seed=SEED, **CFG))
    for key, v in first.items():
        assert torch.equal(again[key], v), key
    assert torch.equal(env.task_episodes, after)
    # restore with a mask: only the masked envs take the snapshot's counts
    now = env.task_episodes
    mask = torch.zeros(N, dtype=torch.bool)
    mask[::3] = True
    env.restore(snap, mask=mask)
    want = torch.where(mask.cuda(), counts, now)
    assert torch.equal(env.task_episodes, want)
    # clone_envs: dst envs take src envs' counts
    src, dst = [1, 2, 5], [10, 20, 50]
    before = env.task_episodes
    env.clone_envs(src, dst)
    before[dst] = before[src]
    assert torch.equal(env.task_episodes, before)
    # refusals by the fingerprint
    plain, _ = make_2d(N)
    other, _ = make_2d(N, k=2)
    for h in (plain, other):
        rec = records(h)
        with pytest.raises(ValueError, match="episodes_per_task"):
            h.restore(snap)
        assert torch.equal(records(h), rec)
    plain.close(); other.close(); env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals and capture
# ---------------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_handle_untouched():
    from metagym_b200 import MgbError, _lib
    N = 64
    env, _ = make_2d(N, k=2)
    lib = env._lib
    env.rollout(8, act_seed=1)
    rec, counts = records(env), env.task_episodes
    assert lib.mgb_maze_set_episodes_per_task(env._h, 3) == MGB_ERR_ARG        # after set_task
    assert b"before mgb_maze_set_task" in lib.mgb_last_error()
    assert lib.mgb_maze_set_episodes_per_task(env._h, -1) == MGB_ERR_ARG
    obs = torch.empty((4, N, 3, 3), dtype=torch.float32, device="cuda")
    rew = torch.empty((4, N), dtype=torch.float64, device="cuda")
    s = _lib.current_stream(torch, env.device)
    assert lib.mgb_maze_rollout(env._h, 4, None, 1, None, obs.data_ptr(), rew.data_ptr(), None, None, None, None, 0,
                                s) == MGB_ERR_ARG
    assert b"done_dev may not be null" in lib.mgb_last_error()
    pol = policy_for("gru", env)
    st = pol.initial_state(N)
    with pytest.raises(MgbError, match="done_dev"):
        env.rollout(4, policy=pol, state=st, out={"obs": obs, "rew": rew, "act": None, "done": None})
    with pytest.raises(MgbError, match="done_dev"):
        env.rollout(4, policy=policy_for("mlp", env), out={"obs": obs, "rew": rew, "act": None, "done": None})
    torch.cuda.synchronize()
    assert torch.equal(records(env), rec) and torch.equal(env.task_episodes, counts)
    assert torch.equal(st, pol.initial_state(N))
    plain, _ = make_2d(N)
    out = torch.empty(N, dtype=torch.int32, device="cuda")
    assert lib.mgb_maze_task_episodes(plain._h, out.data_ptr(), s) == MGB_ERR_ARG
    assert plain.task_episodes is None
    plain.close()
    with pytest.raises(ValueError):
        make_2d(N, k=0)
    # a handle without set_task takes the setter (k = 0 switches trials off again)
    from metagym_b200 import BatchedMetaMaze2D
    fresh = BatchedMetaMaze2D(num_envs=N, squeeze=False, auto_reset=True, max_steps=5, view_grid=1, episodes_per_task=2)
    table, _ = slot_table(7, N)
    fresh._create(7)
    assert lib.mgb_maze_set_episodes_per_task(fresh._h, 0) == 0
    assert lib.mgb_maze_set_episodes_per_task(fresh._h, 4) == 0
    fresh.close(); env.close()


def test_graph_capture_equals_eager():
    """A trial rollout with resampling captured in a CUDA graph: each replay equals an eager launch of a twin, counts
    included."""
    N, T = 160, 8
    eager, _ = make_2d(N, k=2)
    graph, _ = make_2d(N, k=2)
    acts = torch.as_tensor(np.random.RandomState(4).randint(0, 4, (T, N)).astype(np.int32)).cuda()
    out = {"obs": torch.empty((T, N, 3, 3), dtype=torch.float32, device="cuda"),
           "rew": torch.empty((T, N), dtype=torch.float64, device="cuda"),
           "done": torch.empty((T, N), dtype=torch.uint8, device="cuda"), "act": None,
           "task_episodes0": torch.empty(N, dtype=torch.int32, device="cuda")}
    # warm-up launch on both, so the graph starts where the eager twin does
    for e in (eager, graph):
        e.rollout(T, actions=acts, resample=dict(seed=SEED, **CFG))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            graph.rollout(T, actions=acts, out=out, resample=dict(seed=SEED, **CFG))
    torch.cuda.current_stream().wait_stream(s)
    # capture launched nothing: the eager twin runs the captured launch first
    for rep in range(3):
        want = eager.rollout(T, actions=acts, resample=dict(seed=SEED, **CFG))
        g.replay()
        torch.cuda.synchronize()
        for key in ("obs", "rew", "done", "task_episodes0"):
            assert torch.equal(out[key], want[key]), (rep, key)
        assert torch.equal(graph.task_episodes, eager.task_episodes), rep
    eager.close(); graph.close()
