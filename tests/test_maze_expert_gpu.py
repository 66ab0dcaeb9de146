"""GPU tests of the ESCAPE expert (include/mgb200.h "Expert"): the device tables against tests/expert_ref.py after every
call that changes the task table, expert rollouts against open-loop rollouts fed their actions, the labels and draws
against the restatement, the pose cache against the direct renderer, the step label, sharding, graph capture and the
refusals."""
import ctypes

import numpy as np
import pytest
import torch

import expert_ref as xr

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
SEED = (0xbeef << 32) | 5


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    pass


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def tasks(n, K, seed=0):
    from metagym_b200.metamaze import MazeTaskSampler
    return [MazeTaskSampler(n=n, allow_loops=bool(k % 2), crowd_ratio=0.35 * (k % 3), seed=seed * 1000 + k)
            for k in range(K)]


def make(kind, N, tex=None, n=9, K=5, env2task=None, expert=True, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D
    base = dict(num_envs=N, squeeze=False, auto_reset=True, max_steps=40, task_type="ESCAPE", expert=expert)
    if kind == "2D":
        env = BatchedMetaMaze2D(view_grid=1, **dict(base, **kw))
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=(24, 16), obs_dtype="uint8", textures=tex,
                                        cache=(kind == "3D-cache"), **dict(base, **kw))
    env.set_task(tasks(n, K), env2task=env2task)
    env.reset()
    return env


def restated(env, table):
    kind = "2D" if env.KIND == 0 else "3D"
    out = [xr.tables(np.asarray(t.cell_walls), tuple(t.goal), kind) for t in table]
    return np.stack([m for _, m in out]), np.stack([d for d, _ in out]).astype(np.int32)


def check_tables(env, table):
    mask, dist = env.expert_table()
    m, d = restated(env, table)
    assert np.array_equal(mask.cpu().numpy(), m) and np.array_equal(dist.cpu().numpy(), d)


KINDS = ["2D", "3D-cache", "3D-direct"]


@pytest.mark.parametrize("kind", KINDS)
def test_tables_after_set_task_and_update_tasks(kind, textures):
    env = make(kind, 8, textures)
    check_tables(env, env.tasks)
    env.update_tasks([1, 3], tasks(9, 2, seed=7))
    torch.cuda.synchronize()
    check_tables(env, env.tasks)
    m, d = env.expert_table(slots=[3, 0])
    full_m, full_d = env.expert_table()
    assert torch.equal(m, full_m[[3, 0]]) and torch.equal(d, full_d[[3, 0]])


@pytest.mark.parametrize("kind", ["2D", "3D-direct"])
def test_tables_after_resample_tasks_and_restore(kind, textures):
    N = 12
    env = make(kind, N, textures, K=N, env2task=np.arange(N))
    snap = env.snapshot()
    before = env.get_tasks(range(N))
    mask = torch.tensor([k % 3 == 0 for k in range(N)], device="cuda")
    env.resample_tasks(mask, seed=3, allow_loops=True, crowd_ratio=0.35)
    after = env.get_tasks(range(N))
    assert any(not np.array_equal(a.cell_walls, b.cell_walls) for a, b in zip(before, after))
    check_tables(env, after)
    env.restore(snap)
    torch.cuda.synchronize()
    check_tables(env, before)


def twin_replay(kind, tex, out, T, **kw):
    """An expert=False twin stepped with out["act"] by the open-loop rollout."""
    tw = make(kind, out["done"].shape[1], tex, expert=False, **kw)
    final = "final_obs" in out
    return tw, (tw.rollout(T, actions=out["act"], final_obs=final) if kind != "2D" else tw.rollout(T, actions=out["act"]))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("variant", ["plain", "final", "trial_path"])
def test_expert_rollout_is_open_loop_rollout_of_its_actions(kind, variant, textures):
    N, T = 40, 48
    kw = {}
    if variant == "trial_path":
        kw = dict(episodes_per_task=2, record_path=True)
    final = variant == "final"
    if kind == "2D" and final:
        kw["final_obs"] = True
    env = make(kind, N, textures, **kw)
    out = env.rollout(T, expert=0.3, act_seed=SEED, **({} if kind == "2D" else {"final_obs": final}))
    tw, ref = twin_replay(kind, textures, out, T, **kw)
    for k in ("obs", "rew", "done"):
        assert torch.equal(out[k], ref[k]), k
    if final:
        assert torch.equal(out["truncated"], ref["truncated"])
        d = out["done"].bool()
        assert torch.equal(out["final_obs"][d], ref["final_obs"][d])
    for a, b in zip(env.agent_state(), tw.agent_state()):
        assert torch.equal(a, b)
    if variant == "trial_path":
        assert torch.equal(env.task_episodes, tw.task_episodes)
        for a, b in zip(env.trajectory(), tw.trajectory()):
            assert torch.equal(a, b)
    # given actions with labels: the same env side again
    env2 = make(kind, N, textures, **kw)
    out2 = env2.rollout(T, actions=out["act"], want_expert=True, **({} if kind == "2D" else {"final_obs": final}))
    assert torch.equal(out2["expert"], out["expert"]) and torch.equal(out2["obs"], out["obs"])


@pytest.mark.parametrize("kind", ["2D", "3D-cache"])
@pytest.mark.parametrize("eps,mean", [(0.0, False), (0.3, False), (1.0, False), (0.3, True)])
def test_labels_and_actions_equal_the_restatement(kind, eps, mean, textures):
    N, T = 24, 20
    env = make(kind, N, textures, env_index_base=2 ** 32 - 10)
    walk = make(kind, N, textures, env_index_base=2 ** 32 - 10)
    env.rollout(3, expert=0.5, act_seed=1)              # a t_base other than 0
    walk.rollout(3, expert=0.5, act_seed=1)
    t0 = env._counters()
    out = env.rollout(T, expert=eps, deterministic=mean, act_seed=SEED)
    mask_tab, _ = walk.expert_table()
    mask_tab = mask_tab.cpu().numpy()
    e2t = walk.env2task
    genv = np.arange(N, dtype=np.int64) + 2 ** 32 - 10
    for t in range(T):
        ag = walk.agent_state()[0].cpu().numpy()
        ori = ag[:, 2] if kind != "2D" else np.zeros(N, np.int64)
        label = mask_tab[e2t, ori, ag[:, 0], ag[:, 1]]
        assert np.array_equal(out["expert"][t].cpu().numpy(), label), t
        act = xr.expert_actions(SEED, genv, t0 + t, label, eps, mean)
        assert np.array_equal(out["act"][t].cpu().numpy(), act), t
        walk.rollout(1, actions=out["act"][t:t + 1])


@pytest.mark.parametrize("kind", ["2D", "3D-cache"])
def test_eps0_reaches_goal_in_exactly_dist_steps(kind, textures):
    N = 40
    env = make(kind, N, textures, max_steps=400)
    _, dist = env.expert()
    dist = dist.cpu().numpy()
    assert (dist > 0).all() and (dist < 400).all()
    T = int(dist.max())
    out = env.rollout(T, expert=0.0, act_seed=SEED)
    done = out["done"].cpu().numpy().astype(bool)
    first = done.argmax(axis=0)
    assert np.array_equal(first, dist - 1) and done.any(axis=0).all()
    rew = out["rew"].cpu().numpy()[first, np.arange(N)]
    goal = np.array([env.tasks[k].step_reward + env.tasks[k].goal_reward for k in env.env2task])
    assert np.array_equal(rew, goal)


def test_pose_cache_and_direct_renderer_agree(textures):
    outs = []
    for kind in ("3D-cache", "3D-direct"):
        env = make(kind, 32, textures)
        outs.append(env.rollout(40, expert=0.2, act_seed=SEED, final_obs=True))
    for k in ("obs", "rew", "done", "act", "expert", "truncated"):
        assert torch.equal(outs[0][k], outs[1][k]), k
    d = outs[0]["done"].bool()
    assert torch.equal(outs[0]["final_obs"][d], outs[1]["final_obs"][d])


def restated_labels(env, mask_tab):
    """The table entry of every env's current state, read from agent_state() and the env's slot."""
    ag = env.agent_state()[0].cpu().numpy()
    ori = ag[:, 2] if env.KIND != 0 else np.zeros(len(ag), np.int64)
    return mask_tab[env.env2task, ori, ag[:, 0], ag[:, 1]]


@pytest.mark.parametrize("kind", KINDS)
def test_step_label_is_the_table_entry_of_the_state_after_the_step(kind, textures):
    env = make(kind, 16, textures, max_steps=6)
    m, _ = restated(env, env.tasks)
    rng = np.random.RandomState(0)
    finished = 0
    for _ in range(10):
        a = torch.as_tensor(rng.randint(0, 4, 16), dtype=torch.int32, device="cuda")
        _, _, done, info = env.step(a, want_expert=True)
        assert "expert" in info
        assert np.array_equal(info["expert"].cpu().numpy(), restated_labels(env, m))
        finished += int(done.sum())
    assert finished >= 16              # max_steps = 6: labels after auto-resets were checked too


@pytest.mark.parametrize("kind", ["2D", "3D-cache"])
def test_sharding_invariance(kind, textures):
    N, T = 64, 24
    full = make(kind, N, textures)
    ref = full.rollout(T, expert=0.4, act_seed=SEED)
    for base in (0, 32):
        sh = make(kind, 32, textures, env_index_base=base)
        out = sh.rollout(T, expert=0.4, act_seed=SEED)
        for k in ("act", "expert", "obs", "rew", "done"):
            assert torch.equal(out[k], ref[k][:, base:base + 32]), k


def capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            res = fn()
    torch.cuda.current_stream().wait_stream(s)
    return g, res


@pytest.mark.parametrize("kind", ["2D", "3D-cache"])
def test_graph_capture(kind, textures):
    """A captured expert rollout and label replay as the eager calls of a twin at the same step counter."""
    N, T = 32, 16
    env, twin = make(kind, N, textures), make(kind, N, textures)
    out = env.rollout(T, expert=0.3, act_seed=SEED)
    twin.rollout(T, expert=0.3, act_seed=SEED)

    def body():
        env.rollout(T, expert=0.3, act_seed=SEED, out=out)
        return env.expert()[0]
    g, lab = capture(body)
    g.replay()
    torch.cuda.synchronize()
    ref = twin.rollout(T, expert=0.3, act_seed=SEED)
    for k in ("obs", "rew", "done", "act", "expert"):
        assert torch.equal(out[k], ref[k]), k
    assert torch.equal(lab, twin.expert()[0])


@pytest.mark.parametrize("kind", ["2D", "3D-direct"])
def test_graph_capture_of_labelled_steps_and_table_rebuild(kind, textures):
    """step(want_expert=True) and resample_tasks (which rebuilds the drawn slots' tables) captured in one graph: the
    replayed labels and tables equal an eager twin's and the restatement of the drawn tasks."""
    N = 12
    env, twin = (make(kind, N, textures, K=N, env2task=np.arange(N), max_steps=8) for _ in range(2))
    acts = torch.as_tensor(np.random.RandomState(1).randint(0, 4, (3, N)), dtype=torch.int32, device="cuda")
    mask = torch.tensor([k % 2 == 0 for k in range(N)], device="cuda")
    env.step(acts[0], want_expert=True)              # the step's persistent buffers exist before the capture
    twin.step(acts[0], want_expert=True)
    labels = torch.empty((2, N), dtype=torch.uint8, device="cuda")

    def body():
        env.resample_tasks(mask, seed=4, allow_loops=True, crowd_ratio=0.35)
        for t in (1, 2):
            labels[t - 1] = env.step(acts[t], want_expert=True)[3]["expert"]
    g, _ = capture(body)
    g.replay()
    torch.cuda.synchronize()
    twin.resample_tasks(mask, seed=4, allow_loops=True, crowd_ratio=0.35)
    for t in (1, 2):
        assert torch.equal(labels[t - 1], twin.step(acts[t], want_expert=True)[3]["expert"]), t
    drawn = env.get_tasks(range(N))
    check_tables(env, drawn)
    assert torch.equal(env.expert_table()[0], twin.expert_table()[0])


@pytest.mark.parametrize("kind", ["2D", "3D-direct"])
def test_in_launch_resampling_is_refused_on_an_expert_handle(kind, textures):
    """A launch that draws new mazes into task slots cannot rebuild their tables: every such entry point refuses an
    expert handle, and the handle, its tables included, stays as it was."""
    from torch import nn
    from metagym_b200 import _lib
    from metagym_b200.policy import MLPPolicy
    N = 12
    env = make(kind, N, textures, K=N, env2task=np.arange(N))
    agent0, t0 = env.agent_state()[0].clone(), env._counters()
    calls = [lambda: env.rollout(8, resample=dict(seed=1))]
    if kind == "2D":
        pol = MLPPolicy(nn.Sequential(nn.Linear(9, 16), nn.Tanh(), nn.Linear(16, 4)), device=env.device)
        calls += [lambda: env.rollout(8, policy=pol, resample=dict(seed=1)),
                  lambda: env.evaluate(pol, episodes=1, resample=dict(seed=1))]
    for call in calls:
        with pytest.raises(_lib.MgbError, match="in-launch resampling is not available on an expert handle"):
            call()
    torch.cuda.synchronize()
    assert torch.equal(env.agent_state()[0], agent0) and env._counters() == t0
    check_tables(env, env.get_tasks(range(N)))
    # the same table change between launches keeps the tables current
    env.resample_tasks(None, seed=1)
    check_tables(env, env.get_tasks(range(N)))


def test_mirrors_are_refused(textures):
    env = make("2D", 8)
    agent0, t0 = env.agent_state()[0].clone(), env._counters()
    from metagym_b200 import _lib
    for setter in (lambda: env.set_mirrors([1 << 20]), lambda: env.set_multicast(1 << 20)):
        setter()
        for call in (lambda: env.rollout(4, expert=0.1), lambda: env.expert(), lambda: env.expert_table(),
                     lambda: env.step(torch.zeros(8, dtype=torch.int32, device="cuda"), want_expert=True)):
            with pytest.raises(_lib.MgbError, match="output mirrors or multicast"):
                call()
        env.set_mirrors([])
        env.set_multicast(0)
    assert torch.equal(env.agent_state()[0], agent0) and env._counters() == t0
    env.rollout(4, expert=0.1)


def _ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def test_refusals(textures):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D
    from metagym_b200 import _lib
    with pytest.raises(ValueError, match="ESCAPE"):
        BatchedMetaMaze2D(task_type="SURVIVAL", expert=True)
    with pytest.raises(ValueError, match="grid mazes"):
        BatchedMetaMazeContinuous3D(task_type="ESCAPE", expert=True, textures=textures)
    plain = make("2D", 8, expert=False)
    with pytest.raises(ValueError, match="expert=True"):
        plain.rollout(4, expert=0.1)
    with pytest.raises(ValueError, match="expert=True"):
        plain.step(torch.zeros(8, dtype=torch.int32, device="cuda"), want_expert=True)
    env = make("2D", 8)
    with pytest.raises(ValueError, match="resample"):
        env.rollout(4, expert=0.1, resample=dict(seed=1))
    with pytest.raises(ValueError, match="in \\[0, 1\\]"):
        env.rollout(4, expert=1.5)
    L, h = env._lib, env._h
    T, N = 4, 8
    obs = torch.empty((T, N, 3, 3), device="cuda")
    rew = torch.empty((T, N), dtype=torch.float64, device="cuda")
    done = torch.empty((T, N), dtype=torch.uint8, device="cuda")
    st = env._stream()
    agent0, t0 = env.agent_state()[0].clone(), env._counters()

    def call(handle=h, T=T, eps=0.1, mode=0, o=obs):
        return L.mgb_maze_rollout_expert(handle, T, None, ctypes.c_float(eps), mode, 1, None, None, _ptr(o), _ptr(rew),
                                         _ptr(done), None, None, st)
    cases = [(dict(eps=float("nan")), "eps"), (dict(eps=-0.1), "eps"), (dict(eps=1.01), "eps"), (dict(mode=2), "mode"),
             (dict(T=0), "T must be positive"), (dict(o=None), "null argument"), (dict(handle=plain._h), "not an expert")]
    for kw, why in cases:
        assert call(**kw) == MGB_ERR_ARG
        assert why in _lib.load().mgb_last_error().decode(), (kw, _lib.load().mgb_last_error().decode())
    assert L.mgb_maze_set_expert(h, 1) == MGB_ERR_ARG and "before mgb_maze_set_task" in _lib.load().mgb_last_error().decode()
    assert L.mgb_maze_expert(plain._h, _ptr(done), None, st) == MGB_ERR_ARG
    assert L.mgb_maze_expert(h, None, None, st) == MGB_ERR_ARG
    assert L.mgb_maze_expert_table(h, 3, 3, _ptr(done), None, st) == MGB_ERR_ARG and "slot" in _lib.load().mgb_last_error().decode()
    assert L.mgb_maze_step_expert(h, _ptr(done), _ptr(obs), _ptr(rew), _ptr(done), None, None, None, st) == MGB_ERR_ARG
    assert torch.equal(env.agent_state()[0], agent0) and env._counters() == t0
