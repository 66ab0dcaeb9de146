"""GPU tests of time-limit truncation flags for quadrotor steps (mgb_quad_step_ex / mgb_quad_step_host_ex) and of
terminal observations with truncation flags from the fused quadrotor and MetaMaze2D rollouts (mgb_quad_rollout_ex /
mgb_maze_rollout): against the CPU oracle, against step-driven twins bit for bit, and against handles without the new
outputs, whose primary outputs must not move."""
import numpy as np
import pytest

from test_maze_final_obs_gpu import MAX_STEPS, tasks, textures  # noqa: F401  (fixtures)
from test_quadrotor_gpu import (MATRIX_PATHS, MATRIX_TASKS, _done_flip_is_marginal, _kernel_suffix, _matrix_batch,
                                _stream_size, get_state, make_env, set_state)

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
STEP_PATHS = [p for p in MATRIX_PATHS if not p.startswith("rollout")]


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


def oracle_step(ob, act):
    """OracleBatch.step plus `truncated`: which branch of env.py:144-161 ended each episode.  The same step is restated
    once more with a time limit it cannot reach; what ends there is a collision or a failure (terminal), so
    truncated = done of the real step and not done of that one."""
    from oracle import quad_oracle as qo
    if ob.task == "velocity_control":            # no collision rule: only ct == nt and a failure end an episode
        r = ob.step(act)
        r.truncated = r.done & (r.fail == 0)
        return r
    st, ct = ob.state.copy(), ob.ct.copy()
    rows = np.ascontiguousarray(np.asarray(act, np.float32).reshape(ob.n, 4)[ob.idx])
    qo.set_map(ob.map_matrix)
    _, _, done_nolimit, _, _ = qo.env_step(ob.cfg, st, ct, rows, ob.task, ob.dt, 2 ** 31 - 1, ob.healthy, mode="mix")
    r = ob.step(act)
    r.truncated = r.done & ~done_nolimit.astype(bool)
    return r


def _edge_at_time_limit(env, ob, nt):
    """The edge envs of the path matrix (failures, floor and obstacle contacts, and their near misses: rows[k::17]) and
    a few plain ones start at ct = nt - 1, so that their first step also reaches the time limit."""
    st, ct = get_state(env)
    rows = ob.idx
    for k in range(8):
        ct[rows[k::17]] = nt - 1
    ct[rows[8::23]] = nt - 1
    set_state(env, st.astype(np.float32), ct)
    ob.ct[:] = ct[rows]


@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task,terrain", MATRIX_TASKS)
@pytest.mark.parametrize("path", STEP_PATHS)
def test_step_truncation_vs_oracle(torch_mod, quad_golden, monkeypatch, tmp_path, path, task, terrain, config):
    """Every step path (tile, wide, packed, streaming, host by copies, zero-copy and hybrid), both SIMPLE
    instantiations, nt = 7, auto-reset, edge envs whose failure or contact coincides with the time limit: truncated
    exactly on every env whose done agrees with the oracle (flips only where the oracle's deciding quantity is marginal,
    as in the path matrix), and 0 wherever done is 0."""
    torch = torch_mod
    from metagym_b200 import _lib
    kname, env_vars = MATRIX_PATHS[path]
    n = {"wide": 9473, "stream": _stream_size(), "host_zerocopy_stream": _stream_size()}.get(path, 4099)
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    env, ob, rng = _matrix_batch(n, task, terrain, config, quad_golden["map_obst"], str(tmp_path))
    for k in env_vars:
        monkeypatch.delenv(k)
    assert env.step_kernel_name() == kname + _kernel_suffix(config)
    _edge_at_time_limit(env, ob, 7)
    rows = ob.idx
    D = env.obs_dim
    if path.startswith("host"):
        def pinned(shape, dtype):
            return torch.zeros(shape, dtype=dtype).pin_memory()
        h_act, h_obs, h_rew = pinned((n, 4), torch.float32), pinned((n, D), torch.float32), pinned((n,), torch.float32)
        h_done, h_fail, h_final = pinned((n,), torch.uint8), pinned((n,), torch.int32), pinned((n, D), torch.float32)
        h_trunc = pinned((n,), torch.uint8)
    else:
        trunc = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
        fail = torch.zeros((n,), dtype=torch.int32, device="cuda")
        final = torch.zeros((n, D), dtype=torch.float32, device="cuda")
        obs, rew = torch.empty((n, D), device="cuda"), torch.empty((n,), device="cuda")
        done = torch.empty((n,), dtype=torch.uint8, device="cuda")
    accepted, n_trunc, n_term_at_limit = [], 0, 0
    for t in range(12):
        act = rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32)
        ct_before = ob.ct.copy()
        if path.startswith("host"):
            h_act.numpy()[:] = act
            _lib.check(env._lib.mgb_quad_step_host_ex(env._h, h_act.data_ptr(), h_obs.data_ptr(), h_rew.data_ptr(),
                                                      h_done.data_ptr(), h_fail.data_ptr(), h_final.data_ptr(),
                                                      h_trunc.data_ptr(), env._stream()))
            g_done, g_fail, g_trunc = h_done.numpy().copy(), h_fail.numpy().copy(), h_trunc.numpy().copy()
        else:
            a = torch.as_tensor(act).cuda()
            _lib.check(env._lib.mgb_quad_step_ex(env._h, a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(),
                                                 fail.data_ptr(), final.data_ptr(), trunc.data_ptr(), env._stream()))
            g_done, g_fail, g_trunc = done.cpu().numpy(), fail.cpu().numpy(), trunc.cpu().numpy()
        assert set(np.unique(g_trunc)) <= {0, 1}, t                 # written for every env
        assert not (g_trunc.astype(bool) & ~g_done.astype(bool)).any(), t
        r = oracle_step(ob, act)
        gd, gt = g_done[rows].astype(bool), g_trunc[rows].astype(bool)
        flip = gd != r.done
        for i in np.nonzero(flip)[0]:
            assert _done_flip_is_marginal(ob, r, i, g_fail[rows][i]), (t, int(rows[i]))
            accepted.append((t, int(rows[i])))
        ok = ~flip
        assert np.array_equal(g_fail[rows][ok], r.fail[ok]), t
        bad = np.nonzero(ok & (gt != r.truncated))[0]
        assert bad.size == 0, (t, rows[bad][:8], gt[bad][:8], r.truncated[bad][:8])
        n_trunc += int(r.truncated[ok].sum())
        n_term_at_limit += int((ok & r.done & ~r.truncated & (ct_before + 1 == 7)).sum())
        if flip.any():                          # resynchronise the flipped envs with the GPU's state
            gs, gc = get_state(env)
            ob.state[flip], ob.ct[flip] = gs[rows][flip], gc[rows][flip]
            ob.ep[flip] += g_done[rows][flip].astype(np.int64) - r.done[flip].astype(np.int64)
    assert n_trunc > 0
    assert n_term_at_limit > 0, "no terminal event coincided with the time limit"
    assert len(accepted) <= 3, accepted
    env.close()


def test_host_step_reports_truncated_as_numpy(torch_mod):
    """A numpy-action step() of a final_obs=True handle reports truncated as a numpy bool array, equal to the device
    path's torch tensor; the final_obs=False handle reports None."""
    torch = torch_mod
    kw = dict(nt=3, auto_reset=True, rng_seed=4)
    h = make_env(300, "hovering_control", final_obs=True, **kw)
    d = make_env(300, "hovering_control", final_obs=True, **kw)
    off = make_env(300, "hovering_control", **kw)
    assert off.truncated is None
    for e in (h, d, off):
        e.reset()
    rng = np.random.RandomState(1)
    n_trunc = 0
    for t in range(5):
        act = rng.uniform(0.1, 15.0, (300, 4)).astype(np.float32)
        _, _, done_h, _ = h.step(act)
        _, _, done_d, _ = d.step(torch.as_tensor(act).cuda())
        assert isinstance(h.truncated, np.ndarray) and h.truncated.dtype == np.bool_
        assert np.array_equal(h.truncated, d.truncated.cpu().numpy())
        assert np.array_equal(done_h, done_d.cpu().numpy())
        assert np.array_equal(h.final_observation, d.final_observation.cpu().numpy())
        n_trunc += int(h.truncated.sum())
    assert n_trunc >= 300                    # nt = 3: every env reaches the limit on step 3
    for e in (h, d, off):
        e.close()


def test_single_env_truncated_is_squeezed(torch_mod):
    from metagym_b200 import BatchedQuadrotor
    env = BatchedQuadrotor(task="hovering_control", nt=2, num_envs=1, auto_reset=True, final_obs=True)
    env.reset()
    for t in range(2):
        env.step(torch_mod.full((1, 4), 5.0, device="cuda"))
    assert env.truncated.shape == () and bool(env.truncated)
    env.close()


# --------------------------------------------------------------------------------------------------------------------
# quadrotor rollout = steps
# --------------------------------------------------------------------------------------------------------------------
def _quad_pair(task, config, n, final_obs=True, **kw):
    from oracle import quad_oracle as qo
    params = qo.general_params() if config == "general" else None
    vel = task == "velocity_control"
    kw = dict(dict(dt=0.005 if vel else 0.01, nt=3, auto_reset=True, rng_seed=21, simulator_conf=params), **kw)
    if vel:
        kw["seed"] = list(range(3))
    return [make_env(n, task, final_obs=final_obs, **kw) for _ in range(2)]


@pytest.mark.parametrize("config", ["default", "general"])
@pytest.mark.parametrize("task", ["hovering_control", "velocity_control", "no_collision"])
@pytest.mark.parametrize("drawn", [False, True], ids=["given", "drawn"])
def test_quad_rollout_ex_equals_steps(torch_mod, drawn, task, config):
    """nt = 3, T = 8 (every env finishes twice in one launch): rollout_ex against a step_ex-driven twin bit for bit --
    obs, rew, done, truncated, and final_obs where done; rows with done 0 keep the NaN they were filled with; the end
    state and ct equal."""
    torch = torch_mod
    n, T = 4099, 8
    roll, twin = _quad_pair(task, config, n)
    for e in (roll, twin):
        e.reset()
    D = roll.obs_dim
    out = {"obs": torch.empty((T, n, D), device="cuda"), "rew": torch.empty((T, n), device="cuda"),
           "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"),
           "act": torch.empty((T, n, 4), device="cuda") if drawn else None,
           "final_obs": torch.full((T, n, D), float("nan"), device="cuda"),
           "truncated": torch.full((T, n), 7, dtype=torch.uint8, device="cuda")}
    if drawn:
        roll.rollout(T, act_seed=5, out=out)
        acts = out["act"]
    else:
        g = torch.Generator(device="cuda").manual_seed(3)
        acts = torch.rand((T, n, 4), device="cuda", generator=g) * 14.9 + 0.1
        roll.rollout(T, actions=acts, out=out)
    finished = torch.zeros(n, dtype=torch.int32, device="cuda")
    for t in range(T):
        o, r, d, _ = twin.step(acts[t].contiguous())
        assert torch.equal(out["obs"][t], o) and torch.equal(out["rew"][t], r), t
        assert torch.equal(out["done"][t].bool(), d), t
        assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
        assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
        assert torch.isnan(out["final_obs"][t][~d]).all(), t
        finished += d.int()
    assert int(finished.min()) >= 2
    assert bool(out["truncated"].any())
    s1, s2 = roll.state_dict(), twin.state_dict()
    assert torch.equal(s1["state"], s2["state"]) and torch.equal(s1["ct"], s2["ct"])
    for e in (roll, twin):
        e.close()


def test_quad_new_outputs_move_nothing(torch_mod):
    """A final_obs=True handle and a final_obs=False handle give identical obs / rew / done / fail / final_observation /
    state on the step path and obs / rew / done / drawn actions / state on the rollout path; rollout_ex with both new
    outputs NULL equals mgb_quad_rollout."""
    torch = torch_mod
    from metagym_b200 import _lib
    n, T = 9473, 9
    on, _ = _quad_pair("hovering_control", "default", n, nt=4)
    off, off2 = _quad_pair("hovering_control", "default", n, final_obs=False, nt=4)
    for e in (on, off, off2):
        e.reset()
    rng = np.random.RandomState(2)
    for t in range(6):
        a = torch.as_tensor(rng.uniform(0.1, 15.0, (n, 4)).astype(np.float32)).cuda()
        r_on = [x.clone() for x in on.step(a)[:3]]
        r_off = [x.clone() for x in off.step(a)[:3]]
        off2.step(a)
        assert all(torch.equal(x, y) for x, y in zip(r_on, r_off)), t
        assert torch.equal(on.fail_code, off.fail_code) and torch.equal(on.final_observation, off.final_observation)
    ra = on.rollout(T, act_seed=3, want_actions=True)
    rb = off.rollout(T, act_seed=3, want_actions=True)
    assert "final_obs" in ra and "final_obs" not in rb
    for k in ("obs", "rew", "done", "act"):
        assert torch.equal(ra[k], rb[k]), k
    D = off2.obs_dim
    rc = {"obs": torch.empty((T, n, D), device="cuda"), "rew": torch.empty((T, n), device="cuda"),
          "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"), "act": torch.empty((T, n, 4), device="cuda")}
    _lib.check(off2._lib.mgb_quad_rollout_ex(off2._h, T, None, 3, rc["act"].data_ptr(), rc["obs"].data_ptr(),
                                             rc["rew"].data_ptr(), rc["done"].data_ptr(), None, None, off2._stream()))
    for k in ("obs", "rew", "done", "act"):
        assert torch.equal(rc[k], rb[k]), k
    s = [e.state_dict() for e in (on, off, off2)]
    for x in s[1:]:
        assert torch.equal(s[0]["state"], x["state"]) and torch.equal(s[0]["ct"], x["ct"])
    for e in (on, off, off2):
        e.close()


def test_quad_sharding_invariance_full_size(torch_mod):
    """65 536 envs: two env_index_base halves reproduce one full handle's truncated and final_obs, on the step path
    and on the rollout path."""
    torch = torch_mod
    N, T = 65536, 12
    kw = dict(dt=0.005, nt=8, seed=list(range(64)), auto_reset=True, rng_seed=77, final_obs=True)
    full = make_env(N, "velocity_control", **kw)
    lo = make_env(N // 2, "velocity_control", env_index_base=0, **kw)
    hi = make_env(N // 2, "velocity_control", env_index_base=N // 2, **kw)
    for e in (full, lo, hi):
        e.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = torch.rand((T, N, 4), device="cuda", generator=g) * 14.9 + 0.1
    for t in range(T):
        full.step(acts[t])
        lo.step(acts[t, : N // 2].contiguous())
        hi.step(acts[t, N // 2:].contiguous())
        assert torch.equal(full.truncated, torch.cat([lo.truncated, hi.truncated])), t
        assert torch.equal(full.final_observation, torch.cat([lo.final_observation, hi.final_observation])), t
    outs = []
    for e in (full, lo, hi):
        n = e.num_envs
        out = {"obs": torch.empty((T, n, 19), device="cuda"), "rew": torch.empty((T, n), device="cuda"),
               "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"), "act": None,
               "final_obs": torch.zeros((T, n, 19), device="cuda"),
               "truncated": torch.empty((T, n), dtype=torch.uint8, device="cuda")}
        outs.append(e.rollout(T, act_seed=4, out=out))
    for k in ("final_obs", "truncated", "done"):
        assert torch.equal(outs[0][k], torch.cat([outs[1][k], outs[2][k]], dim=1)), k
    assert int(outs[0]["truncated"].sum()) >= N       # nt = 8: every env reaches the limit once in 12 steps
    for e in (full, lo, hi):
        e.close()


def test_quad_graph_capture_of_step(torch_mod):
    """A captured final_obs=True step(), replayed, equals eager steps: obs, rew, done, truncated, final_observation."""
    torch = torch_mod
    n = 4099
    cap, eager = _quad_pair("no_collision", "default", n, nt=3)
    for e in (cap, eager):
        e.reset()
    act = torch.full((n, 4), 0.1, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        cap.step(act)                                # warm-up (allocates nothing new: the buffers are persistent)
        eager.step(act)
    torch.cuda.current_stream().wait_stream(s)
    st, ct = get_state(cap)
    st[0::2, 2], st[0::2, 5] = -4.995, -2.0           # even envs 5 mm above the floor, sinking: they hit it at once
    ct[:] = np.arange(n) % 3
    for e in (cap, eager):
        set_state(e, st.astype(np.float32), ct)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap.step(act)
    seen = 0
    for t in range(7):
        graph.replay()
        o, r, d, _ = eager.step(act)
        torch.cuda.synchronize()
        assert torch.equal(cap._obs, o) and torch.equal(cap._rew, r) and torch.equal(cap._done.bool(), d), t
        assert torch.equal(cap.truncated, eager.truncated), t
        assert torch.equal(cap.final_observation, eager.final_observation), t
        seen |= int(eager.truncated.any()) << 0 | int((d & ~eager.truncated).any()) << 1
    assert seen == 3                                  # both truncations and terminations were replayed
    for e in (cap, eager):
        e.close()


# --------------------------------------------------------------------------------------------------------------------
# MetaMaze2D rollout = steps
# --------------------------------------------------------------------------------------------------------------------
def _maze2d(task_type, view_grid, n, final_obs, auto_reset=True):
    from metagym_b200 import BatchedMetaMaze2D
    return BatchedMetaMaze2D(max_steps=MAX_STEPS, task_type=task_type, view_grid=view_grid, num_envs=n, squeeze=False,
                             auto_reset=auto_reset, final_obs=final_obs)


@pytest.mark.parametrize("drawn", [False, True], ids=["given", "drawn"])
@pytest.mark.parametrize("view_grid", [1, 2])
@pytest.mark.parametrize("task_type", ["SURVIVAL", "ESCAPE"])
def test_maze2d_rollout_ex_equals_steps(torch_mod, tasks, task_type, view_grid, drawn):  # noqa: F811
    """max_steps = 17 over four tasks whose episodes end by death (one on the last allowed step), by the goal and by
    the step limit: rollout_ex against a final_obs=True step twin bit for bit -- obs, rew, done, truncated, final_obs
    where done; NaN kept where done is 0; the agent state at the end.  A final_obs=False handle's rollout gives the same
    primary outputs."""
    torch = torch_mod
    n, T = 64, 60
    roll, twin, plain = (_maze2d(task_type, view_grid, n, f) for f in (True, True, False))
    for e in (roll, twin, plain):
        e.set_task(tasks)
        e.reset()
    W = 2 * view_grid + 1
    out = {"obs": torch.empty((T, n, W, W), device="cuda"), "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
           "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"),
           "act": torch.empty((T, n), dtype=torch.int32, device="cuda") if drawn else None,
           "final_obs": torch.full((T, n, W, W), float("nan"), device="cuda"),
           "truncated": torch.full((T, n), 7, dtype=torch.uint8, device="cuda")}
    if drawn:
        roll.rollout(T, act_seed=8, out=out)
        acts = out["act"]
        ref = plain.rollout(T, act_seed=8, want_actions=True)
        assert torch.equal(ref["act"], acts)
    else:
        acts = torch.as_tensor(np.random.RandomState(5).randint(0, 4, (T, n)).astype(np.int32)).cuda()
        roll.rollout(T, actions=acts, out=out)
        ref = plain.rollout(T, actions=acts)
    assert "final_obs" not in ref
    for k in ("obs", "rew", "done"):
        assert torch.equal(ref[k], out[k]), k
    kinds = np.zeros(3, np.int64)      # terminal, truncated, terminal on the last allowed step
    for t in range(T):
        steps_before = twin.agent_state()[0][:, 3].cpu().numpy()
        o, r, d, info = twin.step(acts[t].contiguous())
        assert torch.equal(out["obs"][t], o) and torch.equal(out["rew"][t], r), t
        assert torch.equal(out["done"][t].bool(), d), t
        assert torch.equal(out["truncated"][t].bool(), twin.truncated), t
        assert torch.equal(out["final_obs"][t][d], twin.final_observation[d]), t
        assert torch.isnan(out["final_obs"][t][~d]).all(), t
        term = (d & ~twin.truncated).cpu().numpy()
        kinds += [term.sum(), twin.truncated.sum().item(), (term & (steps_before + 1 == MAX_STEPS)).sum()]
    ag_r, life_r = roll.agent_state()
    ag_t, life_t = twin.agent_state()
    assert torch.equal(ag_r, ag_t) and torch.equal(life_r, life_t)
    assert kinds[0] > 0 and kinds[1] > 0, kinds
    if task_type == "SURVIVAL":
        assert kinds[2] > 0, kinds     # a death on the last allowed step is terminal, not truncated
    for e in (roll, twin, plain):
        e.close()


# --------------------------------------------------------------------------------------------------------------------
# refusals
# --------------------------------------------------------------------------------------------------------------------
def test_final_obs_refusals(torch_mod, tasks, textures):  # noqa: F811
    torch = torch_mod
    from metagym_b200 import BatchedMetaMazeDiscrete3D, BatchedQuadrotor
    with pytest.raises(ValueError, match="auto_reset"):
        BatchedQuadrotor(task="hovering_control", num_envs=8, final_obs=True)
    T, n = 2, 8
    u8 = torch.zeros((T, n), dtype=torch.uint8, device="cuda")
    # quadrotor: final_obs without auto-reset; either output with mirrors or multicast
    q = make_env(n, "hovering_control")
    q.reset()
    fo = torch.zeros((T, n, q.obs_dim), device="cuda")
    assert q._lib.mgb_quad_rollout_ex(q._h, T, None, 0, None, None, None, None, fo.data_ptr(), None, q._stream()) \
        == MGB_ERR_ARG
    assert q._lib.mgb_quad_rollout_ex(q._h, T, None, 0, None, None, None, None, None, u8.data_ptr(), q._stream()) == 0
    qa = make_env(n, "hovering_control", auto_reset=True, final_obs=True)
    qa.reset()
    for arm in (lambda: qa.set_mirrors([16]), lambda: qa.set_multicast(16)):
        arm()
        for f, tr in ((fo, None), (None, u8)):
            assert qa._lib.mgb_quad_rollout_ex(qa._h, T, None, 0, None, None, None, None, _ptr(f), _ptr(tr),
                                               qa._stream()) == MGB_ERR_ARG
        qa.set_mirrors([])
    assert "truncated" in qa.rollout(T)                # usable again once the mirrors are off
    # MetaMaze2D: the same rules
    m = _maze2d("SURVIVAL", 1, n, False, auto_reset=False)
    m.set_task(tasks)
    m.reset()
    mfo = torch.zeros((T, n, 3, 3), device="cuda")
    assert m._lib.mgb_maze_rollout(m._h, T, None, 0, None, None, None, None, mfo.data_ptr(), None, None, 0,
                                   m._stream()) == MGB_ERR_ARG
    ma = _maze2d("SURVIVAL", 1, n, True)
    ma.set_task(tasks)
    ma.reset()
    for arm in (lambda: ma.set_mirrors([16]), lambda: ma.set_multicast(16)):
        arm()
        for f, tr in ((mfo, None), (None, u8)):
            assert ma._lib.mgb_maze_rollout(ma._h, T, None, 0, None, None, None, None, _ptr(f), _ptr(tr), None, 0,
                                            ma._stream()) == MGB_ERR_ARG
        ma.set_mirrors([])
    # discrete 3-D: the same call runs on the pose cache, as rollout(T, final_obs=True) of a twin does
    d3, twin = (BatchedMetaMazeDiscrete3D(resolution=(32, 32), obs_dtype="uint8", textures=textures, max_steps=MAX_STEPS,
                                          num_envs=n, squeeze=False, auto_reset=True, final_obs=True) for _ in range(2))
    for e in (d3, twin):
        e.set_task(tasks)
        e.reset()
    f3 = torch.zeros((T, n, 32, 32, 3), dtype=torch.uint8, device="cuda")
    for f, tr in ((f3, None), (None, u8)):
        assert d3._lib.mgb_maze_rollout(d3._h, T, None, 0, None, None, None, None, _ptr(f), _ptr(tr), None, 0,
                                        d3._stream()) == 0
        want = twin.rollout(T, final_obs=True)
        d = want["done"].bool()
        assert torch.equal(f3[d], want["final_obs"][d]) if tr is None else torch.equal(u8, want["truncated"])
    assert "final_obs" not in d3.rollout(T)
    torch.cuda.synchronize()
    for e in (q, qa, m, ma, d3, twin):
        e.close()


def _ptr(t):
    return None if t is None else t.data_ptr()
