"""GPU: every compiled critic (VAL) instantiation, checked at the shapes and edges the per-feature critic tests skip.

The library compiles maze2d_rollout_kernel<0, true, REC, RS, POL, true> for the three policy kinds over path recording
(REC) and in-launch resampling (RS), 12 instantiations, and quad_rollout_kernel<SIMPLE, 0, true, true, true> for the
default physics (SIMPLE) and qo.general_params(), 2 more.  Each one is launched here at least once, and each case checks:

- every output that is not the critic's bit for bit against the same policy without a value head (and the trajectory
  with REC, the env and carried state, the snapshot records);
- value and final_value within the float64 bounds of test_critic_rollout_gpu, final_value written exactly where the
  cut fires on a truncated step (a NaN-filled buffer elsewhere);
- adv / ret bit for bit against critic_ref.gae_f32 at the case's (gamma, lambda);
- value_last equal to the next launch's value[0].

On top of that: GAE at the ends of [0, 1], T = 1, deterministic=True, handles built with final_obs=False, the null-output
contract of the three *_critic entry points, batch tails, populations whose CTAs stage several members, value heads
without bias, an MLP without hidden layers whose normalisation folds into the value row, and the shared-memory
footprint with the value row (DESIGN.md "Recurrent policies", "Value heads and GAE").
"""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

import test_lstm_policy_rollout_maze_gpu as lstm_t  # noqa: E402
import test_policy_rollout_gpu as quad_t  # noqa: E402
import test_policy_rollout_maze_gpu as mlp_t  # noqa: E402
import test_rnn_policy_rollout_maze_gpu as gru_t  # noqa: E402
from critic_ref import gae_f32  # noqa: E402
from test_critic_rollout_gpu import (assert_rest_equal, check_final_written, cut_mask, maze_env, maze_reference,  # noqa: E402
                                     nan_out, value_net, with_value, within)
from test_maze2d_resample_rollout_gpu import CFG  # noqa: E402
from test_policy_rollout_gpu import forward_bound  # noqa: E402
from test_policy_rollout_matrix_gpu import (LOG_STD, OPTIN_H100, SEED, Shape, assert_boundary,  # noqa: E402
                                            assert_drops_change_nothing, footprint_env, general, make_quad, maze_outputs,
                                            largest_h, maze_pair, mlp_staged, quad_outputs, sentinel, smem_bytes)
from test_maze_final_obs_gpu import tasks  # noqa: E402,F401  (fixture)

pytestmark = pytest.mark.gpu

MGB_ERR_ARG = -1
U = 2.0 ** -24
GAES = [(0.97, 0.9), (1.0, 1.0), (0.0, 0.5), (0.9, 0.0), (1.0, 0.0)]


@pytest.fixture(autouse=True)
def _needs_gpu(cuda_device):
    return cuda_device


class RefView:
    """What maze_reference and the checks read of a critic: its reset rule and a value layer whose absent bias is a zero
    bias (the float64 bounds read lin.bias)."""

    def __init__(self, critic):
        self.hidden_reset = getattr(critic, "hidden_reset", "episode")
        v = critic._value
        if v.bias is None:
            w = nn.Linear(v.in_features, 1)
            with torch.no_grad():
                w.weight.copy_(v.weight)
                w.bias.zero_()
            v = w
        self._value = v


def without_bias(critic):
    """The critic with its value layer's bias removed (packed as a zero)."""
    v = critic._value
    v.bias = None
    return critic.update(value=v)


def check_gae_at(pol, out, gae):
    cut = cut_mask(pol, out).cpu().numpy()
    adv, ret = gae_f32(out["rew"].cpu().numpy(), cut, out["truncated"].cpu().numpy(), out["value"].cpu().numpy(),
                       out["value_last"].cpu().numpy(), out["final_value"].cpu().numpy(), *gae)
    assert np.array_equal(out["adv"].cpu().numpy(), adv)
    assert np.array_equal(out["ret"].cpu().numpy(), ret)


def maze_roll(env, pol, T, state, rs, gae=None, out=None, deterministic=False):
    kw = dict(state=state, want_hidden=True) if state is not None else {}
    return env.rollout(T, policy=pol, act_seed=SEED, resample=dict(seed=SEED, **CFG) if rs else None, gae=gae,
                       out=out, deterministic=deterministic, **kw)


def maze_critic_case(a, b, shape, T, rs, gae, rec=False, plain=None, module=None, deterministic=False, bias=True,
                     seed=5):
    """The policy on handle a and the same policy with a value head on its identical twin b; every check of the module
    docstring.  Returns (critic, outputs, the mask where final_value was written)."""
    n = a.num_envs
    if plain is None:
        module, plain = shape.policy(a, seed=seed)
    critic = with_value(plain, seed)
    if not bias:
        critic = without_bias(critic)
    sa = sb = None
    if shape.kind != "mlp":
        sa = gru_t.random_state(plain, n)
        sb = sa.clone()
    ref = maze_roll(a, plain, T, sa, rs, deterministic=deterministic)
    out = maze_roll(b, critic, T, sb, rs, gae, nan_out(ref, T, n, b.device), deterministic)
    assert_rest_equal(ref, out)
    assert ("adv" in out) == (gae is not None) and "final_value" in out
    if sa is not None:
        assert torch.equal(sa, sb)
    for x, y in zip(a.agent_state(), b.agent_state()):
        assert torch.equal(x, y)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])
    if rec:
        for x, y in zip(a.trajectory(), b.trajectory()):
            assert torch.equal(x, y)
    with torch.no_grad():
        if shape.kind == "mlp" and plain._mean is not None:
            where = folded_reference(critic, out, T, n)
        else:
            where = maze_reference(shape.kind, plain, RefView(critic), module, out)
    if gae is not None:
        check_gae_at(critic, out, gae)
    nxt = maze_roll(b, critic, 2, sb, rs, deterministic=deterministic)
    assert torch.equal(nxt["value"][0], out["value_last"])
    assert_rest_equal(maze_roll(a, plain, 2, sa, rs, deterministic=deterministic), nxt)     # the twins stay in step
    return critic, out, where


def folded_reference(critic, out, T, n):
    """An MLP without hidden layers and with obs_mean / obs_std: V = ((x - mean) / std) w + b in float64 against the
    kernel's fma chain over the folded float32 row (w / std, b - w mean / std), whose rounding adds one u per term."""
    D = critic.obs_dim
    w = critic._value.weight.detach().double().cpu()[0]
    b = float(critic._value.bias.detach()) if critic._value.bias is not None else 0.0
    mean, std = critic._mean, critic._std
    wf = critic.params.detach().double().cpu()[4 * D:5 * D]
    bf = float(critic.params[5 * D + 4])

    def check(got, x):
        x = x.double().cpu()
        want = ((x - mean) / std) @ w + b
        bound = (D + 2) * U * (x.abs() @ wf.abs() + abs(bf)) + 1e-12 * (1 + want.abs())
        within(got.cpu(), want, bound)
    pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).reshape(T, n, -1)
    check(out["value"], pre)
    where = check_final_written(critic, out)
    check(out["final_value"][where], out["final_obs"].reshape(T, n, -1)[where])
    return where


# ---------------------------------------------------------------------------------------------------------------
# 1. The maze critic matrix: kind x REC x RS, one case per compiled VAL kernel
# ---------------------------------------------------------------------------------------------------------------

# one shape per (REC, RS) in product order: H in {1, 8, 17, 64}, head widths 0, 5, 13 and 64, both activations, both
# task types, feedback on and off, both reset rules ("task" only with resampling, where the rule can fire)
CRITIC_SHAPES = {
    "mlp": [Shape("mlp", (17,), act=nn.ReLU), Shape("mlp", (64, 64), task_type="ESCAPE"),
            Shape("mlp", (5, 64, 13), act=nn.ReLU, view_grid=2), Shape("mlp", (13,), task_type="ESCAPE")],
    "gru": [Shape("gru", H=1, width=5, feedback=False), Shape("gru", H=17, width=13, act=nn.ReLU, reset="task"),
            Shape("gru", H=64, width=0, task_type="ESCAPE"), Shape("gru", H=8, width=64, view_grid=2)],
    "lstm": [Shape("lstm", H=64, width=64, act=nn.ReLU), Shape("lstm", H=8, width=0, feedback=False, task_type="ESCAPE"),
             Shape("lstm", H=17, width=5, view_grid=2), Shape("lstm", H=1, width=13, act=nn.ReLU, reset="task")],
}
MATRIX = [(kind, rec, rs, CRITIC_SHAPES[kind][2 * rec + rs], GAES[(3 * i + 2 * rec + rs) % len(GAES)])
          for i, kind in enumerate(("mlp", "gru", "lstm")) for rec in (0, 1) for rs in (0, 1)]


@pytest.mark.parametrize("kind,rec,rs,shape,gae", MATRIX,
                         ids=["%s-rec%d-rs%d-%r-g%s-l%s" % (k, r, s, sh, g[0], g[1]) for k, r, s, sh, g in MATRIX])
def test_maze_critic_matrix(tasks, kind, rec, rs, shape, gae):  # noqa: F811
    n, T = 300, 40
    a, b = maze_pair(n, shape, rs, rec, True, tasks)
    _, _, where = maze_critic_case(a, b, shape, T, rs, gae, rec=bool(rec))
    assert where.any(), "no truncated cut: final_value is not exercised"
    for e in (a, b):
        e.close()


TRIAL = [("gru", Shape("gru", H=17, width=0, reset="task")), ("lstm", Shape("lstm", H=8, width=13, reset="task")),
         ("mlp", Shape("mlp", (64,)))]


@pytest.mark.parametrize("kind,shape", TRIAL, ids=[k for k, _ in TRIAL])
def test_maze_critic_trial_handle(kind, shape):
    """A k = 2 trial handle with resampling: under the task rule the cut (and GAE's) spans the trial's two episodes."""
    n, T = 300, 30
    a, b = maze_env(n, shape, k=2), maze_env(n, shape, k=2)
    critic, out, where = maze_critic_case(a, b, shape, T, True, (0.9, 0.0))
    assert where.any()
    if kind != "mlp":
        assert (out["done"].bool() & ~cut_mask(critic, out)).any()
    for e in (a, b):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 2. The quadrotor critic instantiations: default physics and qo.general_params(), RK4 on one
# ---------------------------------------------------------------------------------------------------------------

def quad_pair(n, task, simple=True, **kw):
    kw = dict(dict(nt=11, final_obs=True, auto_reset=True, simulator_conf=None if simple else general()), **kw)
    envs = []
    for _ in range(2):
        e = make_quad(n, task, **kw)
        e.reset()
        e.rollout(5)                                 # t_base != 0
        envs.append(e)
    return envs


def quad_critic_case(a, b, T, gae, widths=(64, 17), act=nn.Tanh, plain=None, module=None, deterministic=False,
                     bias=True):
    n = a.num_envs
    if plain is None:
        module, plain = quad_t.make_policy(a, widths, act, 3, LOG_STD)
    critic = with_value(plain, 1)
    if not bias:
        critic = without_bias(critic)
    ref = a.rollout(T, policy=plain, act_seed=SEED, deterministic=deterministic)
    out = b.rollout(T, policy=critic, act_seed=SEED, gae=gae, deterministic=deterministic,
                    out=nan_out(ref, T, n, b.device))
    assert_rest_equal(ref, out)
    assert torch.equal(a.snapshot()["records"], b.snapshot()["records"])
    with torch.no_grad():
        if plain._mean is None:
            net = value_net(RefView(critic), module)
            pre = torch.cat([out["obs0"][None], out["obs"][:-1]], 0).double()
            v, vb = forward_bound(net, pre)
            within(out["value"], v[..., 0], vb[..., 0])
            where = check_final_written(critic, out)
            fv, fb = forward_bound(net, out["final_obs"][where].double())
            within(out["final_value"][where], fv[..., 0], fb[..., 0])
        else:
            where = folded_reference(critic, out, T, n)
    if gae is not None:
        check_gae_at(critic, out, gae)
    nxt = b.rollout(2, policy=critic, act_seed=SEED, deterministic=deterministic)
    assert torch.equal(nxt["value"][0], out["value_last"])
    assert_rest_equal(a.rollout(2, policy=plain, act_seed=SEED, deterministic=deterministic), nxt)
    return critic, out, where


QUAD = [("default", "velocity_control", False, (64, 17), nn.Tanh, (0.97, 0.9)),
        ("general", "hovering_control", False, (33,), nn.ReLU, (1.0, 1.0)),
        ("default-rk4", "no_collision", True, (13, 5), nn.ReLU, (0.0, 0.5)),
        ("general-rk4", "velocity_control", True, (64, 64, 64), nn.Tanh, (1.0, 0.0))]


@pytest.mark.parametrize("phys,task,rk4,widths,act,gae", QUAD, ids=[q[0] for q in QUAD])
def test_quad_critic_matrix(phys, task, rk4, widths, act, gae):
    simple = phys.startswith("default")
    kw = dict(integrator="rk4", rk4_steps=2) if rk4 else {}
    a, b = quad_pair(300, task, simple, **kw)
    assert b.step_kernel_name().endswith("<true>" if simple else "<false>")
    _, _, where = quad_critic_case(a, b, 32, gae, widths, act)
    assert where.any()
    for e in (a, b):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 3. GAE at the ends of [0, 1], T = 1, deterministic=True, value heads without bias, folded normalisation
# ---------------------------------------------------------------------------------------------------------------

EDGES = [(kind, gae) for kind in ("mlp", "gru", "lstm") for gae in GAES[1:]]


@pytest.mark.parametrize("kind,gae", EDGES, ids=["%s-g%s-l%s" % (k, g[0], g[1]) for k, g in EDGES])
def test_maze_gae_edges(kind, gae):
    shape = {"mlp": Shape("mlp", (33, 17)), "gru": Shape("gru", H=17, width=13),
             "lstm": Shape("lstm", H=8, width=5, reset="task")}[kind]
    a, b = maze_env(256, shape), maze_env(256, shape)
    _, out, where = maze_critic_case(a, b, shape, 24, True, gae)
    assert where.any()
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("gae", GAES[1:], ids=["g%s-l%s" % g for g in GAES[1:]])
def test_quad_gae_edges(gae):
    a, b = quad_pair(256, "velocity_control")
    quad_critic_case(a, b, 32, gae)
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm", "quad"])
def test_T1_deterministic_and_no_bias(tasks, kind):  # noqa: F811
    """Three launches of T = 1 (value_last carried across), then a deterministic launch; the value head has no bias."""
    if kind == "quad":
        a, b = quad_pair(200, "hovering_control")
        module, plain = quad_t.make_policy(a, (64, 17), nn.Tanh, 3, LOG_STD)
        for det in (False, False, False, True):
            critic, out, _ = quad_critic_case(a, b, 1 if not det else 16, (0.97, 0.9), plain=plain, module=module,
                                              deterministic=det, bias=False)
            assert (out["logp"] is None) == det
    else:
        shape = {"mlp": Shape("mlp", (8,)), "gru": Shape("gru", H=8, width=5), "lstm": Shape("lstm", H=17, width=0)}[kind]
        a, b = maze_pair(200, shape, False, False, True, tasks)
        module, plain = shape.policy(a, seed=4)
        for det in (False, False, False, True):
            critic, out, _ = maze_critic_case(a, b, shape, 1 if not det else 16, False, (0.9, 0.0), plain=plain,
                                              module=module, deterministic=det, bias=False)
            assert (out["logp"] is None) == det
    assert critic._value.bias is None
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("env_kind", ["maze", "quad"])
def test_folded_normalisation_in_the_value_row(tasks, env_kind):  # noqa: F811
    """An MLP without hidden layers with obs_mean / obs_std: pack() folds the normalisation into the value row too."""
    from metagym_b200.policy import MLPPolicy
    if env_kind == "maze":
        a, b = maze_pair(300, Shape("mlp", ()), True, False, True, tasks)
        D = a._obs[0].numel()
        module, _ = mlp_t.make_policy(a, ())
        kw = {}
    else:
        a, b = quad_pair(300, "velocity_control")
        D = a.obs_dim
        module, _ = quad_t.make_policy(a, (), nn.Tanh, 3, LOG_STD)
        kw = dict(log_std=torch.tensor(LOG_STD))
    g = torch.Generator().manual_seed(7)
    mean, std = torch.randn(D, generator=g) * 0.5, 0.25 + torch.rand(D, generator=g) * 2
    plain = MLPPolicy(module, obs_mean=mean, obs_std=std, device=a.device, **kw)
    if env_kind == "maze":
        _, _, where = maze_critic_case(a, b, Shape("mlp", ()), 40, True, (0.97, 0.9), plain=plain, module=module)
    else:
        _, _, where = quad_critic_case(a, b, 32, (0.97, 0.9), plain=plain, module=module)
    assert where.any()
    for e in (a, b):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 4. Handles built with final_obs=False
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["mlp", "gru", "lstm", "quad"])
def test_final_obs_off(tasks, kind):  # noqa: F811
    """Without gae the launch gets a NULL final_value_dev (and no truncated): value and value_last equal those of a
    final_obs=True twin.  With gae the rollout allocates final_value and truncated itself: adv and ret equal the twin's."""
    n, T = 300, 32
    if kind == "quad":
        off, on = quad_pair(n, "velocity_control", final_obs=False)[0], quad_pair(n, "velocity_control")[0]
        _, pol = quad_t.make_policy(off, (64, 17), nn.Tanh, 3, LOG_STD)
        state = None
    else:
        shape = {"mlp": Shape("mlp", (17, 5)), "gru": Shape("gru", H=17, width=5, reset="task"),
                 "lstm": Shape("lstm", H=8, width=13)}[kind]
        off, on = (maze_pair(n, shape, True, False, fin, tasks)[0] for fin in (False, True))
        _, pol = shape.policy(off, seed=2)
        state = gru_t.random_state(pol, n) if kind != "mlp" else None
    critic = with_value(pol, 3)
    st = [None if state is None else state.clone() for _ in range(2)]

    def roll(env, s, gae):
        if kind == "quad":
            return env.rollout(T, policy=critic, act_seed=SEED, gae=gae)
        return maze_roll(env, critic, T, s, True, gae)
    for gae in (None, (0.9, 0.9)):
        x, y = roll(off, st[0], gae), roll(on, st[1], gae)
        assert "final_obs" not in x and "final_obs" in y
        keys = ["value", "value_last", "act", "rew", "done"]
        if gae is None:
            assert "final_value" not in x and "truncated" not in x
        else:
            keys += ["adv", "ret", "truncated"]
        for k in keys:
            assert torch.equal(x[k], y[k]), (gae, k)
        if state is not None:
            assert torch.equal(st[0], st[1])
    for e in (off, on):
        e.close()


# ---------------------------------------------------------------------------------------------------------------
# 5. The null-output contract of mgb_maze_rollout_critic, mgb_maze_rollout_rnn_critic and mgb_quad_rollout_critic
# ---------------------------------------------------------------------------------------------------------------

ENV_OPTIONAL = ("act", "logp", "obs0", "obs", "final_obs")
ALWAYS = ("rew", "done", "truncated", "value")


def critic_call(env, kind, critic, T, out, state, rs, gae):
    """The *_critic entry point called directly, with exactly the buffers in `out`."""
    from metagym_b200 import _lib
    lib = env._lib
    p = _lib.ptr
    g = out.get
    cr = _lib.Critic(p(g("value")), p(g("value_last")), p(g("final_value")), p(g("adv")), p(g("ret")),
                     *(gae or (1.0, 1.0)))
    pol = critic.struct()
    if kind == "quad":
        rc = lib.mgb_quad_rollout_critic(env._h, T, ctypes.byref(pol), 1, 0, SEED, p(g("act")), p(g("logp")),
                                         p(g("obs0")), p(g("obs")), p(g("rew")), p(g("done")), p(g("final_obs")),
                                         p(g("truncated")), ctypes.byref(cr), env._stream())
    else:
        cfg, seed = env._sampler_cfg(seed=SEED, **CFG) if rs else (None, 0)
        head = [env._h, T, ctypes.byref(pol), 1, 0, SEED, None if cfg is None else ctypes.byref(cfg), seed]
        tail = [p(g(k)) for k in ("act", "logp", "obs0", "obs", "rew", "done", "final_obs", "truncated")]
        if kind == "mlp":
            rc = lib.mgb_maze_rollout_critic(*head, *tail, ctypes.byref(cr), env._stream())
        else:
            rc = lib.mgb_maze_rollout_rnn_critic(*head, p(state), p(g("state0")), p(g("hid")), *tail,
                                                 ctypes.byref(cr), env._stream())
    assert rc == 0, lib.mgb_last_error().decode()


NULL = [("mlp", Shape("mlp", (17, 64)), False, None), ("mlp", Shape("mlp", (5,), act=nn.ReLU), True, (0.97, 0.9)),
        ("gru", Shape("gru", H=17, width=5), False, (0.9, 0.5)), ("gru", Shape("gru", H=8, reset="task"), True, None),
        ("lstm", Shape("lstm", H=17, width=0), True, None),
        ("lstm", Shape("lstm", H=8, width=13, reset="task"), True, (1.0, 1.0)),
        ("quad", None, False, None), ("quad", None, False, (0.97, 0.9))]


@pytest.mark.parametrize("kind,shape,rs,gae", NULL, ids=["%s-%r-rs%d-gae%d" % (k, s, r, g is not None)
                                                          for k, s, r, g in NULL])
def test_critic_null_outputs(tasks, kind, shape, rs, gae):  # noqa: F811
    n, T = 200, 24
    if kind == "quad":
        env, twin = quad_pair(n, "velocity_control")
        _, pol = quad_t.make_policy(env, (64, 17), nn.Tanh, 0, LOG_STD)
    else:
        env, twin = maze_pair(n, shape, rs, True, True, tasks)
        _, pol = shape.policy(env, seed=3)
    twin.close()
    critic = with_value(pol, 4)
    keys = ENV_OPTIONAL + (() if kind in ("mlp", "quad") else ("state0", "hid")) + ("value_last",)
    keys += ("final_value",) if gae is None else ()
    always = ALWAYS + (("final_value", "adv", "ret") if gae is not None else ())
    state0 = None if kind in ("mlp", "quad") else gru_t.random_state(pol, n)
    seen = []

    def alloc(ks):
        if kind == "quad":
            out = quad_outputs(env, T, [k for k in list(ks) + list(ALWAYS[:3]) if k in ENV_OPTIONAL + ALWAYS[:3]])
        else:
            out = maze_outputs(env, kind, pol, T, [k for k in list(ks) + list(ALWAYS[:3])
                                                   if k not in ("value_last", "final_value")])
        for k in ("value", "value_last", "final_value", "adv", "ret"):
            if k in ks or k in always:
                out[k] = sentinel((n,) if k == "value_last" else (T, n), torch.float32, env.device)
        return out

    def run(out, st):
        critic_call(env, kind, critic, T, out, st, rs, gae)
        seen.append([out[k].clone() for k in always])

    assert_drops_change_nothing(env, keys, run, alloc, state0)
    for s in seen[1:]:
        for k, x, y in zip(always, seen[0], s):
            assert torch.equal(x, y), k
    env.close()


# ---------------------------------------------------------------------------------------------------------------
# 6. Batch tails and populations
# ---------------------------------------------------------------------------------------------------------------

TAIL_SHAPES = {"mlp": Shape("mlp", (17, 64)), "gru": Shape("gru", H=17, width=5, reset="task"),
               "lstm": Shape("lstm", H=8, width=0)}
TAILS = [(kind, n) for kind in ("mlp", "gru", "lstm") for n in (1, 31, 129, 161)]


@pytest.mark.parametrize("kind,n", TAILS, ids=["%s-n%d" % t for t in TAILS])
def test_maze_batch_tails(tasks, kind, n):  # noqa: F811
    shape = TAIL_SHAPES[kind]
    a, b = maze_pair(n, shape, True, False, True, tasks)
    maze_critic_case(a, b, shape, 40, True, (0.97, 0.9))
    for e in (a, b):
        e.close()


@pytest.mark.parametrize("n", [1, 65])
def test_quad_batch_tails(n):
    a, b = quad_pair(n, "velocity_control")
    quad_critic_case(a, b, 48, (0.97, 0.9))
    for e in (a, b):
        e.close()


POPS = [("gru", 32, 3), ("gru", 64, 3), ("gru", 32, 5), ("lstm", 32, 5), ("mlp", 32, 5)]


@pytest.mark.parametrize("kind,E,M", POPS, ids=["%s-E%d-M%d" % p for p in POPS])
def test_population_twins(kind, E, M):
    """Member m's block against a handle of its E envs alone, member for member.  E = 32 with M = 5: the first CTA
    stages four members, the last one member of four."""
    from metagym_b200 import PolicyPopulation
    shape = {"gru": Shape("gru", H=17, width=13), "lstm": Shape("lstm", H=8, width=5),
             "mlp": Shape("mlp", (33, 17))}[kind]
    n, T = E * M, 24
    big = maze_env(n, shape)
    pop = PolicyPopulation([with_value(shape.policy(big, seed=3 + 7 * m)[1], m) for m in range(M)])
    state = gru_t.random_state(pop, n) if kind != "mlp" else None
    st0 = None if state is None else state.clone()
    out = maze_roll(big, pop, T, state, True, (0.97, 0.9))
    nxt = maze_roll(big, pop, 2, state, True)
    for m in range(M):
        tw = maze_env(E, shape, base=m * E)
        ts = None if st0 is None else st0[m * E:(m + 1) * E].clone()
        ref = maze_roll(tw, pop.policies[m], T, ts, True, (0.97, 0.9))
        mine = pop.member_slice(out, m)
        where = cut_mask(pop.policies[m], ref) & ref["truncated"].bool()
        for key in ("value", "value_last", "adv", "ret", "act", "logp", "rew", "done", "truncated", "obs", "obs0"):
            assert torch.equal(mine[key], ref[key]), (m, key)
        if state is not None:
            assert torch.equal(mine["hid"], ref["hid"]), m
        assert torch.equal(mine["final_value"][where], ref["final_value"][where]), m
        rn = maze_roll(tw, pop.policies[m], 2, ts, True)
        assert torch.equal(pop.member_slice(nxt, m)["value"], rn["value"]), m
        if state is not None:
            assert torch.equal(pop.member_slice(state, m), ts)
        tw.close()
    big.close()


# ---------------------------------------------------------------------------------------------------------------
# 7. The footprint with a value row
# ---------------------------------------------------------------------------------------------------------------

def value_staged(n_in, widths):
    """mlp_staged with the value row: the output layer has five rows, padded to the group of 4 (8 rows)."""
    s, ins, outs = 0, [n_in] + list(widths), list(widths) + [5]
    for k, (i, o) in enumerate(zip(ins, outs)):
        g = 4 if k == len(outs) - 1 else 8
        rows = (o + g - 1) // g * g
        s = (s + rows * i + rows + 7) // 8 * 8
    return s


def critic_smem_bytes(kind, view_grid, H=0, widths=(), feedback=True, rs=False, maze_n=15):
    """smem_bytes with the value row in the staged output layer (one staged copy)."""
    n_in = (2 * view_grid + 1) ** 2 if kind == "mlp" else H
    return (smem_bytes(kind, view_grid, H, widths, feedback, rs, maze_n)
            + 4 * (value_staged(n_in, widths) - mlp_staged(n_in, widths)))


def largest_h_val(kind, view_grid, width, rs, maze_n=9, optin=OPTIN_H100):
    fits = [H for H in range(1, 65)
            if critic_smem_bytes(kind, view_grid, H, (width,) if width else (), True, rs, maze_n) <= optin]
    return max(fits) if fits else None


# DESIGN.md "Recurrent policies", the "largest H that fits" table with a value head (15 x 15 mazes with resampling)
VALUE_TABLE = {"lstm": [[64, 61, 47, 29, 8, None], [64, 58, 44, 25, 8, None], [64, 56, 36, 14, None, None],
                        [64, 53, 32, 8, None, None]],
               "gru": [[64, 64, 61, 40, 15, None], [64, 64, 57, 36, 10, None], [64, 64, 47, 24, None, None],
                       [64, 61, 43, 24, None, None]]}


def test_value_row_footprint_table():
    for kind, rows in VALUE_TABLE.items():
        for (w, rs), row in zip(((0, False), (0, True), (64, False), (64, True)), rows):
            assert [largest_h_val(kind, vg, w, rs, 15) for vg in range(1, 7)] == row, (kind, w, rs)


# (cell, view_grid, head width, resampling with 9 x 9 mazes, the largest H that fits with a value head); all but the
# GRU at view_grid 4 fit one unit more without the value row
CELL_BOUNDARY = [("gru", 3, 0, True, 59), ("gru", 3, 64, True, 45), ("gru", 4, 0, False, 40), ("lstm", 3, 0, False, 47),
                 ("lstm", 4, 64, False, 14), ("lstm", 3, 13, True, 45)]


def critic_buffers(T, n, dev):
    return {"value": torch.zeros((T, n), device=dev)}


def test_mlp_footprint_with_a_value_row(tasks):  # noqa: F811
    """(64, 64) at view_grid 4 with 31 x 31 mazes' sampler workspaces fits with 32 bytes to spare; its value row needs
    4 (64 + 1) floats more, less the 4 floats of padding to 8 the layer had, and the critic call is refused with the
    exact byte count and nothing touched."""
    from metagym_b200 import _lib
    n, T = 128, 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert optin == OPTIN_H100
    assert optin - smem_bytes("mlp", 4, widths=(64, 64), rs=True, maze_n=31) == 32
    want = critic_smem_bytes("mlp", 4, widths=(64, 64), rs=True, maze_n=31)
    assert want - smem_bytes("mlp", 4, widths=(64, 64), rs=True, maze_n=31) == 4 * (4 * 65 - 4)
    e = footprint_env(n, 4, True, 31, tasks)
    lib = e._lib
    _, plain = mlp_t.make_policy(e, (64, 64))
    critic = with_value(plain, 0)
    cfg, seed = e._sampler_cfg(seed=1, **CFG)
    bufs = critic_buffers(T, n, e.device)
    cr = _lib.Critic(_lib.ptr(bufs["value"]), None, None, None, None, 1.0, 1.0)

    def call():
        return lib.mgb_maze_rollout_critic(e._h, T, ctypes.byref(critic.struct()), 1, 0, SEED, ctypes.byref(cfg), seed,
                                           None, None, None, None, None, None, None, None, ctypes.byref(cr),
                                           e._stream())
    assert_boundary(lib, e, call, want, optin)
    assert float(bufs["value"].abs().sum()) == 0
    with pytest.raises(_lib.MgbError):
        e.rollout(T, policy=critic, resample=dict(seed=1, **CFG))
    e.close()


@pytest.mark.parametrize("kind,vg,w,rs,H", CELL_BOUNDARY, ids=["%s-g%d-w%d-rs%d-H%d" % c for c in CELL_BOUNDARY])
def test_cell_footprint_with_a_value_row(tasks, kind, vg, w, rs, H):  # noqa: F811
    """The largest H that fits with a value head runs, H + 1 is refused with the exact byte count and nothing touched."""
    from metagym_b200 import _lib
    n, T = 128, 4
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert largest_h_val(kind, vg, w, rs, 9, optin) == H
    assert largest_h(kind, vg, w, rs, 9, optin) == H + ((kind, vg, w) != ("gru", 4, 0))
    make = gru_t.make_policy if kind == "gru" else lstm_t.make_policy
    for h in (H, H + 1):
        e = footprint_env(n, vg, rs, 9, tasks)
        lib = e._lib
        critic = with_value(make(e, h, w), 0)
        st = gru_t.random_state(critic, n)
        cfg, seed = e._sampler_cfg(seed=1, **CFG) if rs else (None, 0)
        want = critic_smem_bytes(kind, vg, h, (w,) if w else (), True, rs, 9)
        bufs = critic_buffers(T, n, e.device)
        cr = _lib.Critic(_lib.ptr(bufs["value"]), None, None, None, None, 1.0, 1.0)

        def call():
            return lib.mgb_maze_rollout_rnn_critic(e._h, T, ctypes.byref(critic.struct()), 1, 0, SEED,
                                                   ctypes.byref(cfg) if rs else None, seed, _lib.ptr(st), None, None,
                                                   None, None, None, None, None, None, None, None, ctypes.byref(cr),
                                                   e._stream())
        assert_boundary(lib, e, call, want, optin, st)
        if want > optin:
            assert float(bufs["value"].abs().sum()) == 0
            with pytest.raises(_lib.MgbError):
                e.rollout(T, policy=critic, state=st, resample=dict(seed=1, **CFG) if rs else None)
        else:
            assert bool(torch.isfinite(bufs["value"]).all()) and float(bufs["value"].abs().sum()) > 0
        e.close()
