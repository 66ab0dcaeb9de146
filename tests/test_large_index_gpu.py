"""The quadrotor and MetaMaze kernels at output sizes past 32-bit offsets (byte 2^31, byte 2^32, element index 2^31),
env for env against small twin handles.

Every test (1) skips unless 1.25 x the bytes its shapes need are free, (2) runs one big handle into output buffers that
are prefix views of allocations with a 4 KB tail, (3) compares the envs of the rows that hold or abut each crossed
boundary (tests/util.py straddle_rows), the edge envs and seeded random envs bit for bit with 3-env twins built with
env_index_base = e - 1 -- the default env2task and every Philox stream are keyed by the global env index, so env e of the
twin is env e of the big handle -- and follows a few of them with the CPU oracle, and (4) runs the big handle twice,
from fresh handles, into buffers filled with 0x00 and then 0xFF: per-256 MB digests of every byte the kernels must
write agree between the two runs, and every byte they must leave alone (final_obs rows of envs that did not finish,
the tails) still holds its fill.  A wrapped offset writes some rows twice and leaves others unwritten, which (4)
catches wherever it falls.  The shapes and the boundaries they cross are checked on the CPU by
tests/test_large_index_layout.py."""
import functools
import gc
import time
import traceback

import numpy as np
import pytest

from util import LARGE_SHAPES, QUAD_BENCH_N, QUAD_BIG_N, PATH_N, crossings, straddle_rows, twin_bases

pytestmark = pytest.mark.gpu

TAIL = 4096
CHUNK = 1 << 28                                  # digest chunk: 256 MB
GB = 1e9


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture
def big(torch_mod, request):
    """Releases every allocation of the test when it ends and prints its wall time and peak allocation."""
    torch = torch_mod
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    gc.collect()
    torch.cuda.synchronize()
    # torch's peak: the buffers the library allocates for a handle (state planes, path record) are not in it
    print("\n[large-index] %s: %.1f s, peak %.2f GB allocated by torch" % (request.node.name, time.time() - t0,
                                                                           torch.cuda.max_memory_allocated() / GB))
    torch.cuda.empty_cache()


def releases_on_failure(test):
    """A failing test's traceback keeps its frames alive, and with them its big handles and multi-GB buffers, so that
    every later test would skip for lack of memory: clear the frames' locals before the failure propagates (the `big`
    fixture then collects them and empties the cache)."""
    @functools.wraps(test)
    def run(*args, **kw):
        try:
            return test(*args, **kw)
        except BaseException as ex:
            traceback.clear_frames(ex.__traceback__)
            raise
    return run


def shape_of(name):
    """The (T, n, row_bytes, elem_bytes) layouts of a LARGE_SHAPES entry, each checked to cross what it claims."""
    out = []
    for o, T, n, rb, eb, claim in LARGE_SHAPES[name]:
        assert claim <= crossings(T, n, rb, eb), (name, o)
        out.append((T, n, rb, eb))
    return out


def require(torch, need):
    free = torch.cuda.mem_get_info()[0]
    if free < 1.25 * need:
        pytest.skip("needs 1.25 x %.2f GB free, %.2f / %.2f GB free" % (need / GB, free / GB, need / GB))


class Guarded(object):
    """An output buffer `t` that is a prefix view of an allocation with a TAIL-byte tail no kernel may write."""

    def __init__(self, torch, shape, dtype):
        self.nbytes = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        self.raw = torch.empty(self.nbytes + TAIL, dtype=torch.uint8, device="cuda")
        self.t = self.raw[:self.nbytes].view(dtype).view(shape)

    def fill(self, v):
        self.raw.fill_(v)

    def tail_holds(self, v):
        return bool((self.raw[self.nbytes:] == v).all())


def weights(torch):
    g = torch.Generator(device="cuda")
    g.manual_seed(0x1A26E)
    return torch.randint(-(1 << 62), 1 << 62, (CHUNK // 8,), generator=g, dtype=torch.int64, device="cuda")


def digest(torch, t, w):
    """[chunks, 2] int64: per CHUNK bytes of t, the wrapping sums of its int64 words and of the words times w."""
    b = t.reshape(-1).view(torch.uint8)
    n8 = b.numel() // 8 * 8
    words = b[:n8].view(torch.int64)
    parts = []
    for i in range(0, words.numel(), CHUNK // 8):
        x = words[i:i + CHUNK // 8]
        parts.append(torch.stack([x.sum(), (x * w[:x.numel()]).sum()]))
    if n8 < b.numel():
        x = b[n8:].to(torch.int64)
        parts.append(torch.stack([x.sum(), (x * w[:x.numel()]).sum()]))
    return torch.stack(parts).cpu()


def settle_final(torch, final, done, fill):
    """Rows of final_obs whose done is 0 must still hold `fill`: returns how many do not, and zeroes those rows so that
    the digest of final_obs covers only rows the kernel wrote.  Also returns the number of done rows."""
    d = done.reshape(-1).bool()
    rows = final.reshape(d.numel(), -1).view(torch.uint8)
    step = max(1, CHUNK // rows.shape[1])
    bad = torch.zeros((), dtype=torch.int64, device="cuda")
    for i in range(0, d.numel(), step):
        r, nd = rows[i:i + step], ~d[i:i + step]
        bad += ((r != fill).any(1) & nd).sum()
        r[nd] = 0
    return int(bad), int(d.sum())


def coverage_run(torch, run, w):
    """run(fill) -> (dict name -> Guarded or handle-owned tensor written in full, final Guarded or None, done tensor,
    list of Guarded).  Runs it with fill 0x00 and 0xFF and checks the two-fill contract; returns the second run's
    result (its buffers hold the outputs)."""
    dig = []
    for fill in (0x00, 0xFF):
        full, final, done, guarded, res = run(fill)
        torch.cuda.synchronize()
        for g in guarded:
            assert g.tail_holds(fill), "a kernel wrote past the end of an output"
        d = {k: digest(torch, v, w) for k, v in full.items()}
        if final is not None:
            bad, n_done = settle_final(torch, final, done, fill)
            assert bad == 0, "%d final_obs rows of envs that did not finish were written" % bad
            d["final_obs"] = digest(torch, final, w)
            d["n_done"] = n_done
        dig.append(d)
        if fill == 0x00:
            del full, final, done, guarded, res
            gc.collect()
            torch.cuda.empty_cache()
    for k in dig[0]:
        same = dig[0][k] == dig[1][k] if k == "n_done" else torch.equal(dig[0][k], dig[1][k])
        assert same, "%s: bytes the kernel must write differ between a 0x00-filled and a 0xFF-filled run" % k
    return res


def sampled(T, n, layouts):
    """Envs of the straddling rows of every output layout (T, n, row_bytes, elem_bytes), with the boundary rows."""
    envs, held = set(), {}
    for (TT, nn, rb, eb) in layouts:
        rows, h = straddle_rows(TT, nn, rb, eb)
        envs.update(e for _, e in rows if e < n)
        held.update({k: v for k, v in h.items() if v[1] < n})
    return sorted(envs), held


def free(*objs):
    for o in objs:
        if hasattr(o, "close"):
            o.close()
    gc.collect()


# ---------------------------------------------------------------------------------------------------------------------
# quadrotor
# ---------------------------------------------------------------------------------------------------------------------
QKW = dict(task="velocity_control", dt=0.005, seed=[0, 1, 2, 3, 4], rng_seed=0x5EED1234ABC, squeeze=False,
           auto_reset=True)


def quad_act(torch, n, t):
    g = torch.Generator(device="cuda")
    g.manual_seed(1000 + t)
    return torch.rand((n, 4), generator=g, device="cuda", dtype=torch.float32) * 14.9 + 0.1


def close_obs(a, ref, floor=0.1):
    """smoke()'s metric: component-wise |a - ref| / max(|ref|, floor)."""
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    return float((np.abs(a - ref) / np.maximum(np.abs(ref), floor)).max()) if a.size else 0.0


def quad_oracle(env, base, nt):
    from oracle import quad_oracle as qo
    return qo.OracleBatch(3, "velocity_control", QKW["dt"], nt, rng_seed=QKW["rng_seed"], env_index_base=base,
                          auto_reset=True, targets=env.velocity_targets.cpu().numpy(),
                          env2task=env.env2task.cpu().numpy())


@pytest.mark.parametrize("n", [QUAD_BIG_N, QUAD_BENCH_N], ids=["2^25+37", "bench_streaming"])
@releases_on_failure
def test_quad_step_stream_large(torch_mod, big, n):
    """quad_stream_kernel<true> at 2^25 + 37 envs (obs and final_obs 2.55 GB, past byte 2^31; state planes 3.2 GB) and
    at the 4 194 304 envs bench.py times: three steps with nt = 3, so every env finishes and auto-resets on the last."""
    torch = torch_mod
    from metagym_b200 import BatchedQuadrotor
    from util import B31
    nt, steps, D = 3, 3, 19
    name = "quad_step_stream" if n == QUAD_BIG_N else "quad_step_bench"
    lay = shape_of(name)
    assert lay[0] == (None, n, D * 4, 4)
    if n == QUAD_BIG_N:
        assert LARGE_SHAPES[name][0][5] == {B31}
    n_pad = (n + 127) // 128 * 128
    require(torch, 96 * n_pad + n * (2 * D * 4 + 16 + 4 + 1 + 4 + 1) + 2 * TAIL + 1.0 * GB)
    w = weights(torch)
    envs, held = sampled(None, n, lay)
    bases = twin_bases(envs, n)
    acts = {}

    def run(fill):
        env = BatchedQuadrotor(num_envs=n, nt=nt, final_obs=True, **QKW)
        assert env.step_kernel_name() == "quad_stream_kernel<true>"
        env._obs = env._final_obs = None                  # the handle's own [n, D] buffers, replaced by guarded ones
        gc.collect()
        torch.cuda.empty_cache()
        obs, final = Guarded(torch, (n, D), torch.float32), Guarded(torch, (n, D), torch.float32)
        rew, done = Guarded(torch, (n,), torch.float32), Guarded(torch, (n,), torch.uint8)
        env._obs, env._final_obs = obs.t, final.t          # reset() writes _obs; step() reads _final_obs each call
        env.reset()
        for g in (obs, final, rew, done):
            g.fill(fill)
        env._fail.view(torch.uint8).fill_(fill)
        env._trunc.fill_(fill)
        for t in range(steps):
            a = quad_act(torch, n, t)
            if fill == 0x00:
                for b in bases:
                    acts.setdefault(b, []).append(a[b:b + 3].clone())
            env.step(a, out=(obs.t, rew.t, done.t))
            del a
        full = {"obs": obs.t, "rew": rew.t, "done": done.t, "fail": env._fail, "truncated": env._trunc}
        return full, final.t, done.t, [obs, final, rew, done], (env, obs, final, rew, done)

    env, obs, final, rew, done = coverage_run(torch, run, w)
    assert bool(done.t.bool().all())                       # ct == nt for every env: every row of final_obs was written
    got = {b: dict(obs=obs.t[b:b + 3].cpu(), rew=rew.t[b:b + 3].cpu(), done=done.t[b:b + 3].cpu(),
                   fail=env._fail[b:b + 3].cpu(), trunc=env._trunc[b:b + 3].cpu(), final=final.t[b:b + 3].cpu())
           for b in bases}
    del obs, final, rew, done
    env._obs = env._final_obs = None
    gc.collect()
    sd = env.state_dict()
    for b in bases:
        got[b]["state"], got[b]["ct"] = sd["state"][b:b + 3].cpu(), sd["ct"][b:b + 3].cpu()
    del sd
    free(env)
    for i, b in enumerate(bases):
        tw = BatchedQuadrotor(num_envs=3, nt=nt, final_obs=True, env_index_base=b, **QKW)
        tw.reset()
        for t in range(steps):
            o, r, d, _ = tw.step(acts[b][t])
        g, tsd = got[b], tw.state_dict()
        assert torch.equal(g["obs"], o.cpu()) and torch.equal(g["rew"], r.cpu()), b
        assert torch.equal(g["done"], d.cpu().to(torch.uint8)) and torch.equal(g["fail"], tw.fail_code.cpu()), b
        assert torch.equal(g["trunc"], tw.truncated.cpu().to(torch.uint8)), b
        assert torch.equal(g["final"], tw.final_observation.cpu()), b
        assert torch.equal(g["state"], tsd["state"].cpu()) and torch.equal(g["ct"], tsd["ct"].cpu()), b
        if i < 8:                                          # the independent CPU oracle for a few of them
            ob = quad_oracle(tw, b, nt)
            ob.reset()
            for t in range(steps):
                res = ob.step(acts[b][t].cpu().numpy())
            assert np.array_equal(res.done, g["done"].numpy().astype(bool)), b
            assert close_obs(g["obs"].numpy(), res.obs) < 1e-5, b
            assert close_obs(g["final"].numpy()[res.done], res.final_obs[res.done]) < 1e-5, b
        free(tw)
    print("[large-index] quad step n=%d: twins at %s, boundary rows %s" % (n, bases, held))


@pytest.mark.parametrize("T,nt,final", [(28, 10, False), (14, 5, True)], ids=["T28_actions", "T14_final_obs"])
@releases_on_failure
def test_quad_rollout_large(torch_mod, big, T, nt, final):
    """quad_rollout_kernel<., 0, false> at T = 28 x 4 194 304 envs (obs 8.9 GB, element index 2.23e9 past 2^31) with
    device-drawn actions recorded; quad_rollout_kernel<., 0, true> at T = 14 (obs and final_obs 4.5 GB each, past byte
    2^32).  Auto-reset every nt steps."""
    torch = torch_mod
    from metagym_b200 import BatchedQuadrotor
    n, D, seed = QUAD_BENCH_N, 19, 0xACE5
    name = "quad_rollout_final" if final else "quad_rollout"
    lay = shape_of(name)
    assert all(l[:2] == (T, n) for l in lay)              # the shapes this test runs are the ones the CPU test checks
    n_pad = (n + 127) // 128 * 128
    per = D * 4 * (2 if final else 1) + 4 + 1 + (1 if final else 16)
    require(torch, 96 * n_pad + 2 * n * D * 4 + T * n * per + 5 * TAIL + 1.0 * GB)
    w = weights(torch)
    envs, held = sampled(T, n, lay)
    bases = twin_bases(envs, n)

    def run(fill):
        env = BatchedQuadrotor(num_envs=n, nt=nt, final_obs=final, **QKW)
        env.reset()
        out = {"obs": Guarded(torch, (T, n, D), torch.float32), "rew": Guarded(torch, (T, n), torch.float32),
               "done": Guarded(torch, (T, n), torch.uint8)}
        if final:
            out["final_obs"] = Guarded(torch, (T, n, D), torch.float32)
            out["truncated"] = Guarded(torch, (T, n), torch.uint8)
        else:
            out["act"] = Guarded(torch, (T, n, 4), torch.float32)
        for g in out.values():
            g.fill(fill)
        env.rollout(T, act_seed=seed, want_actions=not final, out={k: g.t for k, g in out.items()})
        full = {k: g.t for k, g in out.items() if k != "final_obs"}
        return full, out["final_obs"].t if final else None, out["done"].t, list(out.values()), (env, out)

    env, out = coverage_run(torch, run, w)
    done = out["done"].t
    if final:
        assert bool(done.any()) and not bool(done.all())
    got = {b: {k: g.t[:, b:b + 3].cpu() for k, g in out.items()} for b in bases}
    del out, done
    gc.collect()
    sd = env.state_dict()
    for b in bases:
        got[b]["state"], got[b]["ct"] = sd["state"][b:b + 3].cpu(), sd["ct"][b:b + 3].cpu()
    del sd
    free(env)
    for i, b in enumerate(bases):
        tw = BatchedQuadrotor(num_envs=3, nt=nt, final_obs=final, env_index_base=b, **QKW)
        tw.reset()
        r = tw.rollout(T, act_seed=seed, want_actions=True)
        g, tsd = got[b], tw.state_dict()
        for k in g:
            if k in ("state", "ct"):
                assert torch.equal(g[k], tsd[k].cpu()), (b, k)
            elif k == "final_obs":
                m = g["done"].bool()
                assert torch.equal(g[k][m], r[k].cpu()[m]), b
            else:
                assert torch.equal(g[k], r[k].cpu()), (b, k)
        if i < 8:
            ob = quad_oracle(tw, b, nt)
            ob.reset()
            acts = r["act"].cpu().numpy()
            for t in range(T):
                res = ob.step(acts[t])
                assert np.array_equal(res.done, g["done"][t].numpy().astype(bool)), (b, t)
                assert close_obs(g["obs"][t].numpy(), res.obs) < 1e-5, (b, t)
                if final:
                    assert close_obs(g["final_obs"][t].numpy()[res.done], res.final_obs[res.done]) < 1e-5, (b, t)
        free(tw)
    print("[large-index] quad rollout T=%d: twins at %s, boundary rows %s" % (T, bases, held))


# ---------------------------------------------------------------------------------------------------------------------
# MetaMaze
# ---------------------------------------------------------------------------------------------------------------------
def maze_tasks(n_cells, k, seed, task_type="SURVIVAL", dying=0):
    """k sampled tasks; the first `dying` lose 0.5 life per step from 0.5, so their envs die on step 2 with life -0.5."""
    from metagym_b200 import MazeTaskSampler
    rs = np.random.RandomState(seed)
    out = []
    for j in range(k):
        t = MazeTaskSampler(n=n_cells, food_density=0.02, food_interval=5, rng=rs)
        if j < dying:
            t = t._replace(step_reward=-0.5, initial_life=0.5)
        elif task_type == "SURVIVAL":
            t = t._replace(initial_life=2.0, max_life=2.0)
        out.append(t)
    return out


def maze_env(kind, n, base=0, **kw):
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D
    from metagym_b200.textures import synthetic_textures
    if kind == "2D":
        return BatchedMetaMaze2D(num_envs=n, env_index_base=base, squeeze=False, **kw)
    cls = BatchedMetaMazeContinuous3D if kind == "C3D" else BatchedMetaMazeDiscrete3D
    return cls(num_envs=n, env_index_base=base, squeeze=False, resolution=(128, 128), textures=synthetic_textures(seed=0),
               **kw)


def maze_state(env):
    out = [t.cpu() for t in env.agent_state()]
    if env.KIND == 2:
        out += [t.cpu() for t in env.pose()]
    return out


def oracle_frame(dtype, v):
    if dtype == "uint8":
        return np.minimum(v, 255).astype(np.uint8)
    return v.astype(np.float32) if dtype == "float32" else v


def maze_oracle_follow(kind, kw, task, acts, n_steps, dtype=None, got=None, ts=None):
    """OracleMaze through n_steps steps of one env with the actions acts[t].  got: the engine's outputs of the env,
    indexable by t (obs, rew, done, optionally final_obs), compared bit for bit at the steps ts (default: all).  With
    kw["auto_reset"] a finished episode restarts; without it the follow ends at the first done.  Returns the cells of the
    current episode's path (start cell first)."""
    from metagym_b200.textures import synthetic_textures
    from oracle.maze_oracle import OracleMaze
    okw = dict(view_grid=kw["view_grid"]) if kind == "2D" else dict(resolution=(128, 128),
                                                                     textures=synthetic_textures(seed=0))
    o = OracleMaze(kind, kw["task_type"], kw["max_steps"], **okw)
    o.set_task(task)
    o.reset()
    path = [tuple(o.agent[:2])]
    ts = set(range(n_steps) if ts is None else ts)
    for t in range(n_steps):
        v, r, d, _ = o.step(acts[t])
        path.append(tuple(o.agent[:2]))
        check = got is not None and t in ts
        if check:
            assert float(got["rew"][t]) == r and bool(got["done"][t]) == d, t
        if d:
            if check and "final_obs" in got:
                assert np.array_equal(got["final_obs"][t], oracle_frame(dtype, v)), t
            if not kw["auto_reset"]:
                return path
            v = o.reset()
            path = [tuple(o.agent[:2])]
        if check:
            assert np.array_equal(got["obs"][t], oracle_frame(dtype, v)), t
    return path


def followed(held):
    """Env 0 and the env of every boundary row, in boundary order: the envs the CPU oracle follows."""
    out = [0]
    for k in sorted(held):
        if held[k][1] not in out:
            out.append(held[k][1])
    return out


MAZE_ROLLOUTS = {
    # name: kind, T, n, obs dtype, final_obs, actions given (else device-drawn and recorded), handle kwargs
    "maze2d_rollout": ("2D", 280, 65536, "float32", False, True, dict(view_grid=5, max_steps=60, task_type="SURVIVAL")),
    "maze3d_rollout_u8": ("3D", 12, 8192, "uint8", True, True, dict(obs_dtype="uint8", max_steps=9, task_type="SURVIVAL")),
    "maze3d_rollout_i32": ("3D", 6, 8192, "int32", False, True, dict(obs_dtype="int32", max_steps=4, task_type="SURVIVAL")),
    "mazec3d_rollout_u8": ("C3D", 12, 8192, "uint8", False, False,
                           dict(obs_dtype="uint8", max_steps=7, task_type="SURVIVAL")),
}


@pytest.mark.parametrize("name", sorted(MAZE_ROLLOUTS))
@releases_on_failure
def test_maze_rollout_large(torch_mod, big, name):
    """2-D rollout (view_grid 5, 65 536 envs x 280 steps: obs 8.9 GB, element index past 2^31), discrete 3-D rollouts on
    the pose cache (128 x 128 uint8 x 12 steps with final_obs: 4.8 GB each, past byte 2^32; int32 x 6 steps: 9.7 GB,
    element index past 2^31) and the continuous 3-D rollout of the direct renderer with device-drawn actions (4.8 GB)."""
    torch = torch_mod
    kind, T, n, dtype, final, given, kw = MAZE_ROLLOUTS[name]
    kw = dict(kw, auto_reset=True)
    if kind == "2D":
        row = (2 * kw["view_grid"] + 1) ** 2 * 4
        shape, tdt = (2 * kw["view_grid"] + 1,) * 2, torch.float32
    else:
        px = {"uint8": 1, "int32": 4, "float32": 4}[dtype]
        row, shape = 128 * 128 * 3 * px, (128, 128, 3)
        tdt = {"uint8": torch.uint8, "int32": torch.int32}[dtype]
    lay = shape_of(name)
    assert all(l[:3] == (T, n, row) for l in lay)
    act_row = 8 if kind == "C3D" else 4
    require(torch, T * n * (row * (2 if final else 1) + 8 + 1 + act_row + (1 if final else 0)) + n * row + 1.5 * GB)
    w = weights(torch)
    tasks = maze_tasks(9 if kind != "2D" else 11, 6, seed=7)
    acts = None
    if given:
        g = torch.Generator(device="cuda")
        g.manual_seed(11)
        acts = torch.randint(0, 4, (T, n), generator=g, device="cuda", dtype=torch.int32)
    envs, held = sampled(T, n, lay)
    bases = twin_bases(envs, n)
    fkw = dict(final_obs=final) if kind != "2D" else {}

    def run(fill):
        env = maze_env(kind, n, **kw)
        env.set_task(tasks)
        env.reset()
        out = {"obs": Guarded(torch, (T, n) + shape, tdt), "rew": Guarded(torch, (T, n), torch.float64),
               "done": Guarded(torch, (T, n), torch.uint8)}
        if final:
            out["final_obs"] = Guarded(torch, (T, n) + shape, tdt)
            out["truncated"] = Guarded(torch, (T, n), torch.uint8)
        if not given:
            out["act"] = Guarded(torch, (T, n, 2) if kind == "C3D" else (T, n), torch.float32 if kind == "C3D" else torch.int32)
        for gd in out.values():
            gd.fill(fill)
        env.rollout(T, actions=acts, act_seed=0xD1CE, want_actions=not given, out={k: gd.t for k, gd in out.items()},
                    **fkw)
        full = {k: gd.t for k, gd in out.items() if k != "final_obs"}
        return full, out["final_obs"].t if final else None, out["done"].t, list(out.values()), (env, out)

    env, out = coverage_run(torch, run, w)
    if final:
        done = out["done"].t
        assert bool(done.any()) and not bool(done.all())
    if kind == "3D":          # the discrete rollout has one path, the pose-cache kernel: the host refuses it without the cache
        assert env.cache_info()["in_use"]
    got = {b: {k: gd.t[:, b:b + 3].cpu() for k, gd in out.items()} for b in bases}
    st = maze_state(env)
    del out
    free(env)
    for b in bases:
        tw = maze_env(kind, 3, base=b, **kw)
        tw.set_task(tasks)
        tw.reset()
        r = tw.rollout(T, actions=None if acts is None else acts[:, b:b + 3], act_seed=0xD1CE, want_actions=not given, **fkw)
        for k, v in got[b].items():
            if k == "final_obs":
                m = got[b]["done"].bool()
                assert torch.equal(v[m], r[k].cpu()[m]), b
            else:
                assert torch.equal(v, r[k].cpu()), (b, k)
        for x, y in zip(st, maze_state(tw)):
            assert torch.equal(x[b:b + 3], y), b
        free(tw)
    # the CPU oracle for env 0 and the envs of the rows that hold the boundaries
    follow = followed(held)
    for e in follow:
        b = [x for x in bases if x <= e < x + 3][0]
        gotn = {k: v[:, e - b].numpy() for k, v in got[b].items()}
        a = (acts[:, e].cpu().numpy() if given else gotn["act"])
        maze_oracle_follow(kind, kw, tasks[e % len(tasks)], a, T, dtype, gotn)
    print("[large-index] %s: twins at %s, oracle envs %s, boundary rows %s" % (name, bases, follow, held))


@releases_on_failure
def test_maze3d_step_fused_large(torch_mod, big):
    """The fused single-step kernel (maze3d_step_kernel, pose cache, uint8 128 x 128) at 90 000 envs of 8 SURVIVAL tasks
    with auto-reset and final_obs: obs and final_obs 4.4 GB each, past byte 2^32.  The envs of tasks 0..3 die on the
    second step, so final_obs holds written and unwritten rows side by side."""
    torch = torch_mod
    lay = shape_of("maze3d_step_u8")
    (_, n, row, _), steps = lay[0], 2
    assert all(l == (None, n, 128 * 128 * 3, 1) for l in lay)
    kw = dict(obs_dtype="uint8", max_steps=50, task_type="SURVIVAL", auto_reset=True, final_obs=True)
    require(torch, 2 * n * row + 2 * TAIL + 1.5 * GB)
    w = weights(torch)
    tasks = maze_tasks(9, 8, seed=5, dying=4)
    envs, held = sampled(None, n, lay)
    bases = twin_bases(envs, n)
    acts = []
    for t in range(steps):
        g = torch.Generator(device="cuda")
        g.manual_seed(40 + t)
        acts.append(torch.randint(0, 4, (n,), generator=g, device="cuda", dtype=torch.int32))

    def run(fill):
        env = maze_env("3D", n, **kw)
        env._obs = env._final = None                      # the handle's own [n, 128, 128, 3] buffers, replaced below
        gc.collect()
        torch.cuda.empty_cache()
        obs, final = Guarded(torch, (n, 128, 128, 3), torch.uint8), Guarded(torch, (n, 128, 128, 3), torch.uint8)
        env._obs, env._final = obs.t, final.t             # step() takes the addresses of _obs and _final
        env.set_task(tasks)
        env.reset()
        for gd in (obs, final):
            gd.fill(fill)
        env._rew.view(torch.uint8).fill_(fill)
        env._done.fill_(fill)
        env._trunc.fill_(fill)
        l0 = env.launch_count
        for t in range(steps):
            env.step(acts[t])
        # one launch per step is the fused kernel; the logic + compose pair with final_obs takes four (list reset, logic,
        # compose, list pass), so a step that left the fused path fails here
        assert env.launch_count - l0 == steps
        full = {"obs": obs.t, "rew": env._rew, "done": env._done, "truncated": env._trunc}
        return full, final.t, env._done, [obs, final], (env, obs, final)

    env, obs, final = coverage_run(torch, run, w)
    assert env.cache_info()["in_use"]
    done = env._done
    assert bool(done.any()) and not bool(done.all())
    got = {b: dict(obs=obs.t[b:b + 3].cpu(), final=final.t[b:b + 3].cpu(), rew=env._rew[b:b + 3].cpu(),
                   done=done[b:b + 3].cpu(), trunc=env._trunc[b:b + 3].cpu()) for b in bases}
    st = maze_state(env)
    del obs, final
    free(env)
    for b in bases:
        tw = maze_env("3D", 3, base=b, **kw)
        tw.set_task(tasks)
        tw.reset()
        for t in range(steps):
            o, r, d, _ = tw.step(acts[t][b:b + 3])
        gb = got[b]
        m = gb["done"].bool()
        assert torch.equal(gb["obs"], o.cpu()) and torch.equal(gb["rew"], r.cpu()), b
        assert torch.equal(gb["done"], d.cpu().to(torch.uint8)), b
        assert torch.equal(gb["trunc"], tw.truncated.cpu().to(torch.uint8)), b
        assert torch.equal(gb["final"][m], tw.final_observation.cpu()[m]), b
        for x, y in zip(st, maze_state(tw)):
            assert torch.equal(x[b:b + 3], y), b
        free(tw)
    follow = followed(held)
    for e in follow:                                      # the CPU oracle: the outputs of the last step
        b = [x for x in bases if x <= e < x + 3][0]
        gb = {k: {steps - 1: v[e - b].numpy()} for k, v in got[b].items()}
        gb["final_obs"] = gb.pop("final")
        maze_oracle_follow("3D", kw, tasks[e % len(tasks)], [int(a[e]) for a in acts], steps, "uint8", gb, [steps - 1])
    print("[large-index] maze3d fused step: twins at %s, oracle envs %s, boundary rows %s" % (bases, follow, held))


@releases_on_failure
def test_maze_god_view_large(torch_mod, big):
    """maze_god_view_kernel (live and trajectory) and maze_god_path_kernel: 6 300 views of 480 x 480 of a 6 300-env
    2-D ESCAPE handle after 30 drawn steps, 4.35 GB, past byte 2^32."""
    torch = torch_mod
    from oracle import maze_godview as gv
    import trajectory_view as tv
    lay = shape_of("god_view")
    (_, n, row, _), S, T = lay[0], 480, 30
    assert row == S * S * 3
    kw = dict(max_steps=200, task_type="ESCAPE", auto_reset=True, record_path=True, view_grid=2)
    require(torch, n * S * S * 3 + TAIL + 1.0 * GB)
    w = weights(torch)
    tasks = maze_tasks(11, 5, seed=9, task_type="ESCAPE")
    envs, held = sampled(None, n, lay)
    bases = twin_bases(envs, n)
    env = maze_env("2D", n, **kw)
    env.set_task(tasks)
    env.reset()
    env.rollout(T, act_seed=77, out={})
    views = Guarded(torch, (n, S, S, 3), torch.uint8)
    got = {}
    for traj in (False, True):
        def run(fill):
            views.fill(fill)
            env.god_view(view_size=S, out=views.t, trajectory=traj)
            return {"views": views.t}, None, None, [views], None
        coverage_run(torch, run, w)
        got[traj] = {b: views.t[b:b + 3].cpu() for b in bases}
    del views
    free(env)
    drawn = {}
    for b in bases:
        tw = maze_env("2D", 3, base=b, **kw)
        tw.set_task(tasks)
        tw.reset()
        drawn[b] = tw.rollout(T, act_seed=77, out={"act": torch.empty((T, 3), dtype=torch.int32, device="cuda")})["act"]
        drawn[b] = drawn[b].cpu().numpy()
        for traj in (False, True):
            assert torch.equal(got[traj][b], tw.god_view(view_size=S, trajectory=traj).cpu()), (b, traj)
        free(tw)
    follow = followed(held)
    for e in follow:                 # the CPU oracle: the agent's cells, then both pictures rasterised from primitives
        b = [x for x in bases if x <= e < x + 3][0]
        task = tasks[e % len(tasks)]
        path = maze_oracle_follow("2D", kw, task, drawn[b][:, e - b], T)
        live = gv.rasterise(gv.live_primitives(0, "ESCAPE", task.cell_walls, task.goal, S, grid=path[-1]), S)
        traj = tv.rasterise(tv.trajectory_primitives("ESCAPE", task.cell_walls, task.goal, S, path[-1], path), S)
        assert np.array_equal(got[False][b][e - b].numpy(), live), e
        assert np.array_equal(got[True][b][e - b].numpy(), traj), e
    print("[large-index] god view: twins at %s, oracle envs %s, boundary rows %s" % (bases, follow, held))


@releases_on_failure
def test_maze_path_record_large(torch_mod, big):
    """path_store into the [max_steps + 1][n_pad] char2 path record of 2 200 000 2-D envs (4.4 GB, element index past 2^31
    at step 976): 990 drawn ESCAPE steps without auto-reset on 31 x 31 mazes, then trajectory() of the sampled envs
    against their twins'.  The record is the handle's own buffer, so there is no two-fill run; the twins' paths are
    compared entry for entry through step 990."""
    torch = torch_mod
    n, T, cap = PATH_N, 990, 1001
    n_pad = (n + 127) // 128 * 128
    kw = dict(max_steps=cap - 1, task_type="ESCAPE", auto_reset=False, record_path=True, view_grid=1)
    require(torch, cap * n_pad * 2 + n * 64 + 1.0 * GB)
    lay = shape_of("path")
    assert lay == [(cap, n_pad, 2, 2)]
    rows, held = straddle_rows(*lay[0])
    envs = sorted({e for _, e in rows if e < n})
    assert all(t <= T for t, _ in held.values())         # every boundary entry is written by the rollout
    bases = twin_bases(envs, n)
    tasks = maze_tasks(31, 4, seed=13, task_type="ESCAPE")
    env = maze_env("2D", n, **kw)
    env.set_task(tasks)
    env.reset()
    env.rollout(T, act_seed=5, out={})
    idx = sorted({e for b in bases for e in range(b, b + 3)})
    cells, lens = env.trajectory(envs=idx)
    cells, lens = cells.cpu(), lens.cpu()
    assert bool((lens == T + 1).all())
    pos = {e: k for k, e in enumerate(idx)}
    free(env)
    drawn = {}
    for b in bases:
        tw = maze_env("2D", 3, base=b, **kw)
        tw.set_task(tasks)
        tw.reset()
        drawn[b] = tw.rollout(T, act_seed=5, out={"act": torch.empty((T, 3), dtype=torch.int32, device="cuda")})["act"]
        drawn[b] = drawn[b].cpu().numpy()
        c2, l2 = tw.trajectory()
        k = [pos[e] for e in range(b, b + 3)]
        assert torch.equal(cells[k], c2.cpu()) and torch.equal(lens[k], l2.cpu()), b
        free(tw)
    # the CPU oracle: the cells of env 0 and of the envs holding the boundary entries, through the first done (without
    # auto-reset an ESCAPE env that reached its goal needs a reset the record does not see)
    follow = followed({k: v for k, v in held.items() if v[1] < n})
    for e in follow:
        b = [x for x in bases if x <= e < x + 3][0]
        path = maze_oracle_follow("2D", kw, tasks[e % len(tasks)], drawn[b][:, e - b], T)
        assert np.array_equal(cells[pos[e], :len(path)].numpy(), np.asarray(path, np.int32)), e
    print("[large-index] path record: twins at %s, boundary entries %s" % (bases, held))
