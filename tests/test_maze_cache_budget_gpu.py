"""MetaMaze discrete-3D pose cache: the memory decisions of the cache at every level they can choose.

Three decisions are restated here in Python from what cache_info() reports, and every level is checked bit for bit
against a cache=False twin (and at some levels against the C oracle):
- pose_cache_fits: the strided table bytes against MGB_MAZE_CACHE_GB (over budget: the direct renderer);
- the host budget loop: the largest variant bits <= MGB_MAZE_VARIANT_BITS whose n_tasks x V variant frames fit the room
  the budget leaves after the base bytes, V = the most frames one task of the table needs at those bits;
- maze3d_plan_kernel: each task takes the largest bits <= the table's whose frames fit its V frames, so a task that
  update_tasks swaps in and that needs more than V frames takes fewer bits than its neighbours."""
import math

import numpy as np
import pytest

from util import MazeTask

pytestmark = pytest.mark.gpu

N_CELLS = 9
RES = (64, 64)
PX3 = RES[0] * RES[1] * 3
MAX_STEPS = 25
BITS_MAX = 7


def maze_task(foods, walls=None, start=(1, 1), goal=(7, 7), initial_life=0.15):
    """A 9x9 SURVIVAL task: `walls` (default: an open 7x7 room inside the border), food of 0.5 on the cells `foods`, each
    back 6 steps after it is eaten.  initial_life 0.15 at -0.01 a step: an env that eats nothing dies at step 15, before
    the step limit, so episodes end both ways."""
    n = N_CELLS
    if walls is None:
        walls = np.ones((n, n), np.int32)
        walls[1:-1, 1:-1] = 0
    walls = np.asarray(walls, np.int32)
    ij = np.add.outer(np.arange(n), np.arange(n))
    texts = np.where(walls == 1, 1 + ij % 6, 0).astype(np.int64)
    food = np.zeros((n, n))
    itv = np.zeros((n, n), np.int32)
    for (i, j) in foods:
        assert walls[i, j] == 0 and (i, j) != tuple(start)
        food[i, j], itv[i, j] = 0.5, 6
    return MazeTask(start=tuple(start), goal=tuple(goal), cell_walls=walls, cell_texts=texts, cell_size=2.0,
                    wall_height=3.2, agent_height=1.6, initial_life=initial_life, max_life=2.0, step_reward=-0.01,
                    goal_reward=0.27, food_rewards=food, food_interval=itv)


def pockets_task(cells, foods):
    """Every cell a wall but the start (1, 1) and the one-cell pockets `cells` (odd coordinates, so walls part them):
    few poses, and so few variant frames however many foods the task has.  The goal is the last pocket."""
    walls = np.ones((N_CELLS, N_CELLS), np.int32)
    walls[1, 1] = 0
    for (i, j) in cells:
        walls[i, j] = 0
    return maze_task(foods, walls=walls, goal=cells[-1])


def wall_row_task(foods):
    """The open room parted by a wall along row 4 with a gap at its east end."""
    walls = np.ones((N_CELLS, N_CELLS), np.int32)
    walls[1:-1, 1:-1] = 0
    walls[4, 1:6] = 1
    return maze_task(foods, walls=walls)


# The ladder's table: poses that see 1 to 7 foods, and tasks whose frame needs stop growing at different bits
LADDER_TASKS = [
    lambda: maze_task([(2, 2), (2, 6), (6, 2), (6, 6), (4, 4), (3, 5), (5, 3)]),
    lambda: maze_task([(3, 3), (3, 5), (5, 5), (4, 2)]),
    lambda: wall_row_task([(2, 3), (2, 5), (6, 3), (6, 6), (5, 6)]),
    lambda: maze_task([(2, 4), (6, 4)]),
]
POCKETS = [(1, 3), (1, 5), (1, 7), (3, 1), (3, 3), (3, 5), (3, 7)]
# The mixed-bits table: tasks that need few frames (the pockets task carries the table's largest food count, so that the
# replacement is allowed), and a replacement in slot 0 that needs more than the table's V frames but no more than its
# n_tasks x V, so a plan that ignored V would write into the neighbours' frames, not past the table.
MIXED_TASKS = [
    lambda: maze_task([(4, 4)]),
    lambda: pockets_task(POCKETS, POCKETS),
    lambda: maze_task([(2, 6)]),
    lambda: maze_task([(6, 2)]),
]
REPLACEMENT = lambda: maze_task([(4, 2), (4, 3), (4, 4), (4, 5)])          # noqa: E731


@pytest.fixture(scope="module")
def torch_mod(cuda_device):
    import torch
    return torch


@pytest.fixture(scope="module")
def textures():
    from metagym_b200.textures import synthetic_textures
    return synthetic_textures(seed=0)


def free_cells(task):
    """Free cells as the pose cache counts them: every non-wall cell and the start cell."""
    walls = np.asarray(task.cell_walls) == 0
    walls[task.start[0], task.start[1]] = True
    return int(walls.sum())


def food_cells(task):
    return int((np.asarray(task.food_rewards) > 0).sum())


def clear_env(monkeypatch):
    for k in ("MGB_MAZE_CACHE", "MGB_MAZE_CACHE_GB", "MGB_MAZE_VARIANT_BITS", "MGB_MAZE_FUSED_STEP"):
        monkeypatch.delenv(k, raising=False)


def make_env(monkeypatch, textures, n, budget=None, fused=True, cache=None, obs_dtype="uint8", task_type="SURVIVAL"):
    """A 64x64 auto-reset handle with terminal frames; budget: the MGB_MAZE_CACHE_GB string (None: the default).  The
    library handle, which reads the variables, is created here for 9x9 tables (set_task keeps it)."""
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    clear_env(monkeypatch)
    if budget is not None:
        monkeypatch.setenv("MGB_MAZE_CACHE_GB", budget)
    monkeypatch.setenv("MGB_MAZE_FUSED_STEP", "1" if fused else "0")
    env = BatchedMetaMazeDiscrete3D(resolution=RES, max_steps=MAX_STEPS, task_type=task_type, num_envs=n, squeeze=False,
                                    auto_reset=True, final_obs=True, obs_dtype=obs_dtype, textures=textures, cache=cache)
    env._create(N_CELLS)
    clear_env(monkeypatch)
    return env


# ---------------------------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------------------------
def need_of(hist):
    """need[b] = sum over 1 <= k <= b of hist[k] (2^k - 1): the variant frames a task needs at b bits, b = 0..7."""
    return [sum(hist[k] * ((1 << k) - 1) for k in range(1, b + 1)) for b in range(BITS_MAX + 1)]


def base_bytes(tasks, obs_dtype="uint8", task_type="SURVIVAL"):
    """pose_cache_fits: n_tasks x S pose slots (S = 4 x the most free cells of a task), each with its packed pixels
    (uint8: c_px + c_rgb8; otherwise c_px + c_px_all), food ids, signature, pose row and crossing lists of max_hits
    = min(food cells, ceil(2 max_vision / min cell) + 3, 2n - 1) entries (ESCAPE: 2) of 16 bytes per column."""
    slots = len(tasks) * 4 * max(free_cells(t) for t in tasks)
    px = RES[0] * RES[1]
    geo = math.ceil(2 * 12.0 / min(t.cell_size for t in tasks)) + 3
    mh = 2 if task_type == "ESCAPE" else max(1, min(max(food_cells(t) for t in tasks), geo, 2 * N_CELLS - 1))
    return float(slots) * (px * (8.0 if obs_dtype == "uint8" else 12.0) + px / 4.0 + 16.0 + RES[0] * (1.0 + mh * 16.0))


def budget_plan(needs, base, budget, var_bits=BITS_MAX):
    """The host loop of ensure_pose_cache -> (bits, V): the largest bits <= var_bits whose n_tasks x V frames fit the room
    the budget (bytes, as the C side computes it) leaves after the base bytes, V = the most frames a task needs there."""
    room = budget - base
    bits, V = var_bits, 0
    while bits > 0:
        V = max(nd[bits] for nd in needs)
        if float(len(needs)) * V * PX3 <= room:
            break
        bits -= 1
    return bits, (V if bits > 0 else 0)


def task_plan(need, var_bits, V):
    """maze3d_plan_kernel for one task -> (bits, frames): the largest bits <= var_bits whose frames fit V."""
    bits = frames = 0
    if var_bits > 0 and V > 0:
        for b in range(1, BITS_MAX + 1):
            if b <= var_bits and need[b] <= V:
                bits, frames = b, need[b]
    return bits, frames


def budget_gb(x):
    """The MGB_MAZE_CACHE_GB string whose atof(...) * 1e9 is the smallest double >= x (within a byte of it), and that
    double."""
    g = x / 1e9
    while g * 1e9 < x:
        g = math.nextafter(g, math.inf)
    while math.nextafter(g, -math.inf) * 1e9 >= x:
        g = math.nextafter(g, -math.inf)
    assert float(repr(g)) == g and x <= g * 1e9 < x + 1
    return repr(g), g * 1e9


def level_budget(needs, base, bits):
    """The budget (bytes) at the midpoint of the room interval in which the budget loop keeps `bits`."""
    K = len(needs)
    V = [max(nd[b] for nd in needs) for b in range(BITS_MAX + 1)]
    lo = 0 if bits == 0 else K * V[bits] * PX3
    hi = 2 * lo if bits == BITS_MAX else K * V[bits + 1] * PX3
    return base + (lo + hi) // 2


@pytest.fixture(scope="module")
def hists(cuda_device, textures):
    """poses_by_food_count of every task the file uses, each from a one-task handle at the same resolution and optics."""
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        clear_env(mp)
        for name, make in ([("ladder%d" % i, m) for i, m in enumerate(LADDER_TASKS)] +
                           [("mixed%d" % i, m) for i, m in enumerate(MIXED_TASKS)] + [("replacement", REPLACEMENT)]):
            task = make()
            env = BatchedMetaMazeDiscrete3D(resolution=RES, max_steps=MAX_STEPS, num_envs=1, squeeze=False,
                                            obs_dtype="uint8", textures=textures)
            env.set_task(task)
            env.reset()
            info = env.cache_info()
            h = info["poses_by_food_count"]
            assert info["in_use"] and info["variant_bits"] == BITS_MAX
            assert sum(h) == info["poses"] == 4 * free_cells(task) and h[8] == 0, (name, h)
            assert info["variant_frames"] == need_of(h)[BITS_MAX], name
            out[name] = h
            env.close()
    return out


def table_needs(hists, prefix, tasks):
    return [need_of(hists["%s%d" % (prefix, i)]) for i in range(len(tasks))]


def assert_engine(env, cache, bits=0, frames=0, nbytes=0):
    """cache_info names the engine: the pose cache with these variant bits, frames and bytes, or the direct renderer
    (cache=False: no cache is reported)."""
    info = env.cache_info()
    got = (info["in_use"], info["variant_bits"], info["variant_frames"], info["bytes"])
    want = (cache, bits, frames, nbytes) if cache else (False, 0, 0, 0)
    assert got == want, (got, want)
    return info


# ---------------------------------------------------------------------------------------------------------------
# bit-for-bit drive against a cache=False twin (and the oracle)
# ---------------------------------------------------------------------------------------------------------------
def make_oracles(textures, tasks, e2t, task_type="SURVIVAL"):
    from oracle.maze_oracle import OracleMaze
    oras = []
    for e in range(len(e2t)):
        o = OracleMaze("3D", task_type, MAX_STEPS, 1, RES, textures=textures)
        o.set_task(tasks[e2t[e]])
        oras.append(o)
    return oras


def frame_of(o, dtype):
    return np.minimum(o, 255).astype(np.uint8) if dtype == "uint8" else o


def drive(torch, cached, direct, steps, seed, oracles=None, reset=True, rollout=True):
    """reset() (reset=True), `steps` random-action steps with auto-reset and a masked reset() half way, then (rollout=True)
    rollout(T) with and without terminal frames: every cached handle's obs, rew, done, truncated, terminal frames and
    reset() frames equal the direct twin's bit for bit, and the oracles' (one per env) through the resets and steps.  The
    oracles do not follow the rollouts: after them only a full reset() brings them back in step.  -> (dones, truncations)."""
    N, dt = direct.num_envs, direct.obs_dtype
    g = torch.Generator(device="cuda").manual_seed(seed)
    acts = torch.randint(0, 4, (steps, N), device="cuda", dtype=torch.int32, generator=g)
    mask = torch.zeros(N, dtype=torch.bool, device="cuda")
    mask[::3] = True

    def check_reset(ref, m):
        for env in cached:
            assert torch.equal(env.reset(mask=m), ref)
        if oracles is not None:
            ref = ref.cpu().numpy()
            for e, o in enumerate(oracles):
                if m is None or bool(m[e]):
                    assert np.array_equal(ref[e], frame_of(o.reset(), dt)), e

    if reset:
        check_reset(direct.reset(), None)
    n_done = n_trunc = 0
    for t in range(steps):
        if t == steps // 2:
            check_reset(direct.reset(mask=mask), mask)
        o, r, d, _ = direct.step(acts[t])
        fin, tr = direct.final_observation, direct.truncated
        for env in cached:
            o2, r2, d2, _ = env.step(acts[t])
            assert torch.equal(o2, o) and torch.equal(r2, r) and torch.equal(d2, d), t
            assert torch.equal(env.truncated, tr) and torch.equal(env.final_observation[d], fin[d]), t
        n_done += int(d.sum())
        n_trunc += int(tr.sum())
        if oracles is not None:
            oh, rh, dh, fh, ah = o.cpu().numpy(), r.cpu().numpy(), d.cpu().numpy(), fin.cpu().numpy(), acts[t].cpu().numpy()
            for e, ora in enumerate(oracles):
                o3, r3, d3, _ = ora.step(int(ah[e]))
                assert rh[e] == r3 and bool(dh[e]) == d3, (t, e)
                if d3:
                    assert np.array_equal(fh[e], frame_of(o3, dt)), (t, e)
                    o3 = ora.reset()
                assert np.array_equal(oh[e], frame_of(o3, dt)), (t, e)
    if not rollout:
        return n_done, n_trunc
    T = 24
    ra = torch.randint(0, 4, (T, N), device="cuda", dtype=torch.int32, generator=g)
    for final in (True, False):
        ref = direct.rollout(T, actions=ra, final_obs=final)
        ref = {k: (v.clone() if v is not None else None) for k, v in ref.items()}
        for env in cached:
            out = env.rollout(T, actions=ra, final_obs=final)
            for k in ("obs", "rew", "done"):
                assert torch.equal(out[k], ref[k]), (k, final)
            if final:
                d = ref["done"].bool()
                assert torch.equal(out["truncated"], ref["truncated"]) and torch.equal(out["final_obs"][d], ref["final_obs"][d])
        n_done += int(ref["done"].sum())
        n_trunc += int(ref["truncated"].sum()) if final else 0
    return n_done, n_trunc


def pair(monkeypatch, textures, n, budget=None, fused=(True,), **kw):
    """Cached handles (one per fused setting) with MGB_MAZE_CACHE_GB = budget, and their cache=False twin."""
    return ([make_env(monkeypatch, textures, n, budget=budget, fused=f, **kw) for f in fused],
            make_env(monkeypatch, textures, n, cache=False, **kw))


def close(*envs):
    for e in envs:
        for x in (e if isinstance(e, list) else [e]):
            x.close()


# ---------------------------------------------------------------------------------------------------------------
# 1. the restatement against the library
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("obs_dtype,task_type", [("uint8", "SURVIVAL"), ("int32", "SURVIVAL"), ("uint8", "ESCAPE")])
@pytest.mark.parametrize("prefix", ["ladder", "mixed"])
def test_bytes_restate_pose_cache_fits(torch_mod, textures, hists, monkeypatch, prefix, obs_dtype, task_type):
    """With the default budget, bytes - n_tasks V px 3 (V from the per-task histograms) equals the restated strided base
    bytes of pose_cache_fits, and every task of a fresh table takes all 7 bits (uint8 SURVIVAL; the other screens
    have no variant frames)."""
    makers = LADDER_TASKS if prefix == "ladder" else MIXED_TASKS
    tasks = [m() for m in makers]
    needs = table_needs(hists, prefix, makers)
    env = make_env(monkeypatch, textures, 2 * len(tasks), obs_dtype=obs_dtype, task_type=task_type)
    env.set_task(tasks)
    env.reset()
    base = base_bytes(tasks, obs_dtype, task_type)
    if obs_dtype == "uint8" and task_type == "SURVIVAL":
        V = max(nd[BITS_MAX] for nd in needs)
        assert_engine(env, True, BITS_MAX, sum(nd[BITS_MAX] for nd in needs), int(base + len(tasks) * V * PX3))
    else:
        assert_engine(env, True, 0, 0, int(base))
    env.close()


def test_ladder_table_reaches_every_level(hists):
    """The ladder's table makes every bits from 7 down to 1 a level of its own (V grows at each), and at some level
    below 7 a task would take more frames if its plan were given the handle's 7 bits instead of the table's."""
    needs = table_needs(hists, "ladder", LADDER_TASKS)
    V = [max(nd[b] for nd in needs) for b in range(BITS_MAX + 1)]
    assert V[1] > 0 and all(V[b] < V[b + 1] for b in range(1, BITS_MAX)), V
    assert any(task_plan(nd, BITS_MAX, V[b])[1] != task_plan(nd, b, V[b])[1] for b in range(1, BITS_MAX) for nd in needs)


# ---------------------------------------------------------------------------------------------------------------
# 2. the budget ladder
# ---------------------------------------------------------------------------------------------------------------
def run_budget(torch, monkeypatch, textures, hists, budget_bytes, want_bits, oracle=False):
    """The ladder's table under MGB_MAZE_CACHE_GB = budget_bytes / 1e9: the restated decision is `want_bits` (None: over
    budget), cache_info reports exactly the restatement on the fused and the two-kernel step paths, and both equal the
    cache=False twin through steps, resets and rollouts (and the oracle through the steps)."""
    tasks = [m() for m in LADDER_TASKS]
    needs = table_needs(hists, "ladder", LADDER_TASKS)
    K, N = len(tasks), 16
    base = base_bytes(tasks)
    gb, budget = budget_gb(budget_bytes)
    fits = base <= budget
    bits, V = budget_plan(needs, base, budget)
    assert (bits if fits else None) == want_bits
    frames = sum(task_plan(nd, bits, V)[1] for nd in needs)
    assert frames == sum(nd[bits] for nd in needs)          # a fresh table: every task takes the table's bits
    cached, direct = pair(monkeypatch, textures, N, budget=gb, fused=(True, False))
    for env in cached + [direct]:
        env.set_task(tasks)
    oras = make_oracles(textures, tasks, np.arange(N) % K) if oracle else None
    n_done, n_trunc = drive(torch, cached, direct, 64, seed=bits, oracles=oras)
    assert 0 < n_trunc < n_done                              # episodes end through the step limit and through life
    for env in cached:
        assert_engine(env, fits, bits, frames, int(base + K * V * PX3))
    close(cached, direct)


@pytest.mark.parametrize("bits", range(BITS_MAX, -1, -1))
def test_budget_ladder(torch_mod, textures, hists, monkeypatch, bits):
    """A budget at the midpoint of the interval in which the budget loop keeps `bits` (7 down to 0)."""
    tasks = [m() for m in LADDER_TASKS]
    target = level_budget(table_needs(hists, "ladder", LADDER_TASKS), base_bytes(tasks), bits)
    run_budget(torch_mod, monkeypatch, textures, hists, target, bits, oracle=bits in (5, 2))


THRESHOLD_BITS = 3


@pytest.mark.parametrize("edge,want", [("base", 0), ("base-1", None), ("threshold-1", THRESHOLD_BITS - 1),
                                       ("threshold", THRESHOLD_BITS), ("threshold+1", THRESHOLD_BITS)])
def test_budget_edges(torch_mod, textures, hists, monkeypatch, edge, want):
    """Exactly the base bytes fits with 0 bits and one byte less renders directly; one byte either side of the
    threshold of 3 bits (n_tasks V_3 px 3 bytes of room)."""
    tasks = [m() for m in LADDER_TASKS]
    needs = table_needs(hists, "ladder", LADDER_TASKS)
    base = int(base_bytes(tasks))
    thr = base + len(tasks) * max(nd[THRESHOLD_BITS] for nd in needs) * PX3
    target = {"base": base, "base-1": base - 1, "threshold-1": thr - 1, "threshold": thr, "threshold+1": thr + 1}[edge]
    run_budget(torch_mod, monkeypatch, textures, hists, target, want)


# ---------------------------------------------------------------------------------------------------------------
# 3. tasks with mixed bits after update_tasks
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["u8_default", "u8_limited", "int32", "escape"])
def test_mixed_bits_after_update_tasks(torch_mod, textures, hists, monkeypatch, case):
    """Slot 0 of a table of tasks that need few frames takes a task that needs more than the table's V frames: it gets
    the largest bits whose frames fit V (fewer than its neighbours'), and envs on it and on its neighbours equal the
    direct twin and the oracle through steps, terminal frames and rollouts; swapped back, the frame count returns.  Once
    with the default budget (7 bits), once with a budget that leaves the table fewer bits, and on int32 and ESCAPE
    screens, which have no variant frames."""
    torch = torch_mod
    tasks = [m() for m in MIXED_TASKS]
    repl = REPLACEMENT()
    needs = table_needs(hists, "mixed", MIXED_TASKS)
    need_r = need_of(hists["replacement"])
    K, N = len(tasks), 16
    dtype = "int32" if case == "int32" else "uint8"
    task_type = "ESCAPE" if case == "escape" else "SURVIVAL"
    base = base_bytes(tasks, dtype, task_type)
    gb, budget = None, 24e9
    if case == "u8_limited":
        V = [max(nd[b] for nd in needs) for b in range(BITS_MAX + 1)]
        lowest = min(b for b in range(1, BITS_MAX) if V[b] < V[b + 1])        # the lowest level above 0
        gb, budget = budget_gb(level_budget(needs, base, lowest))
    if case.startswith("u8"):
        bits, V = budget_plan(needs, base, budget)
        assert (bits < BITS_MAX) == (case == "u8_limited") and bits > 0
        frames0 = sum(task_plan(nd, bits, V)[1] for nd in needs)
        bits_r, frames_r = task_plan(need_r, bits, V)
        assert bits_r < bits and V < need_r[bits] <= K * V, (bits_r, bits, V, need_r)
        frames1 = frames0 - task_plan(needs[0], bits, V)[1] + frames_r
        nbytes = int(base + K * V * PX3)
    else:
        bits = frames0 = frames1 = 0
        nbytes = int(base)
    (cached,), direct = pair(monkeypatch, textures, N, budget=gb, obs_dtype=dtype, task_type=task_type)
    e2t = np.arange(N) % K
    for env in (cached, direct):
        env.set_task(tasks, env2task=e2t)
    oras = make_oracles(textures, tasks, e2t, task_type)
    drive(torch, [cached], direct, 20, seed=1, oracles=oras, rollout=False)
    assert_engine(cached, True, bits, frames0, nbytes)
    for env in (cached, direct):
        env.update_tasks([0], [repl])
    for e in np.flatnonzero(e2t == 0):
        oras[e].set_task(repl)
        oras[e].reset()
    assert_engine(cached, True, bits, frames1, nbytes)
    drive(torch, [cached], direct, 40, seed=2, oracles=oras, reset=False)
    for env in (cached, direct):
        env.update_tasks([0], [tasks[0]])
    for e in np.flatnonzero(e2t == 0):
        oras[e].set_task(tasks[0])
    assert_engine(cached, True, bits, frames0, nbytes)
    n_done, _ = drive(torch, [cached], direct, 40, seed=3, oracles=oras)
    assert n_done > 0
    close(cached, direct)


# ---------------------------------------------------------------------------------------------------------------
# 4. decisions that must not go stale
# ---------------------------------------------------------------------------------------------------------------
def test_set_task_decides_the_engine_for_its_table(torch_mod, textures, hists, monkeypatch):
    """One handle: a table that fits (2 bits), one over the same budget (direct renderer, no cache reported), the first
    one again (the same cache as at first), each equal to a cache=False twin given the same tables."""
    tasks = [m() for m in LADDER_TASKS]
    needs = table_needs(hists, "ladder", LADDER_TASKS)
    base = base_bytes(tasks)
    gb, budget = budget_gb(level_budget(needs, base, 2))
    bits, V = budget_plan(needs, base, budget)
    assert bits == 2 and base_bytes(tasks + tasks) > budget
    want = (True, bits, sum(nd[bits] for nd in needs), int(base + len(tasks) * V * PX3))
    (cached,), direct = pair(monkeypatch, textures, 16, budget=gb)
    for k, table in enumerate([tasks, tasks + tasks, tasks]):
        for env in (cached, direct):
            env.set_task(table)
        drive(torch_mod, [cached], direct, 20, seed=10 + k)
        if k == 1:
            assert_engine(cached, False)
        else:
            assert_engine(cached, *want)
    close(cached, direct)


def test_set_cache_off_and_on_rebuilds_the_same_cache(torch_mod, textures, hists, monkeypatch):
    """set_cache(False) on a built cache switches to the direct renderer mid-episode (no cache reported);
    set_cache(True) rebuilds the same cache_info; the frames equal a cache=False twin throughout."""
    from metagym_b200 import _lib
    tasks = [m() for m in LADDER_TASKS]
    needs = table_needs(hists, "ladder", LADDER_TASKS)
    V = max(nd[BITS_MAX] for nd in needs)
    (cached,), direct = pair(monkeypatch, textures, 16)
    for env in (cached, direct):
        env.set_task(tasks)
    drive(torch_mod, [cached], direct, 20, seed=20, rollout=False)
    info0 = assert_engine(cached, True, BITS_MAX, sum(nd[BITS_MAX] for nd in needs),
                          int(base_bytes(tasks) + len(tasks) * V * PX3))
    for on, seed in ((0, 21), (1, 22)):
        _lib.check(cached._lib.mgb_maze_set_cache(cached._h, on))
        drive(torch_mod, [cached], direct, 20, seed=seed, reset=False)
        info = assert_engine(cached, bool(on), info0["variant_bits"], info0["variant_frames"], info0["bytes"])
        if on:
            assert info == info0
    close(cached, direct)


def test_over_budget_answers_do_not_depend_on_the_first_reset(torch_mod, textures, monkeypatch):
    """What update_tasks and resample_tasks accept depends on the table, the textures and the budget, not on whether a
    reset() has built (or declined to build) the cache.  Over budget (the direct renderer): a replacement with more free
    cells than the table's largest task, a slot replaced twice in one call and device resampling are accepted before
    the first reset() as after it, and the handles then equal a cache=False twin given the same calls.  Within the
    budget: the same calls are refused before the first reset() as after it."""
    from metagym_b200._lib import MgbError
    torch = torch_mod
    tasks = [wall_row_task([(2, 3), (6, 6)]), pockets_task(POCKETS, POCKETS[:3]), wall_row_task([(5, 6)]),
             wall_row_task([(2, 2), (2, 6), (6, 2)])]
    big = maze_task([(3, 3), (5, 5)])
    assert free_cells(big) > max(free_cells(t) for t in tasks)
    N = len(tasks)
    e2t = np.arange(N)
    mask = torch.tensor([1, 0, 1, 1], dtype=torch.uint8, device="cuda")

    def calls(env):
        env.update_tasks([0], [big])
        env.update_tasks([2, 2], [tasks[3], tasks[0]])
        env.resample_tasks(mask, seed=4)

    over, _ = budget_gb(base_bytes(tasks) - 1)
    before, after = [make_env(monkeypatch, textures, N, budget=over) for _ in range(2)]
    direct = make_env(monkeypatch, textures, N, cache=False)
    for env in (before, after, direct):
        env.set_task(tasks, env2task=e2t)
    calls(before)
    after.reset()
    for env in (after, direct):
        calls(env)
    drive(torch, [before, after], direct, 30, seed=30)
    for env in (before, after):
        assert_engine(env, False)
    close(before, after, direct)

    fitting = [make_env(monkeypatch, textures, N) for _ in range(2)]
    for k, env in enumerate(fitting):
        env.set_task(tasks, env2task=e2t)
        if k:
            env.reset()
        with pytest.raises(MgbError, match="free cells"):
            env.update_tasks([0], [big])
        with pytest.raises(MgbError, match="only once per call"):
            env.update_tasks([2, 2], [tasks[3], tasks[0]])
        with pytest.raises(MgbError, match="direct renderer"):
            env.resample_tasks(mask, seed=4)
        env.reset()
        assert env.cache_info()["in_use"]
    close(fitting)
