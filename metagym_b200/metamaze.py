"""Batched drop-ins for metagym.metamaze.MetaMaze2D / MetaMazeDiscrete3D
(reference: metagym/metamaze/envs/maze_env.py:16-75, 155-206) plus a host-side task sampler.

Same constructor kwargs, `set_task` / `reset` / `step` protocol and error messages as the reference, with a leading
batch axis over `num_envs` independent instances stepped by libmgb200 (metagym_b200/csrc/maze.cu).  A task is the
reference's `TaskConfig` namedtuple (metagym/metamaze/envs/maze_task.py:15-17); objects produced by the reference's own
`MazeTaskSampler` are accepted as they are (duck-typed by field name).
"""
import ctypes
import math
from collections import namedtuple

import numpy as np

from . import _lib
from .rollout import Mirrored
from .snapshot import Snapshots
from .spaces import Box, Discrete
from .textures import synthetic_textures

PI = 3.1415926                                       # metagym/metamaze/envs/dynamics.py:6
DISCRETE_ACTIONS = [(-1, 0), (1, 0), (0, -1), (0, 1)]   # maze_env.py:14

TaskConfig = namedtuple("TaskConfig", ["start", "goal", "cell_walls", "cell_texts", "cell_size", "wall_height",
                                       "agent_height", "initial_life", "max_life", "step_reward", "goal_reward",
                                       "food_rewards", "food_interval"])


class _DSU(object):
    def __init__(self, n):
        self.p = list(range(n))

    def find(self, x):
        while self.p[x] != x:
            self.p[x] = self.p[self.p[x]]
            x = self.p[x]
        return x

    def union(self, a, b):
        a, b = self.find(a), self.find(b)
        if a == b:
            return False
        self.p[a] = b
        return True


def _carve_like_reference(n, allow_loops, crowd_ratio, py):
    """The wall-removal process of maze_task.py:84-151, restated on arrays, consuming `py` (a `random.Random` or the
    `random` module) call for call like the reference: one `shuffle` of the walls still standing per round (in their
    row-major order of creation), then walls are examined in shuffled order until one (a) joins different regions
    without closing a loop, (b) joins regions and closes a loop (only with allow_loops), or (c) once a single region is
    left, wins a `random() < 0.2` draw.  A round that runs out of walls takes the last one examined (reference quirk:
    the loop variables simply survive the for statement); a chosen wall with no open neighbour is skipped.
    Rounds continue while more than one region exists or (allow_loops and interior walls exceed crowd_ratio)."""
    walls = np.ones((n, n), dtype=np.int32)
    walls[1:n:2, 1:n:2] = 0
    region = np.full((n, n), -1, dtype=np.int64)
    rooms = [(i, j) for i in range(1, n - 1) for j in range(1, n - 1) if walls[i, j] == 0]
    for k, (i, j) in enumerate(rooms):
        region[i, j] = k
    members = {k: [c] for k, c in enumerate(rooms)}
    standing = [(i, j) for i in range(1, n - 1) for j in range(1, n - 1) if walls[i, j] > 0]
    limit = (n - 2) * (n - 2) * crowd_ratio
    while len(members) > 1 or (allow_loops and len(standing) > limit):
        order = list(standing)
        py.shuffle(order)
        if not order:
            raise RuntimeError("maze sampler: no wall left to remove")
        for i, j in order:
            ids = [int(region[a, b]) for a, b in ((i - 1, j), (i + 1, j), (i, j - 1), (i, j + 1)) if walls[a, b] < 1]
            keep = min(ids) if ids else -1
            others = set(ids) - {keep}
            repeats = max([ids.count(v) for v in ids] + [1])
            if others and repeats < 2:
                break
            if others and repeats > 1 and allow_loops:
                break
            if allow_loops and len(members) < 2 and py.random() < 0.2:
                break
        if keep < 0:
            continue
        walls[i, j] = 0
        region[i, j] = keep
        members[keep].append((i, j))
        standing.remove((i, j))
        for o in others:
            for a, b in members[o]:
                region[a, b] = keep
            members[keep].extend(members.pop(o))
    return walls


def _sample_task_reference_streams(n, allow_loops, cell_size, wall_height, agent_height, step_reward, goal_reward,
                                   food_reward, initial_life, max_life, food_density, food_interval, crowd_ratio,
                                   n_texts, py, npr):
    """maze_task.py:41-190 with the reference's exact random-stream usage: with py = `random` and npr = `numpy.random`
    after `random.seed(s); numpy.random.seed(s)` (or `random.Random(s)` / `numpy.random.RandomState(s)`) the task is
    the reference's task for that seed, array for array (tests/test_maze_sampler.py, fixtures recorded from the
    unmodified reference)."""
    texts = npr.randint(1, n_texts, size=(n, n))
    m = (n - 1) // 2
    sx = py.randint(0, m - 1) * 2 + 1
    sy = py.randint(0, m - 1) * 2 + 1
    goal = (n - 2, n - 2)
    for _ in range(m):                 # the reference's `break` leaves the inner loop only: m rows of up to m draws,
        for _ in range(m):             # the LAST far-enough candidate of a row that found one wins
            ex = py.randint(0, m - 1) * 2 + 1
            ey = py.randint(0, m - 1) * 2 + 1
            if np.sqrt((ex - sx) ** 2 + (ey - sy) ** 2) > 0.45 * n:
                goal = (ex, ey)
                break
    walls = _carve_like_reference(n, allow_loops, crowd_ratio, py)
    inner = texts[1:-1, 1:-1]
    inner[walls[1:-1, 1:-1] < 1] = 0
    def_goal_reward = -np.sqrt(n) * n * step_reward if goal_reward is None else goal_reward
    assert def_goal_reward > 0, "goal reward must be > 0"
    food = np.clip(npr.rand(n, n) * food_reward, 0.10, food_reward)
    food *= 1.0 - walls
    expected = (n - 1) * (n - 1) * food_density
    while np.sum(food) > expected:
        food *= (npr.rand(n, n) < 0.90).astype("float32")
    interval = food_interval * (food > 1.0e-3).astype("int32")
    return TaskConfig(start=(sx, sy), goal=goal, cell_walls=walls, cell_texts=texts, cell_size=cell_size,
                      step_reward=step_reward, goal_reward=def_goal_reward, wall_height=wall_height,
                      agent_height=agent_height, initial_life=initial_life, max_life=max_life, food_rewards=food,
                      food_interval=interval)


def MazeTaskSampler(n=15, allow_loops=True, cell_size=2.0, wall_height=3.2, agent_height=1.6, step_reward=-0.01,
                    goal_reward=None, food_reward=0.50, initial_life=1.0, max_life=2.0, food_density=0.010,
                    food_interval=100, crowd_ratio=0.0, n_texts=7, rng=None, seed=None, py_random=None, np_random=None):
    """Random maze task with the reference sampler's schema, defaults and constraints (maze_task.py:41-190).

    Default (no `rng`): the reference's procedure replayed on the reference's random streams - the global `random` and
    `numpy.random` modules, or `py_random` / `np_random` instances, or both seeded from `seed` - so that
    `random.seed(s); numpy.random.seed(s); MazeTaskSampler(...)` returns exactly the task the reference returns.

    With `rng` (a numpy RandomState): a faster sampler of the same DISTRIBUTION family (rooms on odd coordinates, a
    random spanning tree by Kruskal over the room lattice, then with `allow_loops` interior walls are knocked out until
    at most `crowd_ratio` of the interior is wall); not sample-identical to the reference.
    """
    assert n > 6, "Minimum required cells are 7"
    assert n % 2 != 0, "Cell Numbers can only be odd"
    assert step_reward < 0, "step_reward must be < 0"
    if rng is None:
        import random as _pyrandom
        py = py_random if py_random is not None else (_pyrandom.Random(seed) if seed is not None else _pyrandom)
        npr = np_random if np_random is not None else (np.random.RandomState(seed) if seed is not None else np.random)
        return _sample_task_reference_streams(n, allow_loops, cell_size, wall_height, agent_height, step_reward,
                                              goal_reward, food_reward, initial_life, max_life, food_density,
                                              food_interval, crowd_ratio, n_texts, py, npr)
    rs = rng
    walls = np.ones((n, n), dtype=np.int32)
    walls[1:n:2, 1:n:2] = 0
    m = (n - 1) // 2
    dsu = _DSU(m * m)
    edges = []
    for a in range(m):
        for b in range(m):
            if a + 1 < m:
                edges.append((2 * a + 2, 2 * b + 1, a * m + b, (a + 1) * m + b))
            if b + 1 < m:
                edges.append((2 * a + 1, 2 * b + 2, a * m + b, a * m + b + 1))
    for k in rs.permutation(len(edges)):
        i, j, u, v = edges[k]
        if dsu.union(u, v):
            walls[i, j] = 0
    if allow_loops:
        interior = walls[1:-1, 1:-1]
        budget = interior.size * crowd_ratio
        cand = [(i, j) for i in range(1, n - 1) for j in range(1, n - 1) if walls[i, j] > 0]
        for k in rs.permutation(len(cand)):
            if interior.sum() <= budget:
                break
            i, j = cand[k]
            if walls[i - 1, j] == 0 or walls[i + 1, j] == 0 or walls[i, j - 1] == 0 or walls[i, j + 1] == 0:
                walls[i, j] = 0
    texts = rs.randint(1, n_texts, size=(n, n))
    texts[walls < 1] = 0
    start = (int(rs.randint(0, m)) * 2 + 1, int(rs.randint(0, m)) * 2 + 1)
    goal = (n - 2, n - 2)
    for _ in range(m * m):
        cand = (int(rs.randint(0, m)) * 2 + 1, int(rs.randint(0, m)) * 2 + 1)
        if np.hypot(cand[0] - start[0], cand[1] - start[1]) > 0.45 * n:
            goal = cand
            break
    def_goal_reward = -np.sqrt(n) * n * step_reward if goal_reward is None else goal_reward
    assert def_goal_reward > 0, "goal reward must be > 0"
    food = np.clip(rs.rand(n, n) * food_reward, 0.10, food_reward) * (1.0 - walls)
    expected = (n - 1) * (n - 1) * food_density
    while food.sum() > expected:
        food *= (rs.rand(n, n) < 0.90).astype("float32")
    interval = food_interval * (food > 1.0e-3).astype("int32")
    return TaskConfig(start=start, goal=goal, cell_walls=walls, cell_texts=texts, cell_size=cell_size,
                      step_reward=step_reward, goal_reward=def_goal_reward, wall_height=wall_height,
                      agent_height=agent_height, initial_life=initial_life, max_life=max_life, food_rewards=food,
                      food_interval=interval)


def new_tasks(out):
    """[T, N] bool CUDA tensor: True where env e drew a new maze at step t of the rollout that returned `out` (the
    "task" reset rule of the recurrent policies fires exactly there).  False everywhere when the rollout did not
    resample; `done` for a resampling rollout of a handle without trials; on a trial handle (episodes_per_task=k) the
    finished episodes that were the k-th on their maze, counted from out["task_episodes0"].  `out` is the dict of a
    recurrent rollout or of any rollout of a trial handle (both record whether the launch resampled)."""
    import torch
    done = out["done"].bool()
    if not out.get("resampled", False):
        return torch.zeros_like(done)
    k = out.get("episodes_per_task")
    if k is None:
        return done
    count = out["task_episodes0"].to(done.device, torch.int64)
    drew = torch.empty_like(done)
    for t in range(done.shape[0]):
        count = count + done[t]
        drew[t] = done[t] & (count >= k)
        count = count.masked_fill(drew[t], 0)
    return drew


class _BatchedMazeBase(Snapshots):
    """snapshot() / restore() / clone_envs() (metagym_b200/snapshot.py): exact checkpoint and resume of agent, life, food,
    resample counts, trial episode counts, continuous pose, task slot (and, for one table slot per env on the direct
    renderer, the task itself) and the rollout action counter.  A restore clears need_reset."""
    KIND = None
    _SNAP_PREFIX = "mgb_maze"
    _FINGERPRINT_PARTS = ("configuration (kind, task type, max_steps, view, resolution, obs dtype, optics, auto_reset, "
                          "table shape, path recording, episodes_per_task)", "textures", "task table", "record mode (per-env tasks or a shared table)")

    def _snap_kind(self):
        return ("maze2d", "maze_discrete_3d", "maze_continuous_3d")[self.KIND]

    def _after_restore(self, rec, row_dev, row):
        """A shared-table restore points env2task at the records' slots (int32 7 of a record)."""
        self.need_reset = False
        if self._fingerprint()[3] == 0 and rec.shape[0]:
            slot = rec.view(self._torch.int32)[:, 7].cpu().numpy()
            self.env2task = np.ascontiguousarray(np.where(row >= 0, slot[np.maximum(row, 0)], self.env2task),
                                                 dtype=np.int32)

    def _setup(self, num_envs, device, task_type, max_steps, auto_reset, env_index_base, squeeze, final_obs=False,
               record_path=False, episodes_per_task=None, expert=False):
        import torch
        assert task_type in ("SURVIVAL", "ESCAPE")
        if expert and task_type != "ESCAPE":
            raise ValueError("expert=True is defined for ESCAPE only (SURVIVAL has no single shortest-path target)")
        if expert and self.KIND == 2:
            raise ValueError("expert=True is defined for the grid mazes only (MetaMazeContinuous3D has continuous actions)")
        self.with_expert = bool(expert)
        self._exp = None
        if final_obs and not auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True (without auto-reset obs already is the terminal frame)")
        if episodes_per_task is not None and not (int(episodes_per_task) == episodes_per_task and episodes_per_task >= 1):
            raise ValueError("episodes_per_task must be None or an integer >= 1, got %r" % (episodes_per_task,))
        self.episodes_per_task = None if episodes_per_task is None else int(episodes_per_task)
        self._want_final = bool(final_obs)
        self.record_path = bool(record_path)
        self._torch = torch
        self.num_envs = int(num_envs)
        self.task_type = task_type
        self.max_steps = max_steps
        self.auto_reset = bool(auto_reset)
        self.env_index_base = int(env_index_base)
        self._squeeze = bool(squeeze) and self.num_envs == 1
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if self.device.type != "cuda" or not torch.cuda.is_available():
            raise _lib.MgbError("metagym_b200 runs on CUDA devices only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._lib = _lib.load()
        self._h = None
        self._n_cells = None
        self.action_space = Discrete(4)
        self.need_reset = True                         # maze_env.py:41-42
        self.need_set_task = True
        self._rew = torch.empty((self.num_envs,), dtype=torch.float64, device=self.device)
        self._done = torch.empty((self.num_envs,), dtype=torch.uint8, device=self.device)
        self._own_ptrs = None
        self._final = self._trunc = None

    def _alloc_final(self):
        """Persistent final_obs / truncated buffers (final_obs=True), so that step() can be captured in a CUDA graph."""
        if self._want_final:
            self._final = self._torch.zeros_like(self._obs)
            self._trunc = self._torch.zeros((self.num_envs,), dtype=self._torch.uint8, device=self.device)

    @property
    def final_observation(self):
        """final_obs=True: [N, <obs of one env>] in the obs dtype.  After step(), row e holds the terminal observation
        of env e if done[e] (what an auto_reset=False env would have returned; obs holds the next episode's first
        frame).  Rows of envs that did not finish in that step are left untouched: they keep an earlier terminal frame
        (zeros before the first).  None with final_obs=False."""
        return None if self._final is None else self._out(self._final)

    @property
    def truncated(self):
        """final_obs=True: [N] bool, written by every step(): True iff done and the episode ended only through the step
        limit (max_steps), so terminated = done & ~truncated.  None with final_obs=False."""
        return None if self._trunc is None else self._out(self._trunc.view(self._torch.bool))

    @property
    def task_episodes(self):
        """Trial handles (episodes_per_task=k): CUDA int32 [N], the episodes each env has finished (done) since it was
        last given a maze (set_task, update_tasks, resample_tasks or an in-launch draw); reset() leaves it alone.  A copy,
        stream-ordered.  None for a handle without trials."""
        if self.episodes_per_task is None:
            return None
        if self.need_set_task:
            raise Exception("Must call \"set_task\" before reset")
        out = self._torch.empty((self.num_envs,), dtype=self._torch.int32, device=self.device)
        _lib.check(self._lib.mgb_maze_task_episodes(self._h, out.data_ptr(), self._stream()))
        return out

    def _trial_entries(self, out, resample):
        """A trial handle's rollout dict gains "task_episodes0" (the counts at launch start, copied on the stream before
        the launch; a caller-supplied tensor is filled in place), "episodes_per_task" and "resampled"."""
        if self.episodes_per_task is None:
            return
        te = out.get("task_episodes0")
        if te is None:
            te = self._torch.empty((self.num_envs,), dtype=self._torch.int32, device=self.device)
        _lib.check(self._lib.mgb_maze_task_episodes(self._h, te.data_ptr(), self._stream()))
        out["task_episodes0"] = te
        out["episodes_per_task"] = self.episodes_per_task
        out["resampled"] = resample is not None

    def _stream(self):
        return _lib.current_stream(self._torch, self.device)

    def _make_cfg(self, n_cells):
        raise NotImplementedError

    def _after_create(self):
        pass

    def _create(self, n_cells):
        if self._h is not None:
            if n_cells == self._n_cells:
                return
            self._lib.mgb_maze_destroy(self._h)
            self._h = None
        cfg = self._make_cfg(n_cells)
        h = ctypes.c_void_p()
        _lib.check(self._lib.mgb_maze_create(ctypes.byref(h), self.num_envs, ctypes.byref(cfg), self.device.index,
                                             self.env_index_base))
        self._h, self._n_cells = h, n_cells
        _lib.check(self._lib.mgb_maze_set_options(self._h, int(self.auto_reset)))
        if self.record_path:
            _lib.check(self._lib.mgb_maze_set_path(self._h, 1))
        if self.episodes_per_task is not None:
            _lib.check(self._lib.mgb_maze_set_episodes_per_task(self._h, self.episodes_per_task))
        if self.with_expert:
            _lib.check(self._lib.mgb_maze_set_expert(self._h, 1))
        self._after_create()

    @staticmethod
    def _pack_tasks(tasks):
        """TaskConfigs -> the C ABI's task arrays: walls, texts [K,n,n] int8, food [K,n,n] float64, interval [K,n,n]
        int32, and a MazeTaskScalars[K]."""
        walls = np.ascontiguousarray(np.stack([np.asarray(t.cell_walls) for t in tasks]).astype(np.int8))
        texts = np.ascontiguousarray(np.stack([np.asarray(t.cell_texts) for t in tasks]).astype(np.int8))
        food = np.ascontiguousarray(np.stack([np.asarray(t.food_rewards, dtype=np.float64) for t in tasks]))
        itv = np.ascontiguousarray(np.stack([np.asarray(t.food_interval) for t in tasks]).astype(np.int32))
        sc = (_lib.MazeTaskScalars * len(tasks))()
        for k, t in enumerate(tasks):
            sc[k].start[:] = [int(t.start[0]), int(t.start[1])]
            sc[k].goal[:] = [int(t.goal[0]), int(t.goal[1])]
            sc[k].cell_size, sc[k].wall_height, sc[k].agent_height = t.cell_size, t.wall_height, t.agent_height
            sc[k].initial_life, sc[k].max_life = t.initial_life, t.max_life
            sc[k].step_reward, sc[k].goal_reward = t.step_reward, t.goal_reward
        return walls, texts, food, itv, sc

    def set_task(self, task_config, env2task=None):
        """MazeBase.set_task (maze_base.py:19-38).  `task_config`: one TaskConfig (all envs) or a sequence of them;
        env i then runs task env2task[i] (default: (env_index_base + i) % n_tasks)."""
        tasks = [task_config] if hasattr(task_config, "cell_walls") else list(task_config)
        n = int(np.shape(tasks[0].cell_walls)[0])
        for t in tasks:
            w = np.asarray(t.cell_walls)
            assert t.agent_height < t.wall_height and t.agent_height > 0, \
                "the agent height must be > 0 and < wall height"
            assert w.shape == np.shape(t.cell_texts), "the dimension of walls must be equal to textures"
            assert w.shape[0] == w.shape[1], "only support square shape"
            assert w.shape[0] == n, "all tasks of one batch must share the maze size"
        self._create(n)
        K = len(tasks)
        walls, texts, food, itv, sc = self._pack_tasks(tasks)
        if env2task is None:
            env2task = (np.arange(self.num_envs, dtype=np.int64) + self.env_index_base) % K
        e2t = np.ascontiguousarray(np.asarray(env2task, dtype=np.int32))
        assert e2t.shape == (self.num_envs,)
        self._torch.cuda.synchronize(self.device)
        _lib.check(self._lib.mgb_maze_set_task(self._h, K, walls.ctypes.data, texts.ctypes.data, food.ctypes.data,
                                               itv.ctypes.data, sc, e2t.ctypes.data))
        self.tasks, self.env2task = tasks, e2t
        self.need_set_task = False
        self.need_reset = True

    def update_tasks(self, task_slots, task_configs):
        """Per-episode task resampling: replace entries `task_slots` of the task table by `task_configs`, stream-ordered
        and without a device synchronisation (mgb_maze_update_tasks).  Envs flying a replaced slot restart on the new task.
        With set_task(tasks) of one task per env (env2task = arange), `update_tasks(env_ids, new_tasks)` re-tasks exactly
        those envs.  On the pose cache (MetaMazeDiscrete3D) the replaced tasks' poses and frames are rebuilt in place on
        the stream; there a replacement may not have more free cells (the start cell included) than the largest task
        set_task was given, and a slot may appear only once per call."""
        slots = np.ascontiguousarray(np.asarray(task_slots, dtype=np.int32).reshape(-1))
        tasks = [task_configs] if hasattr(task_configs, "cell_walls") else list(task_configs)
        K = len(tasks)
        assert slots.shape == (K,), "one task per slot"
        walls, texts, food, itv, sc = self._pack_tasks(tasks)
        assert walls.shape[1:] == (self._n_cells, self._n_cells), "all tasks of one batch must share the maze size"
        for t in tasks:
            assert t.agent_height < t.wall_height and t.agent_height > 0, "the agent height must be > 0 and < wall height"
        _lib.check(self._lib.mgb_maze_update_tasks(self._h, K, slots.ctypes.data, walls.ctypes.data, texts.ctypes.data,
                                                   food.ctypes.data, itv.ctypes.data, sc, self._stream()))
        for k, sl in enumerate(slots):
            self.tasks[int(sl)] = tasks[k]

    @staticmethod
    def _sampler_cfg(seed=0, allow_loops=True, cell_size=2.0, wall_height=3.2, agent_height=1.6, step_reward=-0.01,
                     goal_reward=None, food_reward=0.50, initial_life=1.0, max_life=2.0, food_density=0.010,
                     food_interval=100, crowd_ratio=0.0, n_texts=7):
        """resample_tasks' keyword arguments -> (MazeSamplerCfg, seed), for resample_tasks and rollout(resample=...)."""
        if goal_reward is not None and not goal_reward > 0:
            raise ValueError("goal reward must be > 0")
        cfg = _lib.MazeSamplerCfg()
        cfg.allow_loops, cfg.n_texts, cfg.food_interval = int(bool(allow_loops)), int(n_texts), int(food_interval)
        cfg.cell_size, cfg.wall_height, cfg.agent_height = cell_size, wall_height, agent_height
        cfg.step_reward, cfg.goal_reward = step_reward, (0.0 if goal_reward is None else goal_reward)
        cfg.food_reward, cfg.initial_life, cfg.max_life = food_reward, initial_life, max_life
        cfg.food_density, cfg.crowd_ratio = food_density, crowd_ratio
        return cfg, int(seed)

    def resample_tasks(self, mask=None, seed=0, allow_loops=True, cell_size=2.0, wall_height=3.2, agent_height=1.6,
                       step_reward=-0.01, goal_reward=None, food_reward=0.50, initial_life=1.0, max_life=2.0,
                       food_density=0.010, food_interval=100, crowd_ratio=0.0, n_texts=7):
        """Per-episode task resampling on the device (mgb_maze_resample_tasks): every env with mask[e] != 0 (None: all)
        gets a freshly drawn maze (MazeTaskSampler's keyword arguments and distribution family; counter-based draws keyed
        by (seed, global env index, resample count)) and restarts on it.  One stream-ordered kernel.  Needs set_task() with one table slot per env (env2task = arange) and the direct renderer (cache=False).
        goal_reward None is the reference's default -sqrt(n) * n * step_reward; an explicit goal_reward <= 0 raises
        ValueError, as MazeTaskSampler refuses it.

        This call renders nothing.  In the loop `obs, rew, done, _ = env.step(a); env.resample_tasks(done)` with
        auto_reset on, the step has already reset every finished env on its OLD maze, so `obs` shows a re-tasked env in a
        maze it no longer is in.  For the frame on the new maze, follow with `obs = env.reset(mask=done)` (which renders
        every env once more), or let `rollout(T, resample=dict(seed=..., ...))` (every env kind) draw the new maze inside
        the rollout, where obs[t] of a finished env already is its first frame on the new maze."""
        m = None
        if mask is not None:
            m = self._torch.as_tensor(mask, device=self.device).to(self._torch.uint8).contiguous()
        cfg, seed = self._sampler_cfg(seed, allow_loops, cell_size, wall_height, agent_height, step_reward, goal_reward,
                                      food_reward, initial_life, max_life, food_density, food_interval, crowd_ratio, n_texts)
        _lib.check(self._lib.mgb_maze_resample_tasks(self._h, _lib.ptr(m), ctypes.byref(cfg), seed, self._stream()))
        self.need_reset = False

    def get_tasks(self, task_slots):
        """Tasks currently in the table slots `task_slots` (synchronous read-back) -> list of TaskConfig."""
        slots = np.ascontiguousarray(np.asarray(task_slots, dtype=np.int32).reshape(-1))
        K, n = int(slots.size), self._n_cells
        walls = np.empty((K, n, n), np.int8); texts = np.empty((K, n, n), np.int8)
        food = np.empty((K, n, n), np.float64); itv = np.empty((K, n, n), np.int32)
        sc = (_lib.MazeTaskScalars * K)()
        _lib.check(self._lib.mgb_maze_get_tasks(self._h, K, slots.ctypes.data, walls.ctypes.data, texts.ctypes.data,
                                                food.ctypes.data, itv.ctypes.data, sc))
        return [TaskConfig(start=(int(sc[k].start[0]), int(sc[k].start[1])), goal=(int(sc[k].goal[0]), int(sc[k].goal[1])),
                           cell_walls=walls[k].astype(np.int32), cell_texts=texts[k].astype(np.int64),
                           cell_size=sc[k].cell_size, step_reward=sc[k].step_reward, goal_reward=sc[k].goal_reward,
                           wall_height=sc[k].wall_height, agent_height=sc[k].agent_height,
                           initial_life=sc[k].initial_life, max_life=sc[k].max_life, food_rewards=food[k],
                           food_interval=itv[k]) for k in range(K)]

    def sample_task(self, **kwargs):
        """Convenience: draw one task with the host sampler (reference usage: MazeTaskSampler(...), test.py:12)."""
        return MazeTaskSampler(**kwargs)

    def _out(self, t):
        return t[0] if self._squeeze else t

    def reset(self, mask=None):
        if self.need_set_task:
            raise Exception("Must call \"set_task\" before reset")                  # maze_env.py:49-50
        m = None
        if mask is not None:
            m = self._torch.as_tensor(mask, device=self.device).to(self._torch.uint8).contiguous()
        _lib.check(self._lib.mgb_maze_reset(self._h, _lib.ptr(m), self._obs.data_ptr(), self._stream()))
        self.need_reset = False
        return self._out(self._obs)

    def step(self, action=None, want_expert=False):
        """want_expert=True (an expert=True env): info["expert"] is the expert's action mask [N] uint8 of the state each
        env holds after the step, the one its next action acts on (mgb_maze_step_expert; a persistent buffer, so that
        the step can be captured in a CUDA graph)."""
        if want_expert:
            self._require_expert()
        if self.need_reset:
            raise Exception("Must \"reset\" before doing any actions")              # maze_env.py:60-61
        if action is None:
            raise NotImplementedError("keyboard control (action=None) is display-only in the reference")
        torch = self._torch
        act_dtype, shape = getattr(torch, self._ACT_DTYPE), (self.num_envs,) + self._ACT_SHAPE
        if not (hasattr(action, "is_cuda") and action.is_cuda):
            action = torch.as_tensor(np.asarray(action, dtype=self._ACT_HOST_DTYPE).reshape(shape), device=self.device)
        act = action
        if act.dtype is not act_dtype or not act.is_contiguous() or act.shape != shape:
            act = action.to(act_dtype).reshape(shape).contiguous()
        if self._own_ptrs is None or self._own_ptrs[0] != self._obs.data_ptr():
            self._own_ptrs = (self._obs.data_ptr(), self._rew.data_ptr(), self._done.data_ptr(),
                              _lib.ptr(self._final), _lib.ptr(self._trunc))
            self._done_bool = self._done.view(torch.bool)
        if want_expert:
            if self._exp is None:
                self._exp = torch.empty((self.num_envs,), dtype=torch.uint8, device=self.device)
            rc = self._lib.mgb_maze_step_expert(self._h, act.data_ptr(), *self._own_ptrs, self._exp.data_ptr(),
                                                self._stream())
        else:
            rc = self._lib.mgb_maze_step(self._h, act.data_ptr(), *self._own_ptrs, self._stream())
        if rc:
            _lib.check(rc)
        info = _LazySteps(self)
        if want_expert:
            info["expert"] = self._out(self._exp)
        return self._out(self._obs), self._out(self._rew), self._out(self._done_bool), info

    # step() and rollout(): the layout of one env's action, the numpy dtype host actions are read as (None: as given),
    # and whether the "act" output also records actions the caller passed in (or only device-drawn ones)
    _ACT_DTYPE, _ACT_SHAPE, _ACT_HOST_DTYPE = "int32", (), None
    _RECORDS_GIVEN_ACTIONS = True

    def _rollout(self, T, actions, act_seed, want_actions, out, final=False, resample=None):
        """mgb_maze_rollout.  final: also produce the "final_obs" / "truncated" entries.  resample: resample_tasks'
        keyword arguments with seed, to give finished envs a freshly drawn task in the same launch."""
        if self.need_reset:
            raise Exception("Must \"reset\" before doing any actions")
        torch = self._torch
        T, N, dev = int(T), self.num_envs, self.device
        act_dtype, act_shape = getattr(torch, self._ACT_DTYPE), (T, N) + self._ACT_SHAPE
        record = actions is None or self._RECORDS_GIVEN_ACTIONS
        if out is None:
            out = {"obs": torch.empty((T, N) + tuple(self._obs.shape[1:]), dtype=self._obs.dtype, device=dev),
                   "rew": torch.empty((T, N), dtype=torch.float64, device=dev),
                   "done": torch.empty((T, N), dtype=torch.uint8, device=dev),
                   "act": torch.empty(act_shape, dtype=act_dtype, device=dev) if want_actions and record else None}
            if final:
                out["final_obs"] = torch.empty((T, N) + tuple(self._obs.shape[1:]), dtype=self._obs.dtype, device=dev)
                out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
        a = None
        if actions is not None:
            a = torch.as_tensor(actions, dtype=act_dtype, device=dev).reshape(act_shape).contiguous()
        cfg, seed = (None, 0) if resample is None else self._sampler_cfg(**resample)
        self._trial_entries(out, resample)
        _lib.check(self._lib.mgb_maze_rollout(self._h, T, _lib.ptr(a), int(act_seed),
                                              _lib.ptr(out.get("act") if record else None), _lib.ptr(out.get("obs")),
                                              _lib.ptr(out.get("rew")), _lib.ptr(out.get("done")),
                                              _lib.ptr(out.get("final_obs") if final else None),
                                              _lib.ptr(out.get("truncated") if final else None),
                                              None if cfg is None else ctypes.byref(cfg), seed, self._stream()))
        return out

    def _require_expert(self):
        if not self.with_expert:
            raise ValueError("the expert needs an env created with expert=True")
        if self.need_set_task:
            raise Exception("Must call \"set_task\" before reset")

    def _expert_rollout(self, T, actions, eps, deterministic, act_seed, want_expert, out, final, resample):
        """mgb_maze_rollout_expert: rollout() with expert= or want_expert=True."""
        self._require_expert()
        if resample is not None:
            raise ValueError("expert rollouts do not resample in the launch (resample_tasks between rollouts instead)")
        if actions is not None and eps is not None:
            raise ValueError("rollout takes either actions or expert=eps, not both")
        if actions is None and eps is None:
            raise ValueError("want_expert=True without actions needs expert=eps to choose the actions")
        if eps is not None and not (math.isfinite(eps) and 0.0 <= eps <= 1.0):
            raise ValueError("expert=eps must be a finite mixing rate in [0, 1], got %r" % (eps,))
        if self.need_reset:
            raise Exception("Must \"reset\" before doing any actions")
        torch = self._torch
        T, N, dev = int(T), self.num_envs, self.device
        if out is None:
            out = {"obs": torch.empty((T, N) + tuple(self._obs.shape[1:]), dtype=self._obs.dtype, device=dev),
                   "rew": torch.empty((T, N), dtype=torch.float64, device=dev),
                   "done": torch.empty((T, N), dtype=torch.uint8, device=dev)}
            if actions is None:
                out["act"] = torch.empty((T, N), dtype=torch.int32, device=dev)
            out["expert"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
            if final:
                out["final_obs"] = torch.empty((T, N) + tuple(self._obs.shape[1:]), dtype=self._obs.dtype, device=dev)
                out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
        a = None
        if actions is not None:
            a = torch.as_tensor(actions, dtype=torch.int32, device=dev).reshape(T, N).contiguous()
        self._trial_entries(out, None)
        _lib.check(self._lib.mgb_maze_rollout_expert(
            self._h, T, _lib.ptr(a), float(0.0 if eps is None else eps), int(bool(deterministic)), int(act_seed),
            _lib.ptr(out.get("act") if a is None else None), _lib.ptr(out.get("expert")), _lib.ptr(out.get("obs")),
            _lib.ptr(out.get("rew")), _lib.ptr(out.get("done")), _lib.ptr(out.get("final_obs") if final else None),
            _lib.ptr(out.get("truncated") if final else None), self._stream()))
        return out

    def expert(self):
        """An expert=True env's expert on the state every env holds now (mgb_maze_expert): (mask [N] uint8, bit a set
        iff action a starts a shortest path to the goal; dist [N] int32, the fewest actions to the goal, 65535 where it
        cannot be reached).  Stream-ordered."""
        self._require_expert()
        torch = self._torch
        mask = torch.empty((self.num_envs,), dtype=torch.uint8, device=self.device)
        dist = torch.empty((self.num_envs,), dtype=torch.int16, device=self.device)
        _lib.check(self._lib.mgb_maze_expert(self._h, mask.data_ptr(), dist.data_ptr(), self._stream()))
        return self._out(mask), self._out(dist.to(torch.int32) & 0xFFFF)

    def expert_table(self, slots=None):
        """The expert's tables of task-table slots `slots` (None: every slot; mgb_maze_expert_table): (mask [K,P,n,n]
        uint8, dist [K,P,n,n] int32), P = 1 heading plane for MetaMaze2D and 4 (indexed by ori) for MetaMazeDiscrete3D,
        entry [k, ori, gx, gy]."""
        self._require_expert()
        torch = self._torch
        n, P = self._n_cells, 1 if self.KIND == 0 else 4
        sl = list(range(len(self.tasks))) if slots is None else [int(k) for k in np.asarray(slots).reshape(-1)]
        mask = torch.empty((len(sl), P, n, n), dtype=torch.uint8, device=self.device)
        dist = torch.empty((len(sl), P, n, n), dtype=torch.int16, device=self.device)
        if slots is None:
            _lib.check(self._lib.mgb_maze_expert_table(self._h, 0, len(sl), mask.data_ptr(), dist.data_ptr(),
                                                       self._stream()))
        else:
            for k, s in enumerate(sl):
                _lib.check(self._lib.mgb_maze_expert_table(self._h, s, 1, mask[k].data_ptr(), dist[k].data_ptr(),
                                                           self._stream()))
        return mask, dist.to(torch.int32) & 0xFFFF

    def _check_rollout_final(self, final_obs):
        """rollout(..., final_obs=True) of the 3-D envs: the constructor's rule, per call."""
        if final_obs and not self.auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True (without auto-reset obs already is the terminal frame)")
        return bool(final_obs)

    def agent_state(self):
        """-> (agent [N,4] int32 = grid_x, grid_y, ori_index, steps ; life [N] float64)."""
        torch = self._torch
        ag = torch.empty((self.num_envs, 4), dtype=torch.int32, device=self.device)
        life = torch.empty((self.num_envs,), dtype=torch.float64, device=self.device)
        _lib.check(self._lib.mgb_maze_state(self._h, ag.data_ptr(), life.data_ptr(), self._stream()))
        return ag, life

    @property
    def launch_count(self):
        return int(self._lib.mgb_maze_launch_count(self._h)) if self._h else 0

    def _env_index(self, envs):
        """envs -> (int32 CUDA tensor or None for all envs, K).  A host sequence is range-checked; a CUDA tensor is moved
        to the env's device unchecked (no host synchronisation)."""
        if envs is None:
            return None, self.num_envs
        if hasattr(envs, "is_cuda") and envs.is_cuda:
            e = envs.to(device=self.device, dtype=self._torch.int32).reshape(-1).contiguous()
        else:
            idx = np.asarray(envs, dtype=np.int64).reshape(-1)
            if idx.size and (idx.min() < 0 or idx.max() >= self.num_envs):
                raise IndexError("env index out of range [0, %d)" % self.num_envs)
            e = self._torch.as_tensor(idx.astype(np.int32), device=self.device)
        return e, int(e.numel())

    def _require_path(self, what):
        if not self.record_path:
            raise ValueError("%s needs path recording: construct the env with record_path=True" % what)

    def god_view(self, envs=None, view_size=None, out=None, trajectory=False):
        """Top-down views of many envs in one launch (mgb_maze_god_view): the god panel of the reference window
        (render_init + render_update, maze_base.py:100-157): white floor, black walls, the ESCAPE goal in green, SURVIVAL
        food in (f, 255, f) with f = int(255 - 255 food), and the agent (2-D: red cell; 3-D: green disc and heading line).
        The text labels are not drawn.

        trajectory=True (needs record_path=True): the picture of the reference's save_trajectory() instead
        (MazeBase.render_trajectory, maze_base.py:159-189): walls and goal, a red rect at the agent's cell for every kind,
        SURVIVAL food over it, and red lines of width 3 between the centres of consecutive cells of the current episode's
        path.

        envs: local env indices (default: all), a host sequence (checked) or a CUDA tensor, moved to the env's device as
        int32 (not checked: an index out of range gives an all-zero frame; no host synchronisation, so the call can be
        captured in a CUDA graph).
        view_size: the panel's side S in pixels (default: the constructor's render_scale).  Returns (or fills `out`) a
        CUDA uint8 tensor [K, S, S, 3] with image rows top to bottom, as a saved picture shows it: out[k, y, x] is pixel
        (x, y) of the panel, so it is transposed against the x-major 3-D observations."""
        if self.need_set_task:
            raise Exception("Must call \"set_task\" before reset")
        if trajectory:
            self._require_path("god_view(trajectory=True)")
        torch = self._torch
        S = self.render_scale if view_size is None else view_size
        if int(S) != S or not 1 <= int(S) <= 4096:
            raise ValueError("view_size must be an integer in [1, 4096], got %r" % (view_size,))
        S = int(S)
        e, K = self._env_index(envs)
        if out is None:
            out = torch.empty((K, S, S, 3), dtype=torch.uint8, device=self.device)
        elif (tuple(out.shape) != (K, S, S, 3) or out.dtype != torch.uint8 or out.device != self.device
              or not out.is_contiguous()):
            raise ValueError("out must be a contiguous uint8 tensor of shape %s on %s" % ((K, S, S, 3), self.device))
        _lib.check(self._lib.mgb_maze_god_view(self._h, K, _lib.ptr(e), S, 1 if trajectory else 0, _lib.ptr(out),
                                               self._stream()))
        return out

    def trajectory(self, envs=None):
        """The current episode's path of each env (record_path=True): MazeBase._agent_trajectory, the start cell and the
        agent's cell after every step since the last reset (maze_base.py:44,67).  envs as for god_view().  Returns CUDA
        tensors (cells int32 [K, max_steps + 1, 2] = (grid_x, grid_y), -1 past each env's length; lengths int32 [K]),
        without a host synchronisation.  An env without auto-reset stepped on past max_steps keeps max_steps + 1 cells."""
        if self.need_set_task:
            raise Exception("Must call \"set_task\" before reset")
        self._require_path("trajectory()")
        torch = self._torch
        e, K = self._env_index(envs)
        cap = int(self.max_steps) + 1
        cells = torch.empty((K, cap, 2), dtype=torch.int8, device=self.device)
        lens = torch.empty((K,), dtype=torch.int32, device=self.device)
        _lib.check(self._lib.mgb_maze_path(self._h, K, _lib.ptr(e), _lib.ptr(cells), _lib.ptr(lens), self._stream()))
        valid = torch.arange(cap, device=self.device)[None, :, None] < lens[:, None, None]
        return torch.where(valid, cells.to(torch.int32), torch.full_like(cells, -1, dtype=torch.int32)), lens

    def save_trajectory(self, file_name, envs=None):
        """The reference's save_trajectory(file_name) (maze_env.py:82,152; MazeBase.render_trajectory): PNG files of
        god_view(trajectory=True) at render_scale.  With num_envs == 1 and squeeze the file is `file_name`; otherwise
        one file per selected env (envs: host indices, default all), <file_name without extension>_<env index>.png.
        Returns the list of files written."""
        return self._save_trajectory(file_name, envs, None)

    def _save_trajectory(self, file_name, envs, additional):
        import os
        from .png import write_png
        idx = list(range(self.num_envs)) if envs is None else [int(v) for v in np.asarray(envs).reshape(-1)]
        frames = self.god_view(envs=idx, trajectory=True).cpu().numpy()
        if self._squeeze and envs is None:
            names, stems = [file_name], [file_name.split(".")[0]]       # the reference's names (maze_base.py:185,187)
        else:
            stem, _ = os.path.splitext(file_name)
            stems = ["%s_%d" % (stem, e) for e in idx]
            names = [s + ".png" for s in stems]
        written = []
        for name, base, panel in zip(names, stems, frames):
            if additional is None:
                write_png(name, panel)
                written.append(name)
                continue
            # render_trajectory with additional (maze_base.py:161-187): a white (S + aw) x max(S, ah) canvas, the panel
            # at (0, 0), each surface blitted at (S, 0) over the previous one and saved as stem + file_names[i] + ".png"
            surfaces = [np.asarray(s, dtype=np.uint8) for s in additional["surfaces"]]
            S = panel.shape[0]
            ah, aw = surfaces[0].shape[:2]
            canvas = np.full((max(S, ah), S + aw, 3), 255, dtype=np.uint8)
            canvas[:S, :S] = panel
            for surf, suffix in zip(surfaces, additional["file_names"]):
                h, w = min(surf.shape[0], canvas.shape[0]), min(surf.shape[1], aw)
                canvas[:h, S:S + w] = surf[:h, :w]
                out = base + suffix + ".png"
                write_png(out, canvas)
                written.append(out)
        return written

    def render(self, mode="human"):
        """mode="rgb_array": god_view() of every env at render_scale ([S, S, 3] for num_envs=1 with squeeze).  The
        reference's window (mode "human") needs a display, which the batched engine does not have."""
        if mode != "rgb_array":
            raise NotImplementedError("render(mode=%r): the batched engine is headless; use mode=\"rgb_array\"" % (mode,))
        return self._out(self.god_view())

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.mgb_maze_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _LazySteps(dict):
    """info = {"steps": n} (maze_env.py:73): fetched from the device only when somebody looks."""

    def __init__(self, env):
        dict.__init__(self)
        self._env = env

    def __missing__(self, k):
        if k != "steps":
            raise KeyError(k)
        ag, _ = self._env.agent_state()
        v = ag[:, 3]
        self[k] = v[0] if self._env._squeeze else v
        return self[k]

    def __contains__(self, k):
        return k == "steps" or dict.__contains__(self, k)


def _check_policy(env, policy, state):
    """The checks of every policy launch of the MetaMaze2D handle `env` (rollout, evaluate), made before anything
    reaches the device: the kind, the input width, the device, the carried state and a population's envs per member.
    Returns (recurrent, population)."""
    from .policy import GRUPolicy, LSTMPolicy, PolicyPopulation
    torch = env._torch
    N, dev = env.num_envs, env.device
    population = isinstance(policy, PolicyPopulation)
    recurrent = isinstance(policy, (GRUPolicy, LSTMPolicy)) or (population and policy.recurrent)
    if recurrent and state is None:
        raise ValueError("a %s rollout needs its carried state (state=policy.initial_state(num_envs))"
                         % type(policy).__name__)
    if state is not None and not recurrent:
        raise ValueError("state= goes with a GRUPolicy or an LSTMPolicy")
    if recurrent and policy.dist != "categorical":
        raise ValueError("a Gaussian recurrent policy drives the quadrotor; MetaMaze2D takes dist=\"categorical\"")
    if env.need_reset:
        raise Exception("Must \"reset\" before doing any actions")
    if population:
        policy.check_envs(N, _lib.MAZE2D_POLICY_CTA_ENVS)
    D = int(np.prod(env._obs.shape[1:]))
    if policy.obs_dim != D:
        raise ValueError("the policy takes %d observation inputs, the env observes %d" % (policy.obs_dim, D))
    if policy.params.device != dev:
        raise ValueError("the policy's buffer is on %s, the env on %s" % (policy.params.device, dev))
    if recurrent and not (isinstance(state, torch.Tensor) and state.dtype == torch.float32 and state.device == dev
                          and tuple(state.shape) == (N, policy.state_dim) and state.is_contiguous()):
        raise ValueError("state must be a contiguous float32 tensor [%d, %d] on %s" % (N, policy.state_dim, dev))
    return recurrent, population


class BatchedMetaMaze2D(_BatchedMazeBase, Mirrored):
    """MetaMaze2D(enable_render, render_scale, max_steps, task_type, view_grid) x num_envs (maze_env.py:155-172).

    episodes_per_task=k (all three maze kinds; default None: no trials) makes a trial handle for RL^2: each env counts
    the episodes it finishes on its current maze (task_episodes), and a rollout with resample= gives a finished env a
    new maze only when that episode was its k-th there; the others restart on the same maze, and a recurrent policy
    with hidden_reset="task" keeps its state across them.  k = 1 behaves exactly like None.  Without resample= step()
    and rollout() only count; combine task_episodes with resample_tasks(mask) to re-task from the host.  k is fixed for
    the handle's life; a trial handle's snapshot records are 16 bytes longer and restore only into a handle with the
    same k."""
    KIND = 0
    _MIRROR_PREFIX = "mgb_maze"

    def __init__(self, enable_render=False, render_scale=480, max_steps=5000, task_type="SURVIVAL", view_grid=2,
                 num_envs=1, device=0, auto_reset=False, env_index_base=0, squeeze=True, final_obs=False,
                 record_path=False, episodes_per_task=None, expert=False):
        if enable_render:
            raise NotImplementedError("enable_render=True needs a display; the batched engine is headless")
        self.enable_render = False
        self.render_scale = int(render_scale)
        self.view_grid = int(view_grid)
        self._setup(num_envs, device, task_type, max_steps, auto_reset, env_index_base, squeeze, final_obs, record_path,
                    episodes_per_task, expert)
        w = 2 * self.view_grid + 1
        # the reference declares Box(-1, 1, (3,3), int32) but returns float32 (2g+1)^2 arrays (maze_2d.py:92)
        self.observation_space = Box(low=-1, high=1, shape=(w, w), dtype=np.float32)
        self._obs = self._torch.empty((self.num_envs, w, w), dtype=self._torch.float32, device=self.device)
        self._alloc_final()

    def _make_cfg(self, n_cells):
        cfg = _lib.MazeCfg()
        cfg.kind, cfg.task_type = 0, {"SURVIVAL": 0, "ESCAPE": 1}[self.task_type]
        cfg.n_cells, cfg.max_steps, cfg.view_grid = n_cells, self.max_steps, self.view_grid
        return cfg

    def rollout(self, T, actions=None, act_seed=0, want_actions=False, out=None, resample=None, policy=None,
                deterministic=False, state=None, want_hidden=False, gae=None, expert=None, want_expert=False):
        """T steps in one launch (mgb_maze_rollout).  actions: [T,N] int32 CUDA tensor or None (device-drawn uniform
        {0..3}).  Returns dict(obs [T,N,<obs of one env>], rew [T,N] f64, done [T,N] u8, act [T,N] i32 or None).

        With final_obs=True the dict also holds "final_obs" [T,N,<obs of one env>] float32: row (t, e) is the
        terminal window of env e where done[t, e] (what step() reports as final_observation); it is allocated with
        torch.empty, and rows with done 0 are not written, so they hold whatever the buffer held.  And "truncated"
        [T,N] uint8, written for every step: 1 iff done and the episode ended only through max_steps.  A
        caller-supplied `out` may omit either entry, and that output is then not produced.

        resample: None, or resample_tasks' keyword arguments with its seed, e.g. dict(seed=5, crowd_ratio=0.35)
        Every env whose episode ends at step t then gets the maze resample_tasks(done,
        **resample) would give it, in the same launch: obs[t] is its first window on the new maze, final_obs[t] the
        terminal window on the old one.  Needs auto_reset=True and set_task() with one table slot per env, like
        resample_tasks; with n = 31 the view_grid may be at most 6.  On a trial handle (episodes_per_task=k) only an
        episode that is the env's k-th on its maze draws; new_tasks(out) marks where envs drew.

        A trial handle's dict also holds "task_episodes0" [N] int32 (task_episodes at launch start),
        "episodes_per_task" (k) and "resampled".

        policy: an MLPPolicy (metagym_b200.policy) with (2 view_grid + 1)^2 inputs whose four outputs are the logits of
        the actions (mgb_maze_rollout_policy): the action of step t is drawn from their softmax on the window before
        step t, with the Philox stream keyed by act_seed; deterministic=True takes the argmax.  Composes with
        `resample`.  The dict then also holds "act" [T,N] int32, "logp" [T,N] float32 (sampling only) and "obs0"
        [N,<obs of one env>] (the window acted on at t = 0; at t > 0 it is obs[t-1]).  `actions` together with
        `policy` is a ValueError.

        policy may also be a GRUPolicy or an LSTMPolicy (mgb_maze_rollout_rnn; needs auto_reset=True), with state:
        its carried state [N, policy.state_dim] float32 on the env's device (policy.initial_state(N) for fresh envs),
        read at the start and updated in place at the end of the launch.  The dict then also holds "state0" (a copy
        of state as read), "resampled" (whether the launch resampled, which unroll() needs for the "task" reset rule)
        and, with want_hidden=True, "hid" [T,N,H] (the cell's output at every step).

        policy may also be a PolicyPopulation of any of the three kinds (mgb_maze_rollout_population,
        mgb_maze_rollout_rnn_population): member m drives the envs [m E, (m + 1) E), E = N / members, which must be
        32, 64 or a multiple of 128; a recurrent population takes state= as its members would.

        A policy or population with a value head (value=nn.Linear(k, 1); mgb_maze_rollout_critic,
        mgb_maze_rollout_rnn_critic; needs auto_reset=True) also yields "value" [T,N] float32 (V on the input step t
        acts on), "value_last" [N] (V after the last step, with the carried state the launch leaves: the next launch's
        value[0]) and, with final_obs=True or gae, "final_value" [T,N]: V of the terminal window where an episode ended
        truncated and the policy's memory is wiped (every done, or new_tasks(out) under hidden_reset="task"), from the
        memory before the wipe; other entries are not written.  gae=(gamma, lam) also yields "adv" and "ret" [T,N]
        float32, GAE(gamma, lam) cut where the memory is wiped (DESIGN.md "Value heads and GAE").

        expert=eps (an env created with expert=True; mgb_maze_rollout_expert): the action of step t is the shortest-path
        expert's on the state before step t, mixed with uniform actions at rate eps; deterministic=True takes the lowest
        optimal action.  act_seed keys the expert's draws.  The dict also holds "act" [T,N] int32 and "expert" [T,N]
        uint8, the mask of optimal actions of the state each step acted on.  actions=a with want_expert=True steps the
        given actions and labels them.  The env side is bit for bit rollout(T, actions=out["act"]).  Not with resample
        or a policy."""
        if expert is not None or want_expert:
            if policy is not None:
                raise ValueError("rollout takes either a policy or the expert, not both")
            return self._expert_rollout(T, actions, expert, deterministic, act_seed, want_expert, out, self._want_final,
                                        resample)
        if policy is not None:
            if actions is not None:
                raise ValueError("rollout takes either actions or a policy, not both")
            recurrent, population = _check_policy(self, policy, state)
            return self._rollout_policy(T, policy, recurrent, population, state, act_seed, deterministic, out, resample,
                                        want_hidden, gae)
        if state is not None:
            raise ValueError("state= goes with a GRUPolicy or an LSTMPolicy")
        if gae is not None:
            raise ValueError("gae= needs a policy with a value head")
        return self._rollout(T, actions, act_seed, want_actions, out, final=self._want_final, resample=resample)

    def evaluate(self, policy, episodes=1, act_seed=0, deterministic=False, state=None, resample=None):
        """Whole-episode evaluation in one launch (mgb_maze_evaluate; DESIGN.md "Whole-episode evaluation"): every env
        steps under `policy` until its `episodes`-th done, then stops.  Step t is, bit for bit, step t of
        rollout(T, policy=policy, act_seed=act_seed, deterministic=deterministic, state=state, resample=resample),
        with its auto-reset, in-launch resampling, trial counting and path recording, and each env is left as such a
        rollout of its own length leaves it (state, if given, included), so successive calls score consecutive
        episodes.  Episode 0 counts from the state the env holds now: reset() first for clean episodes.  policy is any
        policy rollout() takes, including populations and policies with a value head (never evaluated).  Needs
        auto_reset=True.  The step counter advances by episodes * max_steps.  On a trial handle (episodes_per_task=k,
        with resample and hidden_reset="task") res["return"].mean(1) is the adaptation curve over a trial's episodes.

        Returns {"return": [episodes, N] float64 (the rewards of each episode summed in step order), "length":
        [episodes, N] int32 (its steps; zero-filled first, so an episode the launch did not finish, which the time limit
        rules out, would show as length 0), "truncated": [episodes, N] uint8 (1 iff it ended through max_steps alone)}.
        A population's fitness, member by member: res["return"].mean(0).view(M, -1).mean(1)."""
        recurrent, population = _check_policy(self, policy, state)
        episodes = int(episodes)
        if episodes < 1 or episodes * self.max_steps > 2 ** 31 - 1:
            raise ValueError("episodes must be at least 1, and episodes * max_steps at most 2^31 - 1 steps")
        torch = self._torch
        shape = (episodes, self.num_envs)
        out = {"return": torch.empty(shape, dtype=torch.float64, device=self.device),
               "length": torch.zeros(shape, dtype=torch.int32, device=self.device),
               "truncated": torch.empty(shape, dtype=torch.uint8, device=self.device)}
        cfg, seed = (None, 0) if resample is None else self._sampler_cfg(**resample)
        pol = ctypes.byref(policy.struct(deterministic))
        members, stride = (policy.members, policy.member_stride) if population else (1, 0)
        mlp, rnn = (None, pol) if recurrent else (pol, None)
        _lib.check(self._lib.mgb_maze_evaluate(self._h, episodes, mlp, rnn,
                                               int(policy.has_value), members, stride, int(act_seed),
                                               None if cfg is None else ctypes.byref(cfg), seed, _lib.ptr(state),
                                               *[_lib.ptr(out[k]) for k in ("return", "length", "truncated")],
                                               self._stream()))
        return out

    def _rollout_policy(self, T, policy, recurrent, population, state, act_seed, deterministic, out, resample,
                        want_hidden, gae=None):
        from .policy import critic_args, critic_struct
        torch = self._torch
        T, N, dev = int(T), self.num_envs, self.device
        shape = tuple(self._obs.shape[1:])
        critic = critic_args(policy, gae)
        if out is None:
            out = {"obs": torch.empty((T, N) + shape, dtype=torch.float32, device=dev),
                   "rew": torch.empty((T, N), dtype=torch.float64, device=dev),
                   "done": torch.empty((T, N), dtype=torch.uint8, device=dev),
                   "act": torch.empty((T, N), dtype=torch.int32, device=dev),
                   "logp": None if deterministic else torch.empty((T, N), dtype=torch.float32, device=dev),
                   "obs0": torch.empty((N,) + shape, dtype=torch.float32, device=dev)}
            if recurrent:
                out["state0"] = torch.empty((N, policy.state_dim), dtype=torch.float32, device=dev)
            if recurrent and want_hidden:
                out["hid"] = torch.empty((T, N, policy.hidden), dtype=torch.float32, device=dev)
            if self._want_final:
                out["final_obs"] = torch.empty((T, N) + shape, dtype=torch.float32, device=dev)
                out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
        if recurrent:
            out["resampled"] = resample is not None
        cfg, seed = (None, 0) if resample is None else self._sampler_cfg(**resample)
        self._trial_entries(out, resample)
        pol = policy.struct(deterministic)
        tail = []
        if critic is not None:
            tail = [ctypes.byref(critic_struct(torch, out, T, N, dev, critic, self._want_final))]
            members = [policy.members, policy.member_stride] if population else [1, 0]
            entry = self._lib.mgb_maze_rollout_rnn_critic if recurrent else self._lib.mgb_maze_rollout_critic
        elif population:
            members = [policy.members, policy.member_stride]
            entry = self._lib.mgb_maze_rollout_rnn_population if recurrent else self._lib.mgb_maze_rollout_population
        else:
            members = []
            entry = self._lib.mgb_maze_rollout_rnn if recurrent else self._lib.mgb_maze_rollout_policy
        args = [self._h, T, ctypes.byref(pol)] + members
        args += [int(act_seed), None if cfg is None else ctypes.byref(cfg), seed]
        if recurrent:
            args += [_lib.ptr(state), _lib.ptr(out.get("state0")), _lib.ptr(out.get("hid"))]
        keys = ("act", "logp", "obs0", "obs", "rew", "done", "final_obs", "truncated")
        _lib.check(entry(*args, *[_lib.ptr(out.get(k)) for k in keys], *tail, self._stream()))
        return out

    def save_trajectory(self, file_name, envs=None, additional=None):
        """MetaMaze2D.save_trajectory(file_name, additional) (maze_env.py:211-212), file names as for the 3-D envs.
        additional = {"surfaces": [uint8 [H, W, 3] images], "file_names": [suffixes]}: each surface is placed right of the
        panel on a white (S + W) x max(S, H) canvas (W, H of the first surface), and the canvas is saved as the file
        name before its first "." + file_names[i] + ".png", as the reference does."""
        return self._save_trajectory(file_name, envs, additional)


class BatchedMetaMazeDiscrete3D(_BatchedMazeBase):
    """MetaMazeDiscrete3D(enable_render, render_scale, resolution, max_steps, task_type) x num_envs
    (maze_env.py:16-42).  obs_dtype: 'int32' = exact reference values (what the reference's array holds), 'float32' = the
    same values in the dtype the reference's observation_space declares (maze_env.py:37-39), 'uint8' = min(value, 255).
    textures: (grounds uint8 [n_tex,64,64,3], ceil uint8 [64,64,3]); default = procedural set."""
    KIND = 1

    def __init__(self, enable_render=False, render_scale=480, resolution=(320, 320), max_steps=5000,
                 task_type="SURVIVAL", num_envs=1, device=0, auto_reset=False, env_index_base=0, squeeze=True,
                 obs_dtype="int32", textures=None, max_vision_range=12.0, fol_angle=0.6 * PI, cache=None,
                 final_obs=False, record_path=False, episodes_per_task=None, expert=False):
        if enable_render:
            raise NotImplementedError("enable_render=True needs a display; the batched engine is headless")
        self.enable_render = False
        self.render_scale = int(render_scale)
        self.resolution = (int(resolution[0]), int(resolution[1]))
        assert obs_dtype in ("int32", "uint8", "float32")
        self.obs_dtype = obs_dtype
        self.max_vision_range, self.fol_angle = max_vision_range, fol_angle
        self.cache = cache                  # None: library default (on, MGB_MAZE_CACHE); False: direct renderer only
        self.textures = textures if textures is not None else synthetic_textures(seed=0)
        self._setup(num_envs, device, task_type, max_steps, auto_reset, env_index_base, squeeze, final_obs, record_path,
                    episodes_per_task, expert)
        torch = self._torch
        h, v = self.resolution
        self.observation_space = Box(low=0, high=256, shape=(h, v, 3), dtype=np.float32)     # maze_env.py:37-39
        self._obs = torch.empty((self.num_envs, h, v, 3), device=self.device,
                                dtype={"int32": torch.int32, "uint8": torch.uint8, "float32": torch.float32}[obs_dtype])
        self._alloc_final()

    def _make_cfg(self, n_cells):
        cfg = _lib.MazeCfg()
        cfg.kind, cfg.task_type = 1, {"SURVIVAL": 0, "ESCAPE": 1}[self.task_type]
        cfg.n_cells, cfg.max_steps, cfg.view_grid = n_cells, self.max_steps, 0
        cfg.res_h, cfg.res_v = self.resolution
        cfg.obs_dtype = {"uint8": 0, "int32": 1, "float32": 2}[self.obs_dtype]
        cfg.max_vision, cfg.fov = self.max_vision_range, self.fol_angle       # maze_discrete_3d.py:22-23
        cfg.l_focal, cfg.text_size = 0.20, 1.0                                # maze_discrete_3d.py:116
        return cfg

    def rollout(self, T, actions=None, act_seed=0, want_actions=False, out=None, final_obs=False, resample=None,
                expert=None, deterministic=False, want_expert=False):
        """T steps in one launch: obs [T,N,res_h,res_v,3] (uint8, int32 or float32), rew, done, act as for
        BatchedMetaMaze2D.rollout (mgb_maze_rollout).  Runs on the pose cache when it is in use, otherwise (an env created
        with cache=False, or when `resample` is given) on the direct raycaster; both give the same results.

        final_obs (per call, independent of the constructor's final_obs, which concerns step()): False returns only the
        entries above.  True needs auto_reset=True (ValueError otherwise), and the dict also holds "final_obs"
        [T,N,res_h,res_v,3] in the obs dtype, where row (t, e) is the terminal frame of env e if done[t, e] (what
        step() reports as final_observation; allocated with torch.empty, rows with done 0 are not written), and
        "truncated" [T,N] uint8, written for every step: 1 iff done and the episode ended only through max_steps.  A
        caller-supplied `out` may omit either entry, and that output is then not produced.

        resample: None, or resample_tasks' keyword arguments with its seed, e.g. dict(seed=5, crowd_ratio=0.35).  Every
        env whose episode ends at step t then gets the maze resample_tasks(done, **resample) would give it, in the same
        launch: obs[t] is its first frame on the new maze, final_obs[t] the terminal frame on the old one.  Needs
        auto_reset=True, cache=False and set_task() with one table slot per env, like resample_tasks.  Trial handles
        (episodes_per_task=k): as for BatchedMetaMaze2D.rollout.

        expert=eps, deterministic, want_expert (an env created with expert=True): as for BatchedMetaMaze2D.rollout, on
        the pose cache and on the direct renderer alike."""
        if expert is not None or want_expert:
            return self._expert_rollout(T, actions, expert, deterministic, act_seed, want_expert, out,
                                        self._check_rollout_final(final_obs), resample)
        return self._rollout(T, actions, act_seed, want_actions, out, final=self._check_rollout_final(final_obs),
                             resample=resample)

    def cache_info(self):
        """Pose-cache statistics (valid after the first reset()/step(); synchronises the device): dict(poses, variant_frames, variant_bits, bytes,
        poses_by_food_count [k = 0..7, >= 8], in_use), and the shared-memory plan of the last direct-renderer launch
        (hits_in_global: crossing lists in a global scratch; pipelined: geometry of the next env under the pixels)."""
        out = (ctypes.c_int64 * 16)()
        _lib.check(self._lib.mgb_maze_cache_info(self._h, out))
        return {"poses": int(out[0]), "variant_frames": int(out[1]), "variant_bits": int(out[2]), "bytes": int(out[3]),
                "poses_by_food_count": [int(out[4 + k]) for k in range(9)], "in_use": bool(out[13]),
                "hits_in_global": bool(out[14]), "pipelined": bool(out[15])}

    def _after_create(self):
        if self.cache is not None:
            _lib.check(self._lib.mgb_maze_set_cache(self._h, int(bool(self.cache))))
        grounds = np.ascontiguousarray(self.textures[0], dtype=np.uint8)
        ceil = np.ascontiguousarray(self.textures[1], dtype=np.uint8)
        ts = grounds.shape[1]
        assert grounds.shape[1:] == (ts, ts, 3) and ceil.shape == (ts, ts, 3)
        _lib.check(self._lib.mgb_maze_set_textures(self._h, grounds.ctypes.data, grounds.shape[0], ceil.ctypes.data,
                                                   ts))


class BatchedMetaMazeContinuous3D(BatchedMetaMazeDiscrete3D):
    """MetaMazeContinuous3D(enable_render, render_scale, resolution, max_steps, task_type) x num_envs
    (maze_env.py:85-153).  Actions [N, 2] float32 = (turn_rate, walk_speed) in [-1, 1] (clipped like the reference,
    maze_continuous_3d.py:48-49); float32 position / float64 heading exactly as the reference computes them for
    float32 actions.  Every pose is unique, so this env always uses the direct float64 renderer."""
    KIND = 2
    _ACT_DTYPE, _ACT_SHAPE, _ACT_HOST_DTYPE = "float32", (2,), np.float32
    _RECORDS_GIVEN_ACTIONS = False

    def __init__(self, *args, **kwargs):
        BatchedMetaMazeDiscrete3D.__init__(self, *args, **kwargs)
        self.action_space = Box(low=np.array([-1.0, -1.0]), high=np.array([1.0, 1.0]), dtype=np.float32)

    def _make_cfg(self, n_cells):
        cfg = BatchedMetaMazeDiscrete3D._make_cfg(self, n_cells)
        cfg.kind = 2
        return cfg

    def rollout(self, T, actions=None, act_seed=0, want_actions=False, out=None, final_obs=False, resample=None):
        """T steps in one launch of the direct renderer (mgb_maze_rollout), exactly as T step() calls.
        actions: anything reshapeable to [T,N,2] (turn_rate, walk_speed), clipped to [-1, 1] like step(); None draws them
        on the device, uniform on [-1, 1) like action_space.sample().  Returns dict(obs [T,N,res_h,res_v,3] in the env's
        obs dtype, rew [T,N] f64, done [T,N] u8, act [T,N,2] f32: the drawn actions when want_actions, else None).

        final_obs (per call, independent of the constructor's final_obs, which concerns step()): True needs
        auto_reset=True (ValueError otherwise), and the dict also holds "final_obs" [T,N,res_h,res_v,3] in the obs
        dtype, where row (t, e) is the terminal frame of env e if done[t, e] (allocated with torch.empty, rows with done
        0 are not written), and "truncated" [T,N] uint8, written for every step.  A caller-supplied `out` may omit either
        entry, and that output is then not produced.

        resample: as for BatchedMetaMazeDiscrete3D.rollout: every env whose episode ends at step t gets a freshly drawn
        maze in the same launch, and obs[t] is its first frame on it."""
        return self._rollout(T, actions, act_seed, want_actions, out, final=self._check_rollout_final(final_obs),
                             resample=resample)

    def pose(self):
        """-> (pos [N,2] float32 = _agent_loc, ori [N] float64 = _agent_ori)."""
        torch = self._torch
        pos = torch.empty((self.num_envs, 2), dtype=torch.float32, device=self.device)
        ori = torch.empty((self.num_envs,), dtype=torch.float64, device=self.device)
        _lib.check(self._lib.mgb_maze_pose(self._h, pos.data_ptr(), ori.data_ptr(), self._stream()))
        return pos, ori


MetaMaze2D = BatchedMetaMaze2D
MetaMazeDiscrete3D = BatchedMetaMazeDiscrete3D
MetaMazeContinuous3D = BatchedMetaMazeContinuous3D

