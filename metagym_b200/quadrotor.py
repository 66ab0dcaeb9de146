"""Batched drop-in for metagym.quadrotor.Quadrotor (reference: metagym/quadrotor/env.py:30-305).

Same constructor kwargs, method names and return conventions as the reference env, with a leading batch axis over
`num_envs` independent instances whose state lives in H100 HBM and is advanced by libmgb200's hand-written kernels
(metagym_b200/csrc/quad.cu).  Host code here only parses the config, owns the output tensors and forwards pointers.
"""
import ctypes
import json
import os

import numpy as np

from . import _lib
from .rollout import Mirrored
from .snapshot import Snapshots
from .spaces import Box, Space

TASKS = {"no_collision": 0, "hovering_control": 1, "velocity_control": 2}

# Default physical parameters -- the numbers of the reference's metagym/quadrotor/config.json:1-59.  A user can pass
# `simulator_conf=<path>` to load a different file with the same schema (env.py:57-61).
DEFAULT_SIMULATOR_CONF = {
    "precision": 0.001, "quality": 0.5,
    "inertia": {"xx": 0.0135, "xy": 0.0, "xz": 0.0, "yy": 0.0135, "yz": 0.0, "zz": 0.024},
    "drag": {"m_xx": 0.074, "m_yy": 0.074, "m_zz": 0.0506, "f_xx": 0.12, "f_yy": 0.12, "f_zz": 0.10},
    "gravity_center": {"x": 0.0, "y": 0.0, "z": 0.0},
    "thrust": {"CT": ["1.538e-5", "-2.5e-4", "0.0"], "Mm": "0.010", "Jm": "2.573e-4", "RA": "0.2010",
               "phi": "0.017242179827506"},
    "propeller": [{"x": 0.18, "y": 0.18, "z": 0.0}, {"x": -0.18, "y": 0.18, "z": 0.0},
                  {"x": -0.18, "y": -0.18, "z": 0.0}, {"x": 0.18, "y": -0.18, "z": 0.0}],
    "fail": {"velocity": 100.0, "w": 1000.0, "range": 1000.0},
    "electric": {"min_voltage": 0.10, "max_voltage": 15.0},
    "init_velocity": {"x": 0, "y": 0, "z": 0, "noisy": 2.0},
    "init_angular_velocity": {"x": 0, "y": 0, "z": 0, "noisy": 5.0},
}

OBS_KEYS = ["b_v_x", "b_v_y", "b_v_z", "b_x", "b_y", "b_z", "acc_x", "acc_y", "acc_z", "gyro_x", "gyro_y", "gyro_z",
            "pitch", "roll", "yaw", "z"]                       # env.py:77-83,193-197
VELOCITY_KEYS = ["next_target_g_v_x", "next_target_g_v_y", "next_target_g_v_z"]  # env.py:83-84


def load_simulator_conf(simulator_conf=None):
    """QuadrotorSim.get_config (quadrotorsim.py:223-237): returns the parsed dict."""
    if simulator_conf is None:
        return json.loads(json.dumps(DEFAULT_SIMULATOR_CONF))
    if isinstance(simulator_conf, dict):
        return simulator_conf
    assert os.path.exists(simulator_conf), "Simulator config file does not exist"   # env.py:60-61
    with open(simulator_conf, "r") as f:
        return json.load(f)


def build_cfg(conf, dt, nt, task, healthy_reward, integrator="euler", rk4_steps=1):
    """QuadrotorSim._parse_cfg (quadrotorsim.py:50-109) -> mgb_quad_cfg.  Raises RuntimeError like get_config."""
    try:
        c = _lib.QuadCfg()
        c.precision = float(conf["precision"])
        c.quality = float(conf["quality"])
        ine = conf["inertia"]
        inertia = np.array([[ine["xx"], ine["xy"], ine["xz"]], [ine["xy"], ine["yy"], ine["yz"]],
                            [ine["xz"], ine["yz"], ine["zz"]]], dtype=np.float64).astype(np.float32)
        c.inv_inertia[:] = [float(x) for x in np.linalg.inv(inertia).reshape(-1)]
        d = conf["drag"]
        c.drag_m[:] = [float(d[k]) for k in ("m_xx", "m_yy", "m_zz")]
        c.drag_f[:] = [float(d[k]) for k in ("f_xx", "f_yy", "f_zz")]
        c.gravity_center[:] = [float(conf["gravity_center"][k]) for k in "xyz"]
        th = conf["thrust"]
        c.ct[:] = [float(x) for x in th["CT"]]
        c.mm, c.jm, c.phi, c.ra = float(th["Mm"]), float(th["Jm"]), float(th["phi"]), float(th["RA"])
        c.fail_velocity = float(conf["fail"]["velocity"])
        c.fail_range = float(conf["fail"]["range"])
        c.fail_w = float(conf["fail"]["w"])
        prop = np.array([[q["x"], q["y"], q["z"]] for q in conf["propeller"]], dtype=np.float64).astype(np.float32)
        assert prop.shape == (4, 3)
        c.propeller[:] = [float(x) for x in prop.reshape(-1)]
        c.propeller_norm[:] = [float(np.linalg.norm(prop[i])) for i in range(4)]
        c.min_voltage = float(conf["electric"]["min_voltage"])
        c.max_voltage = float(conf["electric"]["max_voltage"])
        iv = conf.get("init_velocity", {"x": 0, "y": 0, "z": 0, "noisy": 0.0})
        iw = conf.get("init_angular_velocity", {"x": 0, "y": 0, "z": 0, "noisy": 0.0})
        c.init_velocity[:] = [float(iv[k]) for k in "xyz"]
        c.init_velocity_noise = float(iv["noisy"])
        c.init_angular_velocity[:] = [float(iw[k]) for k in "xyz"]
        c.init_angular_velocity_noise = float(iw["noisy"])
    except Exception as e:
        raise RuntimeError("Error in loading configuration: " + str(e))
    c.dt = float(dt)
    c.nt = int(nt)
    c.task = TASKS[task]
    c.healthy_reward = float(healthy_reward)
    # env.py:97-114: the flat map starts the vehicle 5 m above the floor; velocity_control has no map/offset
    c.z_offset = 0.0 if task == "velocity_control" else 5.0
    assert integrator in ("euler", "rk4"), "integrator must be 'euler' (the reference's substeps) or 'rk4'"
    c.integrator = 0 if integrator == "euler" else 1
    c.rk4_steps = int(rk4_steps)
    return c


def velocity_task_actions(conf, nt, seed):
    """The action table define_velocity_control_task draws (quadrotorsim.py:307,311-314): np.random.seed(seed), then
    nt draws of uniform(min_V, max_V, 4) cast to float32.  Uses a private RandomState (same MT19937 stream) so the
    caller's global numpy RNG is left alone -- the one intentional difference from the reference."""
    rs = np.random.RandomState(seed)
    lo, hi = float(conf["electric"]["min_voltage"]), float(conf["electric"]["max_voltage"])
    return rs.uniform(low=lo, high=hi, size=(nt, 4)).astype(np.float32)


class QuadInfo(dict):
    """`info` of Quadrotor.step (env.py:163-164): name -> [N] column view of the observation tensor, built lazily."""

    def __init__(self, obs, keys):
        dict.__init__(self)
        self._obs, self._keys = obs, keys

    def __missing__(self, k):
        if k not in self._keys:
            raise KeyError(k)
        v = self._obs[..., self._keys.index(k)]
        self[k] = v
        return v

    def __contains__(self, k):
        return k in self._keys

    def keys(self):
        return list(self._keys)


def _check_policy(env, policy, state, deterministic):
    """The checks of every policy launch of the quadrotor handle `env` (rollout, evaluate), made before anything reaches
    the device: the kind, the input width, the device, log_std, the carried state and a population's envs per member.
    Returns (recurrent, population)."""
    from .policy import GRUPolicy, LSTMPolicy, PolicyPopulation
    torch = env._torch
    N, D, dev = env.num_envs, env.obs_dim, env.device
    population = isinstance(policy, PolicyPopulation)
    recurrent = isinstance(policy, (GRUPolicy, LSTMPolicy)) or (population and policy.recurrent)
    if recurrent and policy.dist != "gaussian":
        raise ValueError("a categorical recurrent policy drives MetaMaze2D; the quadrotor takes "
                         "dist=\"gaussian\"")
    if recurrent and state is None:
        raise ValueError("a %s rollout needs its carried state (state=policy.initial_state(num_envs))"
                         % type(policy).__name__)
    if state is not None and not recurrent:
        raise ValueError("state= goes with a GRUPolicy or an LSTMPolicy")
    if population:
        policy.check_envs(N, _lib.QUAD_RNN_CTA_ENVS if recurrent else _lib.QUAD_POLICY_CTA_ENVS)
    if policy.obs_dim != D:
        raise ValueError("the policy takes %d inputs, the env observes %d" % (policy.obs_dim, D))
    if policy.params.device != dev:
        raise ValueError("the policy's buffer is on %s, the env on %s" % (policy.params.device, dev))
    if not deterministic and not policy.has_log_std:
        raise ValueError("a stochastic quadrotor policy needs log_std (or pass deterministic=True)")
    if recurrent and not (isinstance(state, torch.Tensor) and state.dtype == torch.float32 and state.device == dev
                          and tuple(state.shape) == (N, policy.state_dim) and state.is_contiguous()):
        raise ValueError("state must be a contiguous float32 tensor [%d, %d] on %s" % (N, policy.state_dim, dev))
    return recurrent, population


class BatchedQuadrotor(Snapshots, Mirrored):
    """`Quadrotor(dt, nt, seed, task, map_file, simulator_conf, healthy_reward)` x num_envs on one H100.

    Extra kwargs: num_envs, device (int or 'cuda:k'), auto_reset (finished envs restart inside the step launch),
    rng_seed (counter-based reset noise), env_index_base (global index of env 0, for multi-GPU sharding),
    squeeze (num_envs == 1 returns reference-shaped arrays), integrator ('euler' = the reference's 1 ms substeps,
    parity-checked; 'rk4' = classical RK4 with rk4_steps steps per env step, validated by convergence only).
    velocity_control: `seed` may be an int (as in the reference) or a sequence of seeds = distinct tasks; env i
    flies task `env2task[i]` (default i % n_tasks).
    final_obs=True (needs auto_reset=True): every step() also reports `truncated`, and rollout() also returns the
    terminal observations and truncation flags of its steps.
    snapshot() / restore() / clone_envs(): exact checkpoint and resume of the whole env state -- rigid body, ct, episode
    counter, velocity task and the rollout action counter -- also into another sharding (metagym_b200/snapshot.py).
    """
    metadata = {"render.modes": []}
    _SNAP_PREFIX = _MIRROR_PREFIX = "mgb_quad"
    _FINGERPRINT_PARTS = ("configuration (physics, dt, nt, task, integrator, auto_reset, rng_seed)", "obstacle map",
                          "velocity-target table", "record layout")

    def __init__(self, dt=0.01, nt=1000, seed=0, task="no_collision", map_file=None, simulator_conf=None,
                 healthy_reward=1.0, num_envs=1, device=0, auto_reset=False, rng_seed=0, env_index_base=0,
                 env2task=None, squeeze=True, integrator="euler", rk4_steps=1, final_obs=False, **kwargs):
        import torch
        assert task in ["velocity_control", "no_collision", "hovering_control"], "Invalid task setting"  # env.py:55
        if final_obs and not auto_reset:
            raise ValueError("final_obs=True needs auto_reset=True (without auto-reset obs already is the terminal frame)")
        self._want_final = bool(final_obs)
        self.dt, self.nt, self.task, self.healthy_reward = dt, nt, task, healthy_reward
        self.num_envs = int(num_envs)
        self._squeeze = bool(squeeze) and self.num_envs == 1
        self._torch = torch
        self.device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
        if self.device.type != "cuda":
            raise _lib.MgbError("metagym_b200 runs on CUDA devices only (no CPU fallback)")
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.MgbError("no CUDA device visible: metagym_b200 has no CPU fallback")
        dev_index = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.device = torch.device("cuda", dev_index)
        self.conf = load_simulator_conf(simulator_conf)
        self._cfg = build_cfg(self.conf, dt, nt, task, healthy_reward, integrator, rk4_steps)
        self.valid_range = self._cfg.fail_range
        lo, hi = self._cfg.min_voltage, self._cfg.max_voltage
        self.action_space = Box(low=np.array([lo] * 4, dtype="float32"), high=np.array([hi] * 4, dtype="float32"),
                                shape=[4])
        self.obs_keys = OBS_KEYS + (VELOCITY_KEYS if task == "velocity_control" else [])
        self.observation_space = Space(shape=[len(self.obs_keys)], dtype="float32")
        self.x_offset = self.y_offset = 0
        self.z_offset = self._cfg.z_offset
        self.map_matrix = None
        if task != "velocity_control":
            self.map_matrix = self.load_map(map_file)                # env.py:105-113
            y_offsets, x_offsets = np.where(self.map_matrix == -1)
            assert len(y_offsets) == 1
            self.y_offset, self.x_offset = int(y_offsets[0]), int(x_offsets[0])
        h = ctypes.c_void_p()
        _lib.check(self._lib.mgb_quad_create(ctypes.byref(h), self.num_envs, ctypes.byref(self._cfg), dev_index,
                                             int(env_index_base)))
        self._h = h
        self.obs_dim = self._lib.mgb_quad_obs_dim(self._h)
        self.auto_reset = bool(auto_reset)
        _lib.check(self._lib.mgb_quad_set_options(self._h, int(self.auto_reset), int(rng_seed)))
        N, D, dev = self.num_envs, self.obs_dim, self.device
        self._obs = torch.empty((N, D), dtype=torch.float32, device=dev)
        self._rew = torch.empty((N,), dtype=torch.float32, device=dev)
        self._done = torch.empty((N,), dtype=torch.uint8, device=dev)
        self._fail = torch.zeros((N,), dtype=torch.int32, device=dev)
        self._own_ptrs = None
        self._host_results = False            # True after a host-path step: fail_code / final_observation are numpy
        self._final_obs = torch.zeros((N, D), dtype=torch.float32, device=dev) if self.auto_reset else None
        # persistent, so that a step with final_obs=True can be captured in a CUDA graph
        self._trunc = torch.zeros((N,), dtype=torch.uint8, device=dev) if self._want_final else None
        # final_obs=True: steps and rollouts go through the *_ex entry points, which also take the truncated output
        ex = "_ex" if self._want_final else ""
        self._step_fn = getattr(self._lib, "mgb_quad_step" + ex)
        self._step_host_fn = getattr(self._lib, "mgb_quad_step_host" + ex)
        self._rollout_fn = getattr(self._lib, "mgb_quad_rollout" + ex)
        self._trunc_ptr = (self._trunc.data_ptr(),) if self._want_final else ()
        if self.map_matrix is not None and map_file is not None:
            m = np.ascontiguousarray(self.map_matrix, dtype=np.int32)
            _lib.check(self._lib.mgb_quad_set_map(self._h, m.ctypes.data, m.shape[0], m.shape[1]))
        if self.map_matrix is not None:
            self.map_matrix = self.map_matrix.copy()
            self.map_matrix[self.y_offset, self.x_offset] = 0         # env.py:113
        self.velocity_targets = None
        self.env_index_base = int(env_index_base)
        if task == "velocity_control":
            seeds = [seed] if np.isscalar(seed) else list(seed)
            self.set_velocity_tasks(seeds, env2task=env2task, env_index_base=env_index_base)

    # ------------------------------------------------------------------------------------------------------
    def _stream(self):
        return _lib.current_stream(self._torch, self.device)

    def set_velocity_tasks(self, seeds, env2task=None, env_index_base=0):
        """define_velocity_control_task (quadrotorsim.py:306-319) for every seed, integrated on the GPU."""
        torch = self._torch
        acts = np.stack([velocity_task_actions(self.conf, self.nt, s) for s in seeds])      # [K, nt, 4]
        act_dev = torch.from_numpy(acts).to(self.device)
        tbl = torch.empty((len(seeds), self.nt, 3), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mgb_quad_make_targets(self._h, act_dev.data_ptr(), len(seeds), tbl.data_ptr(),
                                                   self._stream()))
        if env2task is None:
            env2task = (np.arange(self.num_envs, dtype=np.int64) + int(env_index_base)) % len(seeds)
        e2t = torch.as_tensor(np.asarray(env2task, dtype=np.int32), device=self.device)
        assert e2t.numel() == self.num_envs
        torch.cuda.synchronize(self.device)
        _lib.check(self._lib.mgb_quad_set_targets(self._h, tbl.data_ptr(), len(seeds), e2t.data_ptr()))
        self.velocity_targets = tbl
        self.env2task = e2t

    def sample_task(self, seed):
        """[nt, 3] velocity-target table of `seed` (what the reference builds in its constructor for `seed`,
        quadrotorsim.py:306-319), integrated on the GPU; the env's current tasks are left untouched.  Use
        set_velocity_tasks(seeds) to install tables."""
        torch = self._torch
        acts = velocity_task_actions(self.conf, self.nt, seed)[None]
        act_dev = torch.from_numpy(np.ascontiguousarray(acts)).to(self.device)
        tbl = torch.empty((1, self.nt, 3), dtype=torch.float32, device=self.device)
        _lib.check(self._lib.mgb_quad_make_targets(self._h, act_dev.data_ptr(), 1, tbl.data_ptr(), self._stream()))
        torch.cuda.synchronize(self.device)
        return tbl[0]

    def set_task(self, seeds, env2task=None):
        """Install velocity-target tasks by seed (one seed or a list; env e gets seeds[e % len] unless env2task)."""
        seeds = [int(seeds)] if np.isscalar(seeds) else [int(x) for x in seeds]
        self.set_velocity_tasks(seeds, env2task=env2task, env_index_base=self.env_index_base)

    @staticmethod
    def load_map(map_file):
        """Quadrotor.load_map (env.py:293-305): None = 100x100 flat floor with the start at (50, 50); otherwise a text
        file of space-separated integer rows, -1 marking the start cell."""
        if map_file is None:
            flatten_map = np.zeros([100, 100], dtype=np.int32)
            flatten_map[50, 50] = -1
            return flatten_map
        rows = []
        with open(map_file, "r") as f:
            for line in f.readlines():
                rows.append([int(i) for i in line.split(" ")])
        return np.array(rows)

    def _out(self, t):
        return t[0] if self._squeeze else t

    def reset(self, mask=None, noise=None):
        """Quadrotor.reset (env.py:116-125).  mask: [N] bool/uint8 tensor (None = all).  noise: [N,12] float64 array
        of the np.random.random draws to replay (None = counter-based device noise)."""
        torch = self._torch
        m = None
        if mask is not None:
            m = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous()
        nz = None
        if noise is not None:
            nz = torch.as_tensor(np.asarray(noise, dtype=np.float64).reshape(self.num_envs, 12), device=self.device)
        _lib.check(self._lib.mgb_quad_reset(self._h, _lib.ptr(m), _lib.ptr(nz), self._obs.data_ptr(), self._stream()))
        return self._out(self._obs)

    def step(self, action, out=None):
        """Quadrotor.step (env.py:127-165) -> (obs [N,D], reward [N], done [N] bool, info).

        out: optional (obs, rew, done_u8) CUDA tensors to write into (e.g. slot t of a rollout buffer) instead of the
        env's own output tensors.

        A CUDA tensor action runs fully on the device (stream-ordered, no host sync).  A numpy / host action takes
        the host path (`mgb_quad_step_host`): copies in, steps, copies out, returns numpy arrays.
        """
        torch = self._torch
        if not (hasattr(action, "is_cuda") and action.is_cuda):
            return self._step_host(action)
        act = action
        self._host_results = False
        if act.dtype is not torch.float32 or not act.is_contiguous() or act.numel() != self.num_envs * 4:
            act = action.to(torch.float32).reshape(self.num_envs, 4).contiguous()
        if out is None:                       # the env's own output tensors: addresses and views are fixed
            if self._own_ptrs is None:
                self._own_ptrs = (self._obs.data_ptr(), self._rew.data_ptr(), self._done.data_ptr(),
                                  self._fail.data_ptr(), _lib.ptr(self._final_obs)) + self._trunc_ptr
                self._done_bool = self._done.view(torch.bool)
            p = self._own_ptrs
            obs, rew, done = self._obs, self._rew, None
        else:
            obs, rew, done = out
            p = (obs.data_ptr(), rew.data_ptr(), done.data_ptr(), self._fail.data_ptr(),
                 _lib.ptr(self._final_obs)) + self._trunc_ptr
        rc = self._step_fn(self._h, act.data_ptr(), *p, self._stream())
        if rc:
            _lib.check(rc)
        done_b = self._done_bool if done is None else done.view(torch.bool)
        info = QuadInfo(obs, self.obs_keys)
        return self._out(obs), self._out(rew), self._out(done_b), info

    def _step_host(self, action):
        act = np.ascontiguousarray(np.asarray(action, dtype=np.float32).reshape(self.num_envs, 4))
        if not hasattr(self, "_h_obs"):
            self._h_obs = np.empty((self.num_envs, self.obs_dim), dtype=np.float32)
            self._h_rew = np.empty((self.num_envs,), dtype=np.float32)
            self._h_done = np.empty((self.num_envs,), dtype=np.uint8)
            self._h_fail = np.zeros((self.num_envs,), dtype=np.int32)
            self._h_final = np.zeros((self.num_envs, self.obs_dim), dtype=np.float32) if self.auto_reset else None
            self._h_trunc = np.zeros((self.num_envs,), dtype=np.uint8) if self._want_final else None
            trunc = (self._h_trunc.ctypes.data,) if self._want_final else ()
            self._h_ptrs = (self._h_obs.ctypes.data, self._h_rew.ctypes.data, self._h_done.ctypes.data,
                            self._h_fail.ctypes.data, _lib.ptr(self._h_final)) + trunc
        # enqueued on torch's current stream: ordered after a preceding reset() / rollout() / load_state_dict()
        _lib.check(self._step_host_fn(self._h, act.ctypes.data, *self._h_ptrs, self._stream()))
        self._host_results = True
        info = QuadInfo(self._h_obs, self.obs_keys)
        return (self._out(self._h_obs), self._out(self._h_rew), self._out(self._h_done.view(np.bool_)), info)

    def step_host_buffers(self, act, obs, rew, done):
        """Host path with caller-owned (ideally pinned) buffers; see mgb_quad_step_host."""
        _lib.check(self._lib.mgb_quad_step_host(self._h, _lib.ptr(act), _lib.ptr(obs), _lib.ptr(rew), _lib.ptr(done),
                                                None, None, self._stream()))

    def rollout(self, T, actions=None, act_seed=0, want_actions=False, out=None, policy=None, deterministic=False,
                gae=None, state=None, want_hidden=False):
        """T steps in one launch (state stays in registers).  actions: [T,N,4] CUDA tensor or None (device-drawn
        U(min_voltage, max_voltage)).  Returns dict(obs [T,N,D], rew [T,N], done [T,N], act [T,N,4] or None).

        policy: an MLPPolicy (metagym_b200.policy) whose actions drive the rollout (mgb_quad_rollout_policy): the
        action of step t is drawn from N(mean, exp(log_std)^2), mean = policy(observation before step t), with the
        Philox stream keyed by act_seed; deterministic=True takes the mean.  The dict then also holds "act" [T,N,4]
        (the actions taken), "logp" [T,N] (their log-probabilities; sampling only) and "obs0" [N,D] (the observation
        acted on at t = 0; at t > 0 it is obs[t-1]).  `actions` together with `policy` is a ValueError.
        policy may also be a PolicyPopulation of MLPPolicy members (mgb_quad_rollout_population): member m drives the
        envs [m E, (m + 1) E), E = N / members, which must be 32 or a multiple of 64.
        A policy or population with a value head (MLPPolicy(value=...); mgb_quad_rollout_critic) also yields "value"
        [T,N] (V on the observation step t acts on), "value_last" [N] (V after the last step: the next launch's
        value[0]) and, with final_obs=True or gae, "final_value" [T,N] (V of the terminal observation where an episode
        ended truncated; other entries are not written).  gae=(gamma, lam) also yields "adv" and "ret" [T,N] float32,
        GAE(gamma, lam) computed in the launch (DESIGN.md "Value heads and GAE"); it needs a value head and auto_reset.
        policy may also be a GRUPolicy or an LSTMPolicy with dist="gaussian", or a population of them
        (mgb_quad_rollout_rnn; DESIGN.md "Recurrent quadrotor policies"; needs auto_reset=True), with state: the carried
        state [N, state_dim] float32, contiguous, on the env's device (policy.initial_state(N) to start fresh), read at
        the start and updated in place at the end of the launch.  The dict then also holds "state0" (a copy of state as
        read) and, with want_hidden=True, "hid" [T,N,H] (the cell's output at every step); a population's E must be
        32, 64 or a multiple of 128.

        With final_obs=True the dict also holds "final_obs" [T,N,D] float32: row (t, e) is the terminal observation
        of env e where done[t, e] (what step() reports as final_observation); it is allocated with torch.empty, and
        rows with done 0 are not written, so they hold whatever the buffer held.  And "truncated" [T,N] uint8, written
        for every step: 1 iff done and the episode ended through the time limit nt alone.  A caller-supplied `out` may
        omit either entry, and that output is then not produced."""
        torch = self._torch
        N, D, dev = self.num_envs, self.obs_dim, self.device
        if policy is not None:
            if actions is not None:
                raise ValueError("rollout takes either actions or a policy, not both")
            recurrent, population = _check_policy(self, policy, state, deterministic)
            return self._rollout_policy(T, policy, recurrent, population, act_seed, deterministic, out, gae, state,
                                        want_hidden)
        if state is not None:
            raise ValueError("state= goes with a GRUPolicy or an LSTMPolicy")
        if gae is not None:
            raise ValueError("gae= needs a policy with a value head")
        if out is None:
            out = {"obs": torch.empty((T, N, D), dtype=torch.float32, device=dev),
                   "rew": torch.empty((T, N), dtype=torch.float32, device=dev),
                   "done": torch.empty((T, N), dtype=torch.uint8, device=dev),
                   "act": torch.empty((T, N, 4), dtype=torch.float32, device=dev) if want_actions else None}
            if self._want_final:
                out["final_obs"] = torch.empty((T, N, D), dtype=torch.float32, device=dev)
                out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
        a = None
        if actions is not None:
            a = actions.to(torch.float32).reshape(T, N, 4).contiguous()
        keys = ("act", "obs", "rew", "done") + (("final_obs", "truncated") if self._want_final else ())
        _lib.check(self._rollout_fn(self._h, int(T), _lib.ptr(a), int(act_seed), *[_lib.ptr(out.get(k)) for k in keys],
                                    self._stream()))
        return out

    def evaluate(self, policy, episodes=1, act_seed=0, deterministic=False, state=None):
        """Whole-episode evaluation in one launch (mgb_quad_evaluate; DESIGN.md "Whole-episode evaluation"): every env
        steps under `policy` until its `episodes`-th done, then stops.  Step t is, bit for bit, step t of
        rollout(T, policy=policy, act_seed=act_seed, deterministic=deterministic, state=state), and each env is left as
        such a rollout of its own length leaves it (state, if given, included), so successive calls score consecutive
        episodes.  Episode 0 counts from the state the env holds now: reset() first for clean episodes.  policy is any
        policy rollout() takes, including populations and policies with a value head (never evaluated).  Needs
        auto_reset=True.  The step counter advances by episodes * nt.

        Returns {"return": [episodes, N] float64 (the rewards of each episode summed in step order), "length":
        [episodes, N] int32 (its steps; zero-filled first, so an episode the launch did not finish, which the time limit
        rules out, would show as length 0), "truncated": [episodes, N] uint8 (1 iff it ended through nt alone)}.  A
        population's fitness, member by member: res["return"].mean(0).view(M, -1).mean(1)."""
        recurrent, population = _check_policy(self, policy, state, deterministic)
        episodes = int(episodes)
        if episodes < 1 or episodes * self.nt > 2 ** 31 - 1:
            raise ValueError("episodes must be at least 1, and episodes * nt at most 2^31 - 1 steps")
        torch = self._torch
        shape = (episodes, self.num_envs)
        out = {"return": torch.empty(shape, dtype=torch.float64, device=self.device),
               "length": torch.zeros(shape, dtype=torch.int32, device=self.device),
               "truncated": torch.empty(shape, dtype=torch.uint8, device=self.device)}
        pol = ctypes.byref(policy.struct(deterministic))
        members, stride = (policy.members, policy.member_stride) if population else (1, 0)
        mlp, rnn = (None, pol) if recurrent else (pol, None)
        _lib.check(self._lib.mgb_quad_evaluate(self._h, episodes, mlp, rnn,
                                               int(policy.has_value), members, stride, int(act_seed), _lib.ptr(state),
                                               *[_lib.ptr(out[k]) for k in ("return", "length", "truncated")],
                                               self._stream()))
        return out

    def _rollout_policy(self, T, policy, recurrent, population, act_seed, deterministic, out, gae=None, state=None,
                        want_hidden=False):
        from .policy import critic_args, critic_struct
        torch = self._torch
        N, D, dev = self.num_envs, self.obs_dim, self.device
        critic = critic_args(policy, gae)
        if out is None:
            out = {"obs": torch.empty((T, N, D), dtype=torch.float32, device=dev),
                   "rew": torch.empty((T, N), dtype=torch.float32, device=dev),
                   "done": torch.empty((T, N), dtype=torch.uint8, device=dev),
                   "act": torch.empty((T, N, 4), dtype=torch.float32, device=dev),
                   "logp": None if deterministic else torch.empty((T, N), dtype=torch.float32, device=dev),
                   "obs0": torch.empty((N, D), dtype=torch.float32, device=dev)}
            if recurrent:
                out["state0"] = torch.empty((N, policy.state_dim), dtype=torch.float32, device=dev)
            if recurrent and want_hidden:
                out["hid"] = torch.empty((T, N, policy.hidden), dtype=torch.float32, device=dev)
            if self._want_final:
                out["final_obs"] = torch.empty((T, N, D), dtype=torch.float32, device=dev)
                out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
        pol = policy.struct(deterministic)
        keys = ("act", "logp", "obs0", "obs", "rew", "done", "final_obs", "truncated")
        if recurrent:
            return self._rollout_rnn(T, policy, pol, population, critic, act_seed, state, out, keys)
        if critic is not None:
            cr = critic_struct(torch, out, T, N, dev, critic, self._want_final)
            outs = [_lib.ptr(out.get(k)) for k in keys]
            members, stride = (policy.members, policy.member_stride) if population else (1, 0)
            _lib.check(self._lib.mgb_quad_rollout_critic(self._h, int(T), ctypes.byref(pol), members, stride,
                                                         int(act_seed), *outs, ctypes.byref(cr), self._stream()))
            return out
        outs = [_lib.ptr(out.get(k)) for k in keys]
        if population:
            _lib.check(self._lib.mgb_quad_rollout_population(self._h, int(T), ctypes.byref(pol), policy.members,
                                                             policy.member_stride, int(act_seed), *outs, self._stream()))
        else:
            _lib.check(self._lib.mgb_quad_rollout_policy(self._h, int(T), ctypes.byref(pol), int(act_seed), *outs,
                                                         self._stream()))
        return out

    def _rollout_rnn(self, T, policy, pol, population, critic, act_seed, state, out, keys):
        """mgb_quad_rollout_rnn, its population or its critic call: the entry point's arguments from the checked
        policy, its struct, the carried state and the output dict."""
        from .policy import critic_struct
        members = [policy.members, policy.member_stride] if population else [1, 0]
        tail = []
        if critic is not None:
            tail = [ctypes.byref(critic_struct(self._torch, out, T, self.num_envs, self.device, critic,
                                               self._want_final))]
            entry = self._lib.mgb_quad_rollout_rnn_critic
        elif population:
            entry = self._lib.mgb_quad_rollout_rnn_population
        else:
            members = []
            entry = self._lib.mgb_quad_rollout_rnn
        args = [self._h, int(T), ctypes.byref(pol)] + members + [int(act_seed)]
        args += [_lib.ptr(state), _lib.ptr(out.get("state0")), _lib.ptr(out.get("hid"))]
        _lib.check(entry(*args, *[_lib.ptr(out.get(k)) for k in keys], *tail, self._stream()))
        return out

    @property
    def fail_code(self):
        """[N] int32: MGB_FAIL_* of the last step (the reference raises instead, quadrotorsim.py:212-221).  A torch
        tensor after a device step, a numpy array after a host (numpy-action) step."""
        return self._h_fail if self._host_results else self._fail

    @property
    def final_observation(self):
        return self._h_final if self._host_results else self._final_obs

    @property
    def truncated(self):
        """final_obs=True: [N] bool, written by every step(): True iff done and the episode ended through ct == nt
        alone (env.py:159-161); a collision or a failure in that step is terminal.  So terminated = done & ~truncated.
        A torch tensor after a device step, a numpy array after a host step.  None with final_obs=False."""
        if self._trunc is None:
            return None
        t = self._h_trunc.view(np.bool_) if self._host_results else self._trunc.view(self._torch.bool)
        return self._out(t)

    def raise_on_failure(self):
        """Strict mode helper: re-raise the reference's exception for the first failed env of the last step."""
        codes = self._h_fail if self._host_results else self._fail.cpu().numpy()
        msgs = {1: "The quadrotor exists the valid zone", 2: "The quadrotor has too large velocity to recover",
                3: "The quadrotor has too large angular velocity"}
        bad = np.nonzero(codes)[0]
        if bad.size:
            raise Exception(msgs[int(codes[bad[0]])])

    def state_dict(self):
        """_save_state (quadrotorsim.py:30-40): {'state': [N,22] f32 = p3 v3 w3 prop4 R9, 'ct': [N] i32}."""
        torch = self._torch
        st = torch.empty((self.num_envs, 22), dtype=torch.float32, device=self.device)
        ct = torch.empty((self.num_envs,), dtype=torch.int32, device=self.device)
        _lib.check(self._lib.mgb_quad_state(self._h, st.data_ptr(), ct.data_ptr(), 0, self._stream()))
        return {"state": st, "ct": ct}

    def load_state_dict(self, sd):
        """_restore_state (quadrotorsim.py:42-48)."""
        torch = self._torch
        st = torch.as_tensor(sd["state"], device=self.device).to(torch.float32).reshape(self.num_envs, 22).contiguous()
        ct = sd.get("ct")
        if ct is not None:
            ct = torch.as_tensor(ct, device=self.device).to(torch.int32).contiguous()
        _lib.check(self._lib.mgb_quad_state(self._h, st.data_ptr(), _lib.ptr(ct), 1, self._stream()))
        torch.cuda.current_stream(self.device).synchronize()

    def _snap_kind(self):
        return "quadrotor"

    def _after_restore(self, rec, row_dev, row):
        """env2task follows the restored velocity tasks (int32 24 of a record; mgb_quad_restore skips invalid ones)."""
        if self.task != "velocity_control" or rec.shape[0] == 0:
            return
        torch = self._torch
        task = rec.view(torch.int32)[:, 24][row_dev.clamp(min=0)]
        take = (row_dev >= 0) & (task >= 0) & (task < self.velocity_targets.shape[0])
        self.env2task = torch.where(take, task, self.env2task)

    @property
    def launch_count(self):
        return int(self._lib.mgb_quad_launch_count(self._h))

    def step_kernel_name(self):
        """Name of the CUDA kernel a step() of this batch size launches (reporting only)."""
        return self._lib.mgb_quad_step_kernel(self._h).decode()

    def render(self, mode="human"):
        raise NotImplementedError("display is out of scope for the batched engine (reference: env.py:167-188)")

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.mgb_quad_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# reference name, batched implementation
Quadrotor = BatchedQuadrotor
