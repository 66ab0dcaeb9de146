"""MLP policies for the policy-driven fused rollouts (mgb_quad_rollout_policy, mgb_maze_rollout_policy; DESIGN.md
"Policy-driven rollouts").

MLPPolicy packs a torch ``nn.Sequential`` of ``Linear`` layers alternating with one activation kind (``Tanh`` or
``ReLU``) into the flat float32 buffer the kernels read: each layer in ``nn.Linear`` order, ``W [out, in]`` row-major
then ``b [out]``, first hidden layer to output layer, then ``log_std [4]`` (the quadrotor's Gaussian head; the
MetaMaze2D rollout reads the four outputs as logits and ignores it).  The buffer lives on the env's device and is
read at every launch, so ``update()`` after an optimiser step is seen by a rollout already captured in a CUDA graph.

GRUPolicy and LSTMPolicy pack an ``nn.GRUCell`` or an ``nn.LSTMCell`` and a head for the recurrent MetaMaze2D rollout
(mgb_maze_rollout_rnn; DESIGN.md "Recurrent policies"): ``weight_ih``, ``weight_hh``, ``bias_ih``, ``bias_hh``, then the
head's layers as MLPPolicy packs them.  With dist="gaussian" they drive the quadrotor instead (mgb_quad_rollout_rnn;
DESIGN.md "Recurrent quadrotor policies"): the head's four outputs are the mean of a Gaussian, the feedback is the raw
previous action and reward, and ``log_std [4]`` goes last, as MLPPolicy packs it.  ``unroll()`` recomputes a recurrent rollout's logits and log-probabilities
with autograd, running a float32 CUDA cell through the fused cell sequence (metagym_b200.cell_seq; DESIGN.md "Fused
unroll") and any other cell through a torch loop over the steps.

Each of the three takes an optional value head, value = nn.Linear(k, 1) reading what the output layer reads: the
critic of the *_critic entry points (DESIGN.md "Value heads and GAE").  It packs as a fifth row of the output layer,
W [5][k] then b [5] (torch.cat of the actor's rows and the critic's), so the rollouts also return V(s_t), the bootstrap
values and, on request, GAE advantages.

PolicyPopulation holds M policies of one shape as the rows of one [M, numel] device tensor, and one rollout launch
drives each block of num_envs / M envs with its own member (DESIGN.md "Populations").
"""
import copy
import ctypes

from . import _lib

MAX_HIDDEN = 3     # MGB_POLICY_MAX_HIDDEN
MAX_WIDTH = 64     # MGB_POLICY_MAX_WIDTH
N_OUT = 4


def _layers(module):
    """(linears, activation code) of an nn.Sequential Linear (Act Linear)*; ValueError for anything else."""
    import torch.nn as nn
    if not isinstance(module, nn.Sequential):
        raise ValueError("MLPPolicy takes an nn.Sequential, got %s" % type(module).__name__)
    mods = list(module)
    if not mods or len(mods) % 2 == 0:
        raise ValueError("MLPPolicy needs Linear layers alternating with activations, ending in a Linear")
    lin, acts = mods[0::2], mods[1::2]
    if not all(type(m) is nn.Linear for m in lin):
        raise ValueError("MLPPolicy: every even position must be an nn.Linear")
    kinds = {type(a) for a in acts}
    if kinds - {nn.Tanh, nn.ReLU} or len(kinds) > 1:
        raise ValueError("MLPPolicy: hidden activations must all be nn.Tanh or all nn.ReLU")
    act = _lib.ACT_RELU if kinds == {nn.ReLU} else _lib.ACT_TANH
    if len(lin) - 1 > MAX_HIDDEN:
        raise ValueError("MLPPolicy: at most %d hidden layers" % MAX_HIDDEN)
    for a, b in zip(lin[:-1], lin[1:]):
        if a.out_features != b.in_features:
            raise ValueError("MLPPolicy: layer widths do not chain")
    for m in lin[:-1]:
        if not 1 <= m.out_features <= MAX_WIDTH:
            raise ValueError("MLPPolicy: hidden widths must be 1..%d" % MAX_WIDTH)
    if lin[-1].out_features != N_OUT:
        raise ValueError("MLPPolicy: the output layer must have %d outputs" % N_OUT)
    return lin, act


def _value_head(value, k, name):
    """value (an nn.Linear(k, 1)) or None; ValueError for anything else."""
    import torch.nn as nn
    if value is None:
        return None
    if type(value) is not nn.Linear or value.out_features != 1 or value.in_features != k:
        raise ValueError("%s: value must be an nn.Linear(%d, 1) reading what the output layer reads" % (name, k))
    return value


def _cat_value(W, b, value):
    """The output layer W [4][k], b [4] (float64) with the value row appended when there is one."""
    import torch
    if value is None:
        return W, b
    f64 = lambda t: t.detach().to("cpu", torch.float64)          # noqa: E731
    bv = f64(value.bias) if value.bias is not None else torch.zeros(1, dtype=torch.float64)
    return torch.cat([W, f64(value.weight)], 0), torch.cat([b, bv])


class MLPPolicy(object):
    """A torch MLP packed for the fused policy rollouts.

    module: nn.Sequential of Linear layers alternating with one activation kind (Tanh or ReLU), 0..3 hidden layers of
    width 1..64, ending in a Linear with 4 outputs.  log_std: [4] log standard deviations of the quadrotor's Gaussian
    policy (None: no stochastic quadrotor rollouts).  obs_mean / obs_std: optional [obs_dim] observation normalisation
    (x - mean) / std, folded into the first layer's W and b on the host in float64.  device: where the packed buffer
    lives (the env's CUDA device).  value: an optional nn.Linear(k, 1) value head, k the last hidden width (obs_dim
    with no hidden layer); it packs as row 4 of the output layer, where the normalisation folds into it too.
    """

    def __init__(self, module, log_std=None, obs_mean=None, obs_std=None, device="cuda", value=None):
        import torch
        self._torch = torch
        lin, self.activation = _layers(module)
        self.obs_dim = lin[0].in_features
        self.widths = [m.out_features for m in lin[:-1]]
        self.n_hidden = len(self.widths)
        self._value = _value_head(value, lin[-1].in_features, "MLPPolicy")
        self.has_value = self._value is not None
        self.numel = (sum(m.out_features * (m.in_features + 1) for m in lin) + N_OUT
                      + (lin[-1].in_features + 1 if self.has_value else 0))
        self.device = torch.device(device)
        self.params = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.has_log_std = False
        self._module, self._log_std, self._mean, self._std = module, None, None, None
        self.update(module, log_std, obs_mean, obs_std)

    def _vec(self, x, n, what):
        t = self._torch.as_tensor(x).detach().to("cpu", self._torch.float64).reshape(-1)
        if t.numel() != n:
            raise ValueError("MLPPolicy: %s must have %d entries" % (what, n))
        return t

    def pack(self):
        """The packed float32 buffer on the CPU (what update() copies to the device)."""
        torch = self._torch
        lin, _ = _layers(self._module)
        parts = []
        for k, m in enumerate(lin):
            W = m.weight.detach().to("cpu", torch.float64)
            b = m.bias.detach().to("cpu", torch.float64) if m.bias is not None else torch.zeros(m.out_features,
                                                                                                dtype=torch.float64)
            if k == len(lin) - 1:
                W, b = _cat_value(W, b, self._value)
            if k == 0 and (self._mean is not None or self._std is not None):
                mean = self._mean if self._mean is not None else torch.zeros(self.obs_dim, dtype=torch.float64)
                std = self._std if self._std is not None else torch.ones(self.obs_dim, dtype=torch.float64)
                # W ((x - mean) / std) + b = (W / std) x + (b - W (mean / std))
                b = b - W @ (mean / std)
                W = W / std
            parts += [W.reshape(-1), b]
        parts.append(self._log_std if self._log_std is not None else torch.zeros(N_OUT, dtype=torch.float64))
        return torch.cat(parts).to(torch.float32)

    def update(self, module=None, log_std=None, obs_mean=None, obs_std=None, value=None):
        """Repack into the same device buffer (copy_, stream-ordered): a graph captured on this policy sees the new
        weights.  Arguments left None keep their previous values; the module must keep its layer shapes, and a value
        head can only replace the policy's own."""
        if module is not None:
            lin, act = _layers(module)
            if (lin[0].in_features != self.obs_dim or [m.out_features for m in lin[:-1]] != self.widths
                    or act != self.activation):
                raise ValueError("MLPPolicy.update: the module must keep the layer shapes and the activation")
        if value is not None:
            if not self.has_value:
                raise ValueError("MLPPolicy.update: this policy was built without a value head")
            _value_head(value, self.widths[-1] if self.widths else self.obs_dim, "MLPPolicy")
        if log_std is not None:
            self._vec(log_std, N_OUT, "log_std")
        # normalisation is checked before anything changes: a zero or non-finite std would fold into inf / NaN weights
        mean = None if obs_mean is None else self._vec(obs_mean, self.obs_dim, "obs_mean")
        std = None if obs_std is None else self._vec(obs_std, self.obs_dim, "obs_std")
        if mean is not None and not self._torch.isfinite(mean).all():
            raise ValueError("MLPPolicy: obs_mean must be finite")
        if std is not None and not (self._torch.isfinite(std).all() and (std > 0).all()):
            raise ValueError("MLPPolicy: obs_std must be finite and strictly positive")
        if module is not None:
            self._module = module
        if log_std is not None:
            self._log_std = self._vec(log_std, N_OUT, "log_std")
            self.has_log_std = True
        if mean is not None:
            self._mean = mean
        if std is not None:
            self._std = std
        if value is not None:
            self._value = value
        self.params.copy_(self.pack(), non_blocking=False)
        return self

    def evaluate(self, obs):
        """(out [..., 4], value [...]) of observations obs [..., obs_dim] through the torch modules, with the
        observation normalisation, in the module's dtype and device (autograd flows): the reference of the value
        the critic rollouts return, and what a PPO update evaluates."""
        if not self.has_value:
            raise ValueError("MLPPolicy.evaluate needs a value head")
        torch = self._torch
        lin, _ = _layers(self._module)
        w = lin[0].weight
        x = torch.as_tensor(obs).to(w.device, w.dtype)
        if self._mean is not None:
            x = x - self._mean.to(w.device, w.dtype)
        if self._std is not None:
            x = x / self._std.to(w.device, w.dtype)
        mods = list(self._module)
        for m in mods[:-1]:
            x = m(x)
        return mods[-1](x), self._value(x)[..., 0]

    def struct(self, deterministic=False):
        """The mgb_policy the C entry points take."""
        w = (ctypes.c_int32 * 3)(*(self.widths + [0] * (3 - self.n_hidden)))
        return _lib.Policy(self.params.data_ptr(), self.n_hidden, w, self.activation,
                           _lib.POLICY_MEAN if deterministic else _lib.POLICY_SAMPLE)


FEEDBACK = 5        # onehot(prev action) or the raw prev action (4) + prev reward (1)
MAX_RNN_HIDDEN = 64  # MGB_RNN_MAX_HIDDEN
_RESETS = {"episode": _lib.RNN_RESET_EPISODE, "task": _lib.RNN_RESET_TASK}
_DISTS = ("categorical", "gaussian")
LOG_2PI_2 = 3.6757541328186907    # 2 log(2 pi): the constant of a 4-dimensional Gaussian log-density


def gaussian_logp(act, mean, log_std):
    """log N(act; mean, exp(log_std)^2) summed over the last axis of four: sum_k (-((a - mean) / sigma)^2 / 2 - log_std_k)
    - 2 log(2 pi), the logp of the quadrotor's policy rollouts (autograd flows through mean and log_std)."""
    z = (act - mean) / log_std.exp()
    return (-0.5 * z * z - log_std).sum(-1) - LOG_2PI_2


def _head_layers(head, H, name="GRUPolicy"):
    """(linears, activation code) of Linear(H, 4) or Linear(H, w) Act Linear(w, 4); ValueError for anything else."""
    import torch.nn as nn
    if type(head) is nn.Linear:
        head = nn.Sequential(head)
    try:
        lin, act = _layers(head)
    except ValueError as err:
        raise ValueError("%s head: %s" % (name, err))
    if len(lin) > 2:
        raise ValueError("%s: the head has at most one hidden layer" % name)
    if lin[0].in_features != H:
        raise ValueError("%s: the head takes %d inputs, the cell has %d units" % (name, lin[0].in_features, H))
    return lin, act


class _RecurrentPolicy(object):
    """What GRUPolicy and LSTMPolicy share: validation, the head, packing, update() and the unroll skeleton.  A
    subclass names its torch cell type (_torch_cell), its gate count, how many H-wide rows its carried memory has and
    its MGB_RNN_CELL_* code, and runs one step of its cell in _step()."""
    _gates = 0          # 3 (r, z, n) or 4 (i, f, g, o)
    _memory = 0         # H-wide rows of the carried memory before the feedback: 1 (h) or 2 (h, c)
    _cell_code = 0      # MGB_RNN_CELL_*

    def __init__(self, cell, head, log_std=None, feedback=True, hidden_reset="episode", obs_mean=None, obs_std=None,
                 device="cuda", value=None, dist="categorical"):
        import torch
        self._torch = torch
        name, kind = type(self).__name__, self._torch_cell()
        if type(cell) is not kind:
            raise ValueError("%s takes an nn.%s, got %s" % (name, kind.__name__, type(cell).__name__))
        if dist not in _DISTS:
            raise ValueError("%s: dist must be \"categorical\" (MetaMaze2D) or \"gaussian\" (the quadrotor)" % name)
        if log_std is not None and dist != "gaussian":
            raise ValueError("%s: the MetaMaze2D head is categorical and has no log_std" % name)
        if feedback not in (True, False, 0, 1):
            raise ValueError("%s: feedback must be True or False" % name)
        if hidden_reset not in _RESETS:
            raise ValueError("%s: hidden_reset must be \"episode\" or \"task\"" % name)
        if dist == "gaussian" and hidden_reset != "episode":
            raise ValueError("%s: a Gaussian (quadrotor) policy needs hidden_reset=\"episode\" (a quadrotor task never "
                             "changes inside a launch)" % name)
        self.dist = dist
        self.gaussian = dist == "gaussian"
        self.feedback = bool(feedback)
        self.hidden_reset = hidden_reset
        self.hidden = cell.hidden_size
        if not 1 <= self.hidden <= MAX_RNN_HIDDEN:
            raise ValueError("%s: the cell's hidden size must be 1..%d" % (name, MAX_RNN_HIDDEN))
        self.obs_dim = cell.input_size - FEEDBACK * self.feedback
        if self.obs_dim < 1:
            raise ValueError("%s: with feedback the cell takes obs_dim + 5 inputs" % name)
        lin, self.activation = _head_layers(head, self.hidden, name)
        self.head_width = lin[0].out_features if len(lin) == 2 else 0
        self.state_dim = self._memory * self.hidden + FEEDBACK * self.feedback
        H, n_in = self.hidden, cell.input_size
        self._value = _value_head(value, lin[-1].in_features, name)
        self.has_value = self._value is not None
        self.numel = (self._gates * H * (n_in + H + 2) + sum(m.out_features * (m.in_features + 1) for m in lin)
                      + (lin[-1].in_features + 1 if self.has_value else 0) + (N_OUT if self.gaussian else 0))
        self.device = torch.device(device)
        self.params = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.has_log_std = False
        self._cell, self._head, self._mean, self._std = cell, head, None, None
        self._log_std, self._log_std_arg = None, None
        self.update(cell, head, obs_mean, obs_std, log_std=log_std)

    def _torch_cell(self):
        raise NotImplementedError

    def _vec(self, x, n, what):
        t = self._torch.as_tensor(x).detach().to("cpu", self._torch.float64).reshape(-1)
        if t.numel() != n:
            raise ValueError("%s: %s must have %d entries" % (type(self).__name__, what, n))
        return t

    def pack(self):
        """The packed float32 buffer on the CPU (what update() copies to the device)."""
        torch = self._torch
        cell, H, D = self._cell, self.hidden, self.obs_dim
        f64 = lambda t: t.detach().to("cpu", torch.float64)          # noqa: E731
        zeros = torch.zeros(self._gates * H, dtype=torch.float64)
        Wi, Wh = f64(cell.weight_ih).clone(), f64(cell.weight_hh)
        bi = f64(cell.bias_ih) if cell.bias_ih is not None else zeros
        bh = f64(cell.bias_hh) if cell.bias_hh is not None else zeros
        if self._mean is not None or self._std is not None:
            mean = self._mean if self._mean is not None else torch.zeros(D, dtype=torch.float64)
            std = self._std if self._std is not None else torch.ones(D, dtype=torch.float64)
            # W ((x - mean) / std) + b = (W / std) x + (b - W (mean / std)), on the obs columns only
            bi = bi - Wi[:, :D] @ (mean / std)
            Wi[:, :D] = Wi[:, :D] / std
        parts = [Wi.reshape(-1), Wh.reshape(-1), bi, bh]
        lin, _ = _head_layers(self._head, H, type(self).__name__)
        for k, m in enumerate(lin):
            W, b = f64(m.weight), f64(m.bias) if m.bias is not None else torch.zeros(m.out_features, dtype=torch.float64)
            if k == len(lin) - 1:
                W, b = _cat_value(W, b, self._value)
            parts += [W.reshape(-1), b]
        if self.gaussian:
            parts.append(self._log_std if self._log_std is not None else torch.zeros(N_OUT, dtype=torch.float64))
        return torch.cat(parts).to(torch.float32)

    def update(self, cell=None, head=None, obs_mean=None, obs_std=None, value=None, log_std=None):
        """Repack into the same device buffer (copy_, stream-ordered): a graph captured on this policy sees the new
        weights.  Arguments left None keep their previous values; cell and head must keep their shapes, and a value
        head can only replace the policy's own.  log_std [4]: a Gaussian policy's log standard deviations (unroll()
        differentiates through the tensor passed here)."""
        name = type(self).__name__
        if log_std is not None:
            if not self.gaussian:
                raise ValueError("%s: the MetaMaze2D head is categorical and has no log_std" % name)
            self._vec(log_std, N_OUT, "log_std")
        if cell is not None and (type(cell) is not self._torch_cell() or cell.input_size != self._cell.input_size
                                 or cell.hidden_size != self.hidden):
            raise ValueError("%s.update: the cell must keep its input and hidden sizes" % name)
        if head is not None:
            lin, act = _head_layers(head, self.hidden, name)
            if (lin[0].out_features if len(lin) == 2 else 0) != self.head_width or act != self.activation:
                raise ValueError("%s.update: the head must keep its layer shapes and activation" % name)
        if value is not None:
            if not self.has_value:
                raise ValueError("%s.update: this policy was built without a value head" % name)
            _value_head(value, self.head_width or self.hidden, name)
        mean = None if obs_mean is None else self._vec(obs_mean, self.obs_dim, "obs_mean")
        std = None if obs_std is None else self._vec(obs_std, self.obs_dim, "obs_std")
        if mean is not None and not self._torch.isfinite(mean).all():
            raise ValueError("%s: obs_mean must be finite" % name)
        if std is not None and not (self._torch.isfinite(std).all() and (std > 0).all()):
            raise ValueError("%s: obs_std must be finite and strictly positive" % name)
        if cell is not None:
            self._cell = cell
        if head is not None:
            self._head = head
        if mean is not None:
            self._mean = mean
        if std is not None:
            self._std = std
        if value is not None:
            self._value = value
        if log_std is not None:
            self._log_std = self._vec(log_std, N_OUT, "log_std")
            self._log_std_arg = log_std
            self.has_log_std = True
        self.params.copy_(self.pack(), non_blocking=False)
        return self

    def struct(self, deterministic=False):
        """The mgb_rnn_policy the C entry point takes."""
        return _lib.RnnPolicy(self.params.data_ptr(), self.hidden, int(self.feedback), _RESETS[self.hidden_reset],
                              int(self.head_width > 0), self.head_width, self.activation,
                              _lib.POLICY_MEAN if deterministic else _lib.POLICY_SAMPLE, self._cell_code)

    def initial_state(self, num_envs):
        """[num_envs, state_dim] float32 zeros on the policy's device: the state of envs that start fresh."""
        return self._torch.zeros((int(num_envs), self.state_dim), dtype=self._torch.float32, device=self.device)

    def _step(self, x, mem):
        """(h, memory carried to the next step) of one cell step; mem holds the _memory H-wide rows of the state."""
        raise NotImplementedError

    def unroll(self, out, value=False):
        """Recompute a recurrent rollout with autograd through the cell and head: returns (logits [T, N, 4],
        logp [T, N]), logp the log-probability of out["act"], and with value=True (a policy with a value head) also
        value [T, N], V(s_t).  A Gaussian policy returns (mean [T, N, 4], logp [T, N]) instead, and autograd also
        reaches the log_std tensor it was given.  Uses out's obs0, obs, act, rew, done, state0 and
        resampled (and on a trial handle task_episodes0 and episodes_per_task), and applies the kernel's input
        construction and reset rule, in the cell's dtype and device.  A float32 cell on CUDA runs through the fused
        cell sequence (metagym_b200.cell_seq; DESIGN.md "Fused unroll"), with the head batched over all T N rows; any
        other cell, or one whose footprint the device's shared memory cannot hold, runs the torch step loop."""
        if value and not self.has_value:
            raise ValueError("unroll(value=True) needs a value head")
        from . import cell_seq
        if not cell_seq.fits(self._cell):
            return self._unroll_reference(out, value)
        torch = self._torch
        obs, act, rew, wipe, state0 = self._unroll_inputs(out)
        X = self._cell_input(obs, act, rew, wipe, state0).detach().transpose(1, 2).contiguous()
        h = cell_seq.run(self._cell, self._cell_code, X, wipe.contiguous(), state0[:, :self._memory * self.hidden])
        z = h
        mods = list(self._head) if isinstance(self._head, torch.nn.Sequential) else [self._head]
        for m in mods[:-1]:
            z = m(z)
        logits = mods[-1](z)
        logp = self._logp(logits, act)
        if value:
            return logits, logp, self._value(z)[..., 0]
        return logits, logp

    def _logp(self, out4, act):
        """log pi(act) of the head's outputs out4 [..., 4]: the categorical logits, or the Gaussian mean with log_std."""
        torch = self._torch
        if not self.gaussian:
            return torch.log_softmax(out4, -1).gather(-1, act[..., None])[..., 0]
        ls = self._log_std_arg if self._log_std_arg is not None else torch.zeros(N_OUT)
        ls = torch.as_tensor(ls).reshape(N_OUT).to(out4.device, out4.dtype)
        return gaussian_logp(act, out4, ls)

    def _unroll_inputs(self, out):
        """(obs [T, N, D] normalised, act [T, N] int64, rew [T, N] as the kernel feeds it back, wipe [T, N] bool, state0
        [N, state_dim]) of a rollout dict, in the cell's dtype and device."""
        from .metamaze import new_tasks
        torch = self._torch
        D = self.obs_dim
        w = self._cell.weight_ih
        dt, dev = w.dtype, w.device
        act = out["act"].to(dev, dt) if self.gaussian else out["act"].to(dev).long()
        T, N = act.shape[:2]
        obs = torch.cat([out["obs0"].reshape(1, N, -1), out["obs"][:T - 1].reshape(T - 1, N, -1)], 0).to(dev, dt)
        if self._mean is not None or self._std is not None:
            mean = self._mean if self._mean is not None else torch.zeros(D, dtype=torch.float64)
            std = self._std if self._std is not None else torch.ones(D, dtype=torch.float64)
            obs = (obs - mean.to(dev, dt)) / std.to(dev, dt)
        rew = out["rew"].to(dev).float().to(dt)          # the kernel feeds (float)r back
        done = out["done"].to(dev).bool()
        state0 = out["state0"].to(dev, dt)
        wipe = done if self.hidden_reset == "episode" else new_tasks(out).to(dev)
        return obs, act, rew, wipe, state0

    def _cell_input(self, obs, act, rew, wipe, state0):
        """x [T, N, in] of every step at once: the observation, then with feedback state0's feedback at t = 0 and
        (onehot(a_{t-1}) or the Gaussian's raw a_{t-1}, r_{t-1}) after, zeros where wipe[t-1]."""
        if not self.feedback:
            return obs
        torch = self._torch
        fb = torch.cat([self._action_feedback(act).to(obs.dtype), rew[..., None]], -1)
        fb = fb.masked_fill(wipe[..., None], 0.)
        return torch.cat([obs, torch.cat([state0[None, :, self._memory * self.hidden:], fb[:-1]], 0)], 2)

    def _action_feedback(self, act):
        """The four feedback entries of the actions act: onehot(act), or the Gaussian's raw actions."""
        return act if self.gaussian else self._torch.nn.functional.one_hot(act, 4)

    def _unroll_reference(self, out, value=False):
        """unroll() as a torch loop over the steps: the path of CPU and float64 cells and of cells beyond the kernels'
        footprint, and the reference the fused path is tested against."""
        if value and not self.has_value:
            raise ValueError("unroll(value=True) needs a value head")
        torch = self._torch
        head = self._head
        dt = self._cell.weight_ih.dtype
        obs, act, rew, wipe, state0 = self._unroll_inputs(out)
        T, N = act.shape[:2]
        nm = self._memory * self.hidden
        mem, fb = state0[:, :nm], state0[:, nm:]
        logits, logp, vals = [], [], []
        mods = list(head) if isinstance(head, torch.nn.Sequential) else [head]
        for t in range(T):
            x = torch.cat([obs[t], fb], 1) if self.feedback else obs[t]
            h, new_mem = self._step(x, mem)
            z = h
            for m in mods[:-1]:
                z = m(z)
            lg = mods[-1](z)
            if value:
                vals.append(self._value(z)[:, 0])
            logits.append(lg)
            logp.append(self._logp(lg, act[t]))
            keep = ~wipe[t]
            mem = torch.where(keep[:, None], new_mem, torch.zeros_like(new_mem))
            if self.feedback:
                new_fb = torch.cat([self._action_feedback(act[t]).to(dt), rew[t][:, None]], 1)
                fb = torch.where(keep[:, None], new_fb, torch.zeros_like(new_fb))
        if value:
            return torch.stack(logits), torch.stack(logp), torch.stack(vals)
        return torch.stack(logits), torch.stack(logp)


class GRUPolicy(_RecurrentPolicy):
    """A torch GRUCell and head packed for the recurrent MetaMaze2D rollout (BatchedMetaMaze2D.rollout(policy=, state=)).

    cell: nn.GRUCell(obs_dim + 5 feedback, H), H 1..64.  head: nn.Linear(H, 4), or nn.Sequential(Linear(H, w), Tanh or
    ReLU, Linear(w, 4)) with w 1..64; its four outputs are the logits of the actions.  feedback: the cell's input ends
    with onehot(prev action) and the prev reward.  hidden_reset: "episode" zeroes an env's state at every done; "task"
    only where the env drew a new maze inside the launch (rollout with resample=; on a trial handle the k-th episode on
    a maze, metamaze.new_tasks); after set_task / update_tasks /
    resample_tasks the caller zeroes the rows itself.  log_std: the maze's categorical head has none; it must be None.
    obs_mean / obs_std: optional [obs_dim] normalisation (x - mean) / std of the observation inputs, folded into the
    obs columns of weight_ih and into bias_ih on the host in float64.  device: where the packed buffer lives.
    The carried state is [N, H + 5 feedback] = [h, onehot(prev action), prev reward].

    dist="gaussian" makes it a quadrotor policy (BatchedQuadrotor.rollout(policy=, state=); mgb_quad_rollout_rnn): the
    head's four outputs are the mean of the Gaussian the actions are drawn from, log_std [4] (optional; without it only
    deterministic rollouts run) is packed last, the feedback is (a_{t-1}, r_{t-1}) with the raw action drawn, and
    hidden_reset must be "episode".  The cell then takes obs_dim (16, or 19 for velocity_control) + 5 inputs.
    """
    _gates, _memory, _cell_code = 3, 1, _lib.RNN_CELL_GRU

    def _torch_cell(self):
        return self._torch.nn.GRUCell

    def _step(self, x, mem):
        h = self._cell(x, mem)
        return h, h


class LSTMPolicy(_RecurrentPolicy):
    """A torch LSTMCell and head packed for the recurrent MetaMaze2D rollout (BatchedMetaMaze2D.rollout(policy=,
    state=)): GRUPolicy's interface and semantics with nn.LSTMCell(obs_dim + 5 feedback, H), H 1..64, whose four gates
    (i, f, g, o) are packed in torch's order.  The carried state is [N, 2H + 5 feedback] = [h, c, onehot(prev action),
    prev reward]; the reset rule zeroes the whole row, h and c included.  log_std and dist="gaussian": as GRUPolicy.
    """
    _gates, _memory, _cell_code = 4, 2, _lib.RNN_CELL_LSTM

    def __init__(self, cell, head, feedback=True, hidden_reset="episode", obs_mean=None, obs_std=None, device="cuda",
                 value=None, log_std=None, dist="categorical"):
        if log_std is not None and dist != "gaussian":
            raise TypeError("LSTMPolicy: log_std goes with dist=\"gaussian\" (the MetaMaze2D head is categorical)")
        super().__init__(cell, head, log_std, feedback, hidden_reset, obs_mean, obs_std, device, value, dist)

    def _torch_cell(self):
        return self._torch.nn.LSTMCell

    def _step(self, x, mem):
        H = self.hidden
        h, c = self._cell(x, (mem[:, :H], mem[:, H:]))
        return h, self._torch.cat([h, c], 1)


def critic_args(policy, gae):
    """(gamma, lam) for a rollout of `policy` that goes to a *_critic entry point, or None for one that does not.  A
    policy or population with a value head always goes there (gamma = lam = 1 without gae: the launch computes no GAE
    then and does not read them); gae without a value head is a ValueError."""
    if not policy.has_value:
        if gae is not None:
            raise ValueError("gae= needs a policy with a value head (value=nn.Linear(k, 1))")
        return None
    if gae is None:
        return None, None
    gamma, lam = gae
    return float(gamma), float(lam)


def critic_struct(torch, out, T, N, dev, critic, want_final):
    """The mgb_critic of a rollout whose outputs are `out`: allocates (torch.empty) the entries out lacks, "value" [T, N]
    and "value_last" [N], with want_final or gae "final_value" [T, N], and with gae "adv", "ret" [T, N] and the
    "truncated" [T, N] GAE reads."""
    gamma, lam = critic
    gae = gamma is not None
    keys = ["value", "value_last"] + (["final_value"] if want_final or gae else []) + (["adv", "ret"] if gae else [])
    for k in keys:
        if out.get(k) is None:
            out[k] = torch.empty((N,) if k == "value_last" else (T, N), dtype=torch.float32, device=dev)
    if gae and out.get("truncated") is None:
        out["truncated"] = torch.empty((T, N), dtype=torch.uint8, device=dev)
    return _lib.Critic(*[_lib.ptr(out.get(k)) for k in ("value", "value_last", "final_value", "adv", "ret")],
                       1.0 if gamma is None else gamma, 1.0 if lam is None else lam)


class PolicyPopulation(object):
    """M policies of one shape that drive one fused rollout together (DESIGN.md "Populations"): with E = N / M, member
    m acts for the envs [m E, (m + 1) E) of the handle, and everything else (draws keyed by the global env index, reset
    rules, trials, resampling, the optional outputs, the carried state) is what a handle of those E envs with
    env_index_base + m E would see with member m alone.

    policies: M MLPPolicy, GRUPolicy or LSTMPolicy objects of one class and one shape: the same layer widths,
    activation, feedback and hidden_reset, and all or none with log_std.  The observation normalisation may differ,
    since it is folded into each member's row.  The population owns `params`, a [M, numel] float32 tensor on the
    members' device; each member's `params` becomes the view of its row, so pop.policies[m].update(...) writes into the
    population, and a rollout captured in a CUDA graph sees that write and any direct write into pop.params.

    E must be a multiple of 32 that divides the kernel's CTA env count or is a multiple of it: 32 or a multiple of 64
    on the quadrotor with MLP members, 32, 64 or a multiple of 128 with recurrent members and on MetaMaze2D.  With
    M = 1 any N is accepted.
    """

    def __init__(self, policies):
        import torch
        self._torch = torch
        policies = list(policies)
        if not policies:
            raise ValueError("PolicyPopulation needs at least one policy")
        kind = type(policies[0])
        if kind not in (MLPPolicy, GRUPolicy, LSTMPolicy):
            raise ValueError("PolicyPopulation takes MLPPolicy, GRUPolicy or LSTMPolicy members, got %s" % kind.__name__)
        if any(type(p) is not kind for p in policies):
            raise ValueError("PolicyPopulation: every member must be a %s" % kind.__name__)
        if len({id(p) for p in policies}) != len(policies):
            raise ValueError("PolicyPopulation: a policy may be a member once")
        shapes = {self._shape(p) for p in policies}
        if len(shapes) != 1:
            raise ValueError("PolicyPopulation: the members must have one shape (layer widths, activation, feedback, "
                             "hidden_reset, log_std, value head) and one device")
        self.policies = policies
        self.kind = kind
        self.recurrent = kind is not MLPPolicy
        first = policies[0]
        self.numel, self.obs_dim, self.device = first.numel, first.obs_dim, first.device
        if self.recurrent:
            self.hidden, self.state_dim = first.hidden, first.state_dim
        self.params = torch.empty((len(policies), self.numel), dtype=torch.float32, device=self.device)
        for m, p in enumerate(policies):
            self.params[m].copy_(p.params)
            p.params = self.params[m]

    @staticmethod
    def _shape(p):
        if isinstance(p, MLPPolicy):
            return (p.obs_dim, tuple(p.widths), p.activation, p.has_log_std, p.has_value, p.device)
        return (p.obs_dim, p.hidden, p.head_width, p.activation, p.feedback, p.hidden_reset, p.has_value, p.device,
                p.dist, p.has_log_std)

    @classmethod
    def from_template(cls, policy, members):
        """`members` copies of one policy, for evolution strategies: each row starts as policy's packed buffer, and an
        ES step is one torch op on pop.params followed by one launch.  For an MLPPolicy or a cell and head whose layers
        all have biases and that has no normalisation, a row equals torch.nn.utils.parameters_to_vector over the
        module's parameters (MLPPolicy: the Sequential's; GRUPolicy / LSTMPolicy: the cell's, then the head's), followed
        on an MLPPolicy by its 4 log_std floats (zeros without log_std; the maze does not read them).  The copies share
        the template's torch modules until a member's update() gives it its own, so unroll() describes the rows only
        while they hold what the modules pack."""
        members = int(members)
        if members < 1:
            raise ValueError("PolicyPopulation.from_template: members must be at least 1")
        return cls([policy] + [copy.copy(policy) for _ in range(members - 1)])

    @property
    def members(self):
        return len(self.policies)

    @property
    def has_log_std(self):
        return all(p.has_log_std for p in self.policies)

    @property
    def has_value(self):
        return self.policies[0].has_value

    @property
    def dist(self):
        """The members' action distribution: "gaussian" for MLP members and Gaussian recurrent ones, else
        "categorical"."""
        return getattr(self.policies[0], "dist", "gaussian")

    def envs_per_member(self, num_envs):
        """E = num_envs / members; ValueError when num_envs is not a multiple of members."""
        num_envs = int(num_envs)
        if num_envs % self.members:
            raise ValueError("a population of %d members needs num_envs (%d) to be a multiple of it"
                             % (self.members, num_envs))
        return num_envs // self.members

    def check_envs(self, num_envs, cta_envs):
        """E for a handle of num_envs envs whose policy kernel runs cta_envs envs per CTA; ValueError naming the
        granularity rule when E is not a multiple of 32 that divides cta_envs or is a multiple of it."""
        E = self.envs_per_member(num_envs)
        if self.members > 1 and (E % _lib.POLICY_MEMBER_WARP or (cta_envs % E if E < cta_envs else E % cta_envs)):
            raise ValueError("a population needs envs per member (num_envs / members = %d) to be a multiple of %d that "
                             "divides %d or is a multiple of it" % (E, _lib.POLICY_MEMBER_WARP, cta_envs))
        return E

    def struct(self, deterministic=False):
        """The policy struct of the C entry points, pointing at row 0; the rows are member_stride floats apart."""
        st = self.policies[0].struct(deterministic)
        st.params_dev = self.params.data_ptr()
        return st

    @property
    def member_stride(self):
        return self.params.stride(0)

    _ENV_ROWS = ("obs0", "state0", "task_episodes0", "value_last")   # [N, ...]; every other tensor entry is [T, N, ...]

    def member_slice(self, out, m):
        """Member m's env columns of a rollout dict (every [T, N, ...] output, and the rows of obs0, state0,
        task_episodes0 and value_last; other entries are copied), or its rows of an [N, ...] tensor such as the carried state."""
        torch = self._torch
        if isinstance(out, torch.Tensor):
            E = self.envs_per_member(out.shape[0])
            return out[m * E:(m + 1) * E]
        E = self.envs_per_member(out["done"].shape[1])
        sl = slice(m * E, (m + 1) * E)
        res = {}
        for k, v in out.items():
            if isinstance(v, torch.Tensor):
                res[k] = v[sl] if k in self._ENV_ROWS else v[:, sl]
            else:
                res[k] = v
        return res

    def initial_state(self, num_envs):
        """[num_envs, state_dim] float32 zeros on the population's device (recurrent populations)."""
        if not self.recurrent:
            raise ValueError("initial_state: an MLP population carries no state")
        return self.policies[0].initial_state(num_envs)

    def unroll(self, out, value=False):
        """The members' unroll() over their env slices of `out`, concatenated along the env axis: (logits [T, N, 4],
        logp [T, N]), and with value=True value [T, N] (recurrent populations)."""
        if not self.recurrent:
            raise ValueError("unroll: an MLP population has nothing to unroll")
        parts = [p.unroll(self.member_slice(out, m), value) for m, p in enumerate(self.policies)]
        torch = self._torch
        return tuple(torch.cat([q[i] for q in parts], 1) for i in range(len(parts[0])))
