"""MLP policies for the policy-driven fused rollouts (mgb_quad_rollout_policy, mgb_maze_rollout_policy; DESIGN.md
"Policy-driven rollouts").

MLPPolicy packs a torch ``nn.Sequential`` of ``Linear`` layers alternating with one activation kind (``Tanh`` or
``ReLU``) into the flat float32 buffer the kernels read: each layer in ``nn.Linear`` order, ``W [out, in]`` row-major
then ``b [out]``, first hidden layer to output layer, then ``log_std [4]`` (the quadrotor's Gaussian head; the
MetaMaze2D rollout reads the four outputs as logits and ignores it).  The buffer lives on the env's device and is
read at every launch, so ``update()`` after an optimiser step is seen by a rollout already captured in a CUDA graph.
"""
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


class MLPPolicy(object):
    """A torch MLP packed for the fused policy rollouts.

    module: nn.Sequential of Linear layers alternating with one activation kind (Tanh or ReLU), 0..3 hidden layers of
    width 1..64, ending in a Linear with 4 outputs.  log_std: [4] log standard deviations of the quadrotor's Gaussian
    policy (None: no stochastic quadrotor rollouts).  obs_mean / obs_std: optional [obs_dim] observation normalisation
    (x - mean) / std, folded into the first layer's W and b on the host in float64.  device: where the packed buffer
    lives (the env's CUDA device).
    """

    def __init__(self, module, log_std=None, obs_mean=None, obs_std=None, device="cuda"):
        import torch
        self._torch = torch
        lin, self.activation = _layers(module)
        self.obs_dim = lin[0].in_features
        self.widths = [m.out_features for m in lin[:-1]]
        self.n_hidden = len(self.widths)
        self.numel = sum(m.out_features * (m.in_features + 1) for m in lin) + N_OUT
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
            if k == 0 and (self._mean is not None or self._std is not None):
                mean = self._mean if self._mean is not None else torch.zeros(self.obs_dim, dtype=torch.float64)
                std = self._std if self._std is not None else torch.ones(self.obs_dim, dtype=torch.float64)
                # W ((x - mean) / std) + b = (W / std) x + (b - W (mean / std))
                b = b - W @ (mean / std)
                W = W / std
            parts += [W.reshape(-1), b]
        parts.append(self._log_std if self._log_std is not None else torch.zeros(N_OUT, dtype=torch.float64))
        return torch.cat(parts).to(torch.float32)

    def update(self, module=None, log_std=None, obs_mean=None, obs_std=None):
        """Repack into the same device buffer (copy_, stream-ordered): a graph captured on this policy sees the new
        weights.  Arguments left None keep their previous values; the module must keep its layer shapes."""
        if module is not None:
            lin, act = _layers(module)
            if (lin[0].in_features != self.obs_dim or [m.out_features for m in lin[:-1]] != self.widths
                    or act != self.activation):
                raise ValueError("MLPPolicy.update: the module must keep the layer shapes and the activation")
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
        self.params.copy_(self.pack(), non_blocking=False)
        return self

    def struct(self, deterministic=False):
        """The mgb_policy the C entry points take."""
        w = (ctypes.c_int32 * 3)(*(self.widths + [0] * (3 - self.n_hidden)))
        return _lib.Policy(self.params.data_ptr(), self.n_hidden, w, self.activation,
                           _lib.POLICY_MEAN if deterministic else _lib.POLICY_SAMPLE)
