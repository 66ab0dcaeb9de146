"""Multi-GPU plumbing: shard independent envs over ranks and collate rollout chunks for the learner.

Envs never interact (SURVEY.md 8e), so the data path has NO collective: rank r steps the contiguous global env block
[r*n_local, (r+1)*n_local) with `env_index_base = r*n_local` (per-env random streams are keyed by the global index, so
results do not depend on the sharding).  The one collective is the all-gather of a rollout chunk
{obs, act, rew, done}[T, n_local, ...] -> [T, world*n_local, ...] on every rank (NCCL over NVLink/NVSwitch on GPUs; the
same code runs on gloo for the CPU tests).
"""
import os

import numpy as np

from . import _lib


def shard_range(num_envs_global, rank, world_size):
    """Contiguous block of global env indices owned by `rank` -> (base, count).  Remainder goes to the low ranks."""
    q, r = divmod(int(num_envs_global), int(world_size))
    count = q + (1 if rank < r else 0)
    base = rank * q + min(rank, r)
    return base, count


def dist_env():
    """(rank, local_rank, world_size) from the torchrun environment (1 process = 1 GPU)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")),
            int(os.environ.get("WORLD_SIZE", "1")))


def all_gather_rollout(chunk, group=None, scratch=None):
    """chunk: dict name -> tensor [T, n_local, ...] (same n_local on every rank).  Returns dict name -> tensor
    [T, world*n_local, ...] ordered by global env index.  One all_gather_into_tensor per field.
    scratch: optional dict the receive buffers are kept in between calls (no allocator traffic in steady state)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    out = {}
    for k, v in chunk.items():
        if v is None:
            continue
        if world == 1:
            out[k] = v
            continue
        src = v
        if src.dtype == torch.bool:
            src = src.to(torch.uint8)
        src = src.contiguous()
        # gather along a new leading rank axis, then fold it into the env axis: [W, T, n, ...] -> [T, W*n, ...]
        T, n = src.shape[0], src.shape[1]
        shape = (world * T,) + tuple(src.shape[1:])
        buf = None if scratch is None else scratch.get(k)
        if buf is None or tuple(buf.shape) != shape or buf.dtype != src.dtype or buf.device != src.device:
            buf = torch.empty(shape, dtype=src.dtype, device=src.device)
            if scratch is not None:
                scratch[k] = buf
        dist.all_gather_into_tensor(buf, src, group=group)        # rank-major concatenation along dim 0
        g = buf.view((world, T) + tuple(src.shape[1:])).movedim(0, 1).reshape((T, world * n) + tuple(src.shape[2:]))
        out[k] = g.to(torch.bool) if v.dtype == torch.bool else g
    return out


class RolloutArena:
    """All fields of a T-step rollout chunk carved out of ONE byte allocation, so that the engine's rollout kernels write
    straight into it (the C ABI takes plain pointers) and the learner-side collation is ONE all_gather_into_tensor
    instead of one per field.

        arena = RolloutArena({"obs": ((T, n, 19), torch.float32), "rew": ((T, n), torch.float32), ...}, device)
        env.rollout(T, out={"obs": arena["obs"], ...})
        views, work = arena.all_gather(async_op=True)      # views[name]: [world, T, n, ...], zero-copy
    Rank r's block is the global env range shard_range(...) gives it, so `views[name][r, t, i]` is global env
    `r*n + i`; `ordered(views)` copies into [T, world*n, ...] when one flat env axis is wanted."""

    ALIGN = 256

    def _layout(self, fields):
        import torch
        self.fields, self.offsets, off = {}, {}, 0
        for k, (shape, dtype) in fields.items():
            nbytes = int(torch.empty((), dtype=dtype).element_size())
            for d in shape:
                nbytes *= int(d)
            self.fields[k], self.offsets[k] = (tuple(int(d) for d in shape), dtype, nbytes), off
            off += -(-nbytes // self.ALIGN) * self.ALIGN
        self.nbytes = off

    def __init__(self, fields, device):
        import torch
        self._layout(fields)
        self.buf = torch.zeros(self.nbytes, dtype=torch.uint8, device=device)
        self.views = {k: self.buf[self.offsets[k]:self.offsets[k] + nb].view(dt).view(shape)
                      for k, (shape, dt, nb) in self.fields.items()}
        self._recv = None

    def __getitem__(self, k):
        return self.views[k]

    def payload_bytes(self):
        return sum(nb for _, _, nb in self.fields.values())

    def all_gather(self, group=None, async_op=False):
        """-> (dict name -> [world, *field shape] views of the receive arena, work handle or None)."""
        import torch
        import torch.distributed as dist
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world == 1:
            return {k: v.unsqueeze(0) for k, v in self.views.items()}, None
        if self._recv is None or self._recv.numel() != world * self.nbytes:
            self._recv = torch.empty(world * self.nbytes, dtype=torch.uint8, device=self.buf.device)
        work = dist.all_gather_into_tensor(self._recv, self.buf, group=group, async_op=async_op)
        recv = self._recv.view(world, self.nbytes)
        out = {}
        for k, (shape, dt, nb) in self.fields.items():
            o = self.offsets[k]
            out[k] = recv[:, o:o + nb].view(dt).view((world,) + shape)
        return out, (work if async_op else None)

    @staticmethod
    def ordered(views):
        """[world, T, n, ...] -> [T, world*n, ...] (global env order; this one copies)."""
        return {k: v.movedim(0, 1).reshape((v.shape[1], v.shape[0] * v.shape[2]) + tuple(v.shape[3:]))
                for k, v in views.items()}


class Mirrored(object):
    """set_mirrors() / set_multicast() of an env whose fused rollout can store its outputs into every rank's slot of a
    PeerArena or MulticastArena.  The class sets _MIRROR_PREFIX (C entry points <prefix>_set_mirrors ...)."""
    _MIRROR_PREFIX = None

    def _set_window(self, window):
        """window = (base address, bytes) of this rank's arena slot: rollouts writing elsewhere are refused while
        mirrors are on (arena.attach(env) passes it)."""
        base, nbytes = (0, 0) if window is None else (int(window[0]), int(window[1]))
        _lib.check(getattr(self._lib, self._MIRROR_PREFIX + "_set_mirror_window")(self._h, base, nbytes))

    def set_mirrors(self, byte_deltas, window=None):
        """Every output of rollout() is also stored at `pointer + delta` for each delta (PeerArena.mirrors: the kernel
        then writes the trajectory straight into the other ranks' receive arenas over NVLink)."""
        self._set_window(window)
        d = np.ascontiguousarray(np.asarray(list(byte_deltas), dtype=np.int64))
        _lib.check(getattr(self._lib, self._MIRROR_PREFIX + "_set_mirrors")(self._h, int(d.size),
                                                                              _lib.ptr(d) if d.size else None))

    def set_multicast(self, byte_delta, window=None):
        """rollout() outputs are stored through an NVSwitch multicast mapping at `pointer + byte_delta`
        (MulticastArena.multicast_delta); 0 switches it off."""
        self._set_window(window)
        _lib.check(getattr(self._lib, self._MIRROR_PREFIX + "_set_multicast")(self._h, int(byte_delta)))


class _RawDeviceMemory:
    """__cuda_array_interface__ carrier: lets torch view memory this library allocated (mgb_peer_alloc / mgb_peer_open)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


class PeerArena(RolloutArena):
    """RolloutArena whose all-gather is done by the rollout kernels themselves.

    Every rank allocates a receive arena [world][arena bytes] with mgb_peer_alloc, the 64-byte cudaIpc handles are
    exchanged once, and each rank maps the others' arenas (NVLink peer mappings).  `views` (what the env's rollout()
    writes) is slot `rank` of the LOCAL receive arena; `env.set_mirrors(arena.mirrors)` makes the fused rollout kernel
    store every output also into slot `rank` of each peer's arena.  After `sync()` (a stream-ordered one-element
    all-reduce: all kernels of the chunk have completed on every rank) `gathered[name]` is [world, T, n, ...], no copy,
    no data-path NCCL call.  Use two arenas alternately: rank r may already write chunk k+1 into arena B while the
    learner of rank s still reads chunk k from arena A; the sync of chunk k+1 orders the reuse of A for chunk k+2."""

    def __init__(self, fields, device, group=None):
        import ctypes
        import torch
        import torch.distributed as dist
        from . import _lib
        self._lib, self._libmod = _lib.load(), _lib
        dev = torch.device(device)
        self.device_index = dev.index if dev.index is not None else torch.cuda.current_device()
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if self.world - 1 > 7:
            raise ValueError("PeerArena: at most 8 ranks (MGB_MAX_MIRRORS = 7)")
        self._layout(fields)
        p = ctypes.c_void_p()
        _lib.check(self._lib.mgb_peer_alloc(self.device_index, self.world * self.nbytes, ctypes.byref(p)))
        self._base = int(p.value)
        self._peer_ptrs = {}
        self.mirrors = []
        if self.world > 1:
            handle = (ctypes.c_uint8 * 64)()
            _lib.check(self._lib.mgb_peer_export(self.device_index, self._base, handle))
            mine = torch.tensor(list(handle), dtype=torch.uint8, device=dev)
            every = torch.empty(self.world * 64, dtype=torch.uint8, device=dev)
            dist.all_gather_into_tensor(every, mine, group=group)
            every = every.cpu().numpy().reshape(self.world, 64)
            for r in range(self.world):
                if r == self.rank:
                    continue
                q = ctypes.c_void_p()
                hb = (ctypes.c_uint8 * 64)(*[int(x) for x in every[r]])
                _lib.check(self._lib.mgb_peer_open(self.device_index, hb, ctypes.byref(q)))
                self._peer_ptrs[r] = int(q.value)
                self.mirrors.append(int(q.value) - self._base)
            self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self._recv = torch.as_tensor(_RawDeviceMemory(self._base, self.world * self.nbytes), device=dev)
        recv = self._recv.view(self.world, self.nbytes)
        self.buf = recv[self.rank]
        self.views, self.gathered = {}, {}
        for k, (shape, dt, nb) in self.fields.items():
            o = self.offsets[k]
            self.views[k] = self.buf[o:o + nb].view(dt).view(shape)
            self.gathered[k] = recv[:, o:o + nb].view(dt).view((self.world,) + shape)

    def attach(self, *envs):
        """Point the envs' fused rollouts at this arena: mirrors on, and only outputs inside this rank's slot accepted."""
        for env in envs:
            env.set_mirrors(self.mirrors, window=(self.buf.data_ptr(), self.nbytes))

    @staticmethod
    def detach(*envs):
        for env in envs:
            env.set_mirrors([])

    def sync(self, async_op=False):
        """Stream-ordered rendezvous: complete (on the stream) once every rank's kernels enqueued so far have finished,
        i.e. all peer stores of this chunk have landed here.  The data never goes through NCCL.
        async_op=True returns (gathered, work): the rendezvous runs beside the next chunk's rollout; call work.wait()
        before reading `gathered`; rotate >= 4 arenas then (scripts/bench_mixed.py spells out the ordering argument)."""
        work = None
        if self.world > 1:
            import torch.distributed as dist
            work = dist.all_reduce(self._flag, group=self.group, async_op=async_op)
        return (self.gathered, work) if async_op else self.gathered

    def close(self):
        if self._base is None:
            return
        import torch
        torch.cuda.synchronize(self.device_index)
        self.views = self.gathered = self.buf = self._recv = None
        for q in self._peer_ptrs.values():
            self._lib.mgb_peer_close(self.device_index, q)
        self._peer_ptrs = {}
        if self.world > 1:
            import torch.distributed as dist
            dist.barrier(group=self.group)        # nobody frees memory a peer still has mapped
        self._lib.mgb_peer_free(self.device_index, self._base)
        self._base = None


class MulticastArena(RolloutArena):
    """PeerArena's sibling for NVSwitch multicast (NVLS): the receive arena [world][arena] of every rank is bound to ONE
    multicast object, and the rollout kernels store each output once, with multimem.st, at
    `pointer + multicast_delta`; the switch replicates the store into all ranks' arenas (this rank's included), so the
    all-gather costs every GPU its own chunk bytes of NVLink egress instead of (world-1) times that.

    Allocation, handle exchange and the cuMulticast* binding are torch.distributed._symmetric_memory's (plumbing);
    `env.set_multicast(arena.multicast_delta)`, `env.rollout(T, out=arena.views...)`, `arena.sync()` as for PeerArena."""

    def __init__(self, fields, device, group=None):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm
        dev = torch.device(device)
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self._layout(fields)
        self._recv = symm.empty(self.world * self.nbytes, dtype=torch.uint8, device=dev)
        self._recv.zero_()
        self._handle = symm.rendezvous(self._recv, self.group)
        mc = int(self._handle.multicast_ptr)
        if mc == 0:
            raise RuntimeError("MulticastArena: this GPU group has no NVSwitch multicast support")
        self.multicast_delta = mc - int(self._recv.data_ptr())
        recv = self._recv.view(self.world, self.nbytes)
        self.buf = recv[self.rank]
        self.views, self.gathered = {}, {}
        for k, (shape, dt, nb) in self.fields.items():
            o = self.offsets[k]
            self.views[k] = self.buf[o:o + nb].view(dt).view(shape)
            self.gathered[k] = recv[:, o:o + nb].view(dt).view((self.world,) + shape)
        self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        torch.cuda.synchronize(dev)
        dist.barrier(group=self.group)

    def attach(self, *envs):
        for env in envs:
            env.set_multicast(self.multicast_delta, window=(self.buf.data_ptr(), self.nbytes))

    @staticmethod
    def detach(*envs):
        for env in envs:
            env.set_multicast(0)

    def sync(self, async_op=False):
        import torch.distributed as dist
        work = dist.all_reduce(self._flag, group=self.group, async_op=async_op)
        return (self.gathered, work) if async_op else self.gathered


def rollout_bytes(chunk):
    return sum(int(v.numel()) * v.element_size() for v in chunk.values() if v is not None)
