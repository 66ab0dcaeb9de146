"""Exact snapshot, restore and clone of batched env state (DESIGN.md "Snapshot, restore and clone").

A snapshot is a dict of tensors that torch.save can write: one fixed-size record per env on the device, the global index
of every record's env, the handle-level counters and a fingerprint of what a compatible handle must share.  Records are
matched to envs by global index, so a snapshot can be restored into any handle (or set of handles) whose
env_index_base ranges cover the envs being restored: every per-env random stream is keyed by the global index, so a
restored env continues bit for bit whatever the sharding.
"""
import ctypes

import numpy as np

from . import _lib

VERSION = 1
FINGERPRINT_WORDS = 4


def build_row_map(global_index, env_index_base, num_envs, mask=None):
    """Row of the records to load into every local env -> int64 [num_envs], -1 = leave the env untouched.

    Local env e (global index env_index_base + e) gets the row r with global_index[r] == env_index_base + e.  mask=None:
    every local env is restored and must be covered; otherwise only envs with mask[e] set are (and must be covered).
    Raises ValueError for a global index held twice and for an env to restore that no record covers."""
    gi = np.asarray(global_index, dtype=np.int64).reshape(-1)
    if np.unique(gi).size != gi.size:
        raise ValueError("the snapshot holds an env twice (duplicate global indices)")
    local = gi - int(env_index_base)
    inside = (local >= 0) & (local < num_envs)
    row = np.full(num_envs, -1, dtype=np.int64)
    row[local[inside]] = np.nonzero(inside)[0]
    if mask is None:
        want = np.ones(num_envs, dtype=bool)
    else:
        want = np.asarray(mask).astype(bool).reshape(-1)
        if want.shape != (num_envs,):
            raise ValueError("mask must have one entry per local env (%d), got %d" % (num_envs, want.size))
    missing = np.nonzero(want & (row < 0))[0]
    if missing.size:
        raise ValueError("the snapshot does not cover %d env(s) to restore, e.g. global index %d"
                         % (missing.size, int(env_index_base) + int(missing[0])))
    row[~want] = -1
    return row


def clone_row_map(src, dst, num_envs):
    """Row map of clone_envs: env dst[i] loads record src[i] of a snapshot of the same handle, other envs -1."""
    src = np.asarray(src, dtype=np.int64).reshape(-1)
    dst = np.asarray(dst, dtype=np.int64).reshape(-1)
    if src.shape != dst.shape:
        raise ValueError("src and dst must have the same length (%d != %d)" % (src.size, dst.size))
    for name, v in (("src", src), ("dst", dst)):
        if v.size and (v.min() < 0 or v.max() >= num_envs):
            raise ValueError("%s holds an index outside [0, %d)" % (name, num_envs))
    if np.unique(dst).size != dst.size:
        raise ValueError("dst must not name an env twice")
    row = np.full(num_envs, -1, dtype=np.int64)
    row[dst] = src
    return row


def _host(t):
    """Tensor or array -> numpy on the host."""
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


class Snapshots(object):
    """snapshot() / restore() / clone_envs() of one handle kind.  The class sets _SNAP_PREFIX (C entry points
    <prefix>_snapshot ...), _FINGERPRINT_PARTS (what each fingerprint word covers, for refusals) and implements _snap_kind()
    and _after_restore(records, row_dev, row)."""
    _SNAP_PREFIX = None
    _FINGERPRINT_PARTS = ()

    def _snap_call(self, name, *args):
        self._snap_handle()
        return getattr(self._lib, self._SNAP_PREFIX + "_" + name)(self._h, *args)

    def _snap_handle(self):
        if not getattr(self, "_h", None):
            raise _lib.MgbError("no env state yet: call set_task() first")

    def _record_bytes(self):
        b = int(self._snap_call("record_bytes"))
        _lib.check(b if b < 0 else 0)
        return b

    def _fingerprint(self):
        out = (_lib.c_u64 * FINGERPRINT_WORDS)()
        _lib.check(self._snap_call("fingerprint", out))
        return np.array(out[:], dtype=np.uint64).view(np.int64)

    def _counters(self, value=None):
        t = _lib.c_u64(0 if value is None else int(value) & (2 ** 64 - 1))
        _lib.check(self._snap_call("counters", ctypes.byref(t), 0 if value is None else 1))
        return int(t.value)

    def snapshot(self, out=None):
        """-> dict(version, kind, fingerprint int64 [4], counters int64 [1] (the rollout action counter t_base),
        global_index int64 [N], records uint8 [N, B] on the device): the exact state of every env.

        out: a previous snapshot of this handle, written in place: then nothing is allocated on the device, the host is
        not synchronised, and the call can be captured in a CUDA graph (the counters and fingerprint, host values, are
        those at capture time)."""
        torch = self._torch
        N = self.num_envs
        if out is None:
            out = {"version": VERSION, "kind": self._snap_kind(),
                   "fingerprint": torch.zeros(FINGERPRINT_WORDS, dtype=torch.int64),
                   "counters": torch.zeros(1, dtype=torch.int64),
                   "global_index": torch.arange(N, dtype=torch.int64) + self.env_index_base,
                   "records": torch.empty((N, self._record_bytes()), dtype=torch.uint8, device=self.device)}
        rec = out["records"]
        if rec.device != self.device or rec.dtype != torch.uint8 or rec.dim() != 2 or rec.shape[0] != N \
                or not rec.is_contiguous() or rec.data_ptr() % 16:
            raise ValueError("out['records'] must be a contiguous, 16-byte aligned uint8 [%d, B] tensor on %s"
                             % (N, self.device))
        _lib.check(self._snap_call("snapshot", rec.data_ptr(), self._stream()))
        out["counters"].numpy()[0] = np.int64(np.uint64(self._counters()))
        out["fingerprint"].numpy()[:] = self._fingerprint()
        return out

    def _check_compatible(self, snaps):
        mine = self._fingerprint()
        first = snaps[0]
        for s in snaps:
            if s.get("version") != VERSION:
                raise ValueError("snapshot version %r, this library reads version %d" % (s.get("version"), VERSION))
            if s.get("kind") != self._snap_kind():
                raise ValueError("snapshot of a %r handle, this is a %r handle" % (s.get("kind"), self._snap_kind()))
            if not np.array_equal(_host(s["counters"]), _host(first["counters"])):
                raise ValueError("the snapshots disagree on the handle counters: they are not shards of one run")
            fp = _host(s["fingerprint"]).astype(np.int64).reshape(-1)
            if fp.shape != mine.shape or not np.array_equal(fp, mine):
                parts = [self._FINGERPRINT_PARTS[k] for k in range(min(fp.size, mine.size)) if fp[k] != mine[k]]
                raise ValueError("snapshot is incompatible with this handle: %s differ(s)" % (", ".join(parts) or "layout"))

    def restore(self, snap, mask=None):
        """Load the state of env global index g from the record of g, for every local env (mask=None) or the envs with
        mask[e] set (other envs untouched).  snap: a snapshot, or a list of snapshots of the shards of one run (their
        union).  Tensors may be on the CPU.  ValueError, before anything is written, when the snapshot does not fit this
        handle (fingerprint, kind, version) or does not cover an env to restore.  A full restore (mask=None) also sets the
        handle counters; a masked one leaves them."""
        torch = self._torch
        snaps = list(snap) if isinstance(snap, (list, tuple)) else [snap]
        if not snaps:
            raise ValueError("no snapshot given")
        self._check_compatible(snaps)
        B = self._record_bytes()
        for s in snaps:
            if s["records"].dim() != 2 or s["records"].shape[1] != B:
                raise ValueError("records of %s bytes, this handle's are %d" % (tuple(s["records"].shape[1:]), B))
        gi = np.concatenate([_host(s["global_index"]).astype(np.int64).reshape(-1) for s in snaps])
        row = build_row_map(gi, self.env_index_base, self.num_envs, None if mask is None else _host(mask))
        recs = [s["records"].to(self.device, torch.uint8) for s in snaps]
        rec = recs[0] if len(recs) == 1 else torch.cat(recs)
        if not rec.is_contiguous() or rec.data_ptr() % 16:
            rec = rec.contiguous().clone()
        self._restore_rows(rec, row)
        if mask is None:
            self._counters(np.uint64(np.int64(_host(snaps[0]["counters"]).reshape(-1)[0])))

    def _restore_rows(self, rec, row):
        row_dev = self._torch.from_numpy(row).to(self.device)
        _lib.check(self._snap_call("restore", rec.data_ptr(), int(rec.shape[0]), row_dev.data_ptr(), self._stream()))
        self._after_restore(rec, row_dev, row)

    def clone_envs(self, src, dst):
        """Env dst[i] becomes an exact copy of env src[i] (state and task); src, dst: local indices of equal length, dst
        without repeats.  Random streams stay keyed by each env's own global index, so a clone matches its source under
        the same given actions only until its next auto-reset or device-drawn action."""
        row = clone_row_map(_host(src), _host(dst), self.num_envs)
        scratch = getattr(self, "_clone_scratch", None)
        if scratch is None or scratch["records"].shape[1] != self._record_bytes():
            scratch = self._clone_scratch = self.snapshot()
        else:
            self.snapshot(out=scratch)
        self._restore_rows(scratch["records"], row)
