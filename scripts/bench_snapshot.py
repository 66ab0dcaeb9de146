"""Time snapshot(), restore() and clone_envs() with CUDA events, and report algorithmic bytes over kernel time.

Shapes: 65 536 quadrotor envs (velocity_control), MetaMazeDiscrete3D at 1024 and 16 384 envs on the pose cache and on the
direct renderer (one task-table slot per env, so records carry their tasks), MetaMaze2D at 16 384 envs.  Bytes are what
the kernels must move: a snapshot reads the env state and writes the records, a restore reads the records (and the row
map) and writes the state, a clone does both.  The share of the 3.35 TB/s HBM3 data-sheet bandwidth of an H100 SXM is
bytes / time / 3.35e12.  A record holds the env state densely, so the state side is counted as
one record per env.  The card's name and power limit are read in the same run.

usage: python scripts/bench_snapshot.py [--iters 50] [--out results/bench_snapshot.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:       # reporting only
        return "unknown (%s)" % e


def timed(torch, fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e-3 / iters


def measure(torch, name, env, iters):
    """Kernel time: back-to-back calls of the C entry points (the kernels and their launches).  Call time: the Python
    methods, which also check the fingerprint, build the row map on the host and copy it to the device."""
    from metagym_b200.snapshot import clone_row_map
    N = env.num_envs
    snap = env.snapshot()
    scratch = env.snapshot()
    rec, tmp = snap["records"], scratch["records"]
    B = rec.shape[1]
    state_per_env = B      # a record holds the env state densely (up to 28 bytes of padding), so state ~ record
    src, dst = np.arange(N // 2), np.arange(N // 2, N)
    row_all = torch.arange(N, dtype=torch.int64, device=env.device)
    row_clone = torch.from_numpy(clone_row_map(src, dst, N)).to(env.device)
    st = env._stream()
    kernel = {
        "snapshot": timed(torch, lambda: env._snap_call("snapshot", rec.data_ptr(), st), iters),
        "restore": timed(torch, lambda: env._snap_call("restore", rec.data_ptr(), N, row_all.data_ptr(), st), iters),
        "clone": timed(torch, lambda: (env._snap_call("snapshot", tmp.data_ptr(), st),
                                       env._snap_call("restore", tmp.data_ptr(), N, row_clone.data_ptr(), st)), iters)}
    call = {"snapshot": timed(torch, lambda: env.snapshot(out=snap), iters),
            "restore": timed(torch, lambda: env.restore(snap), iters),
            "clone": timed(torch, lambda: env.clone_envs(src, dst), iters)}
    # algorithmic bytes: snapshot = state read + records written; restore = records + row map read + state written;
    # clone = a snapshot of every env plus a restore of the dst half (and the row map)
    nbytes = {"snapshot": N * (state_per_env + B), "restore": N * (B + 8 + state_per_env),
              "clone": N * (state_per_env + B) + len(dst) * (B + state_per_env) + N * 8}
    res = {"case": name, "envs": N, "record_bytes": int(B)}
    for k in ("snapshot", "restore", "clone"):
        t = kernel[k]
        res[k] = {"kernel_us": round(t * 1e6, 2), "call_us": round(call[k] * 1e6, 2), "bytes": int(nbytes[k]),
                  "TBps": round(nbytes[k] / t / 1e12, 3), "share_of_3.35TBps": round(nbytes[k] / t / PEAK, 3)}
    print(json.dumps(res))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_snapshot.py needs a CUDA device")
    from metagym_b200 import BatchedQuadrotor, BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, MazeTaskSampler
    gpu = card()
    print("card:", gpu)
    results = []
    q = BatchedQuadrotor(task="velocity_control", dt=0.005, nt=1000, seed=list(range(64)), num_envs=65536, device=0,
                         auto_reset=True, squeeze=False)
    q.reset()
    results.append(measure(torch, "quadrotor", q, args.iters))
    del q
    tasks = [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=np.random.RandomState(s)) for s in range(64)]
    for n in (1024, 16384):
        for cache in (True, False):
            e2t = np.arange(n) if not cache else None
            tt = tasks if cache else [tasks[k % 64] for k in range(n)]
            env = BatchedMetaMazeDiscrete3D(resolution=(128, 128), max_steps=200, num_envs=n, device=0, auto_reset=True,
                                            obs_dtype="uint8", cache=cache, squeeze=False)
            env.set_task(tt, env2task=e2t)
            env.reset()
            results.append(measure(torch, "maze3d_%s" % ("cache" if cache else "direct"), env, args.iters))
            del env
    m = BatchedMetaMaze2D(max_steps=200, num_envs=16384, device=0, auto_reset=True, squeeze=False)
    m.set_task(tasks)
    m.reset()
    results.append(measure(torch, "maze2d", m, args.iters))
    out = {"card": gpu, "results": results}
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
