"""Time the batched MetaMaze god view (mgb_maze_god_view) against its output-bytes floor.

    python scripts/bench_god_view.py [--envs 1024] [--view 480] [--iters 50]

Prints the card's name and power limit, then for a discrete 3-D batch and a 2-D batch (SURVIVAL, 15x15 tasks) the time of
one god_view() launch over all envs (CUDA events around `iters` launches) and the output rate.  The floor is the output
itself: K * S * S * 3 bytes at the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  For comparison it also times
torch's fill of the same output tensor, a plain write of the same bytes.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e


def main():
    import numpy as np
    import torch
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, MazeTaskSampler
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--view", type=int, default=480)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    K, S = args.envs, args.view
    print("card:", card())
    rs = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, food_density=0.1, rng=rs) for _ in range(64)]
    floor_s = K * S * S * 3 / 3.35e12
    for name, cls, kw in (("discrete3d", BatchedMetaMazeDiscrete3D, dict(resolution=(16, 16), obs_dtype="uint8")),
                          ("maze2d", BatchedMetaMaze2D, {})):
        env = cls(num_envs=K, squeeze=False, render_scale=S, **kw)
        env.set_task(tasks)
        env.reset()
        for _ in range(5):
            env.step(torch.randint(0, 4, (K,), dtype=torch.int32, device="cuda"))
        out = torch.empty((K, S, S, 3), dtype=torch.uint8, device="cuda")
        for _ in range(5):
            env.god_view(out=out)
        times = []
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                env.god_view(out=out)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b) / 1e3 / args.iters)
        t = float(np.median(times))
        fills = []                                     # the card's plain write rate over the same bytes (torch fill)
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                out.fill_(1)
            b.record()
            torch.cuda.synchronize()
            fills.append(a.elapsed_time(b) / 1e3 / args.iters)
        tf = float(np.median(fills))
        print(json.dumps({"workload": "god_view_live", "kind": name, "envs": K, "view": S, "ms": round(t * 1e3, 4),
                          "ms_range": [round(min(times) * 1e3, 4), round(max(times) * 1e3, 4)],
                          "GB_per_s": round(K * S * S * 3 / t / 1e9, 1), "floor_ms": round(floor_s * 1e3, 4),
                          "share_of_floor": round(floor_s / t, 3), "fill_same_bytes_ms": round(tf * 1e3, 4)}))
        env.close()


if __name__ == "__main__":
    main()
