"""Cost of update_tasks on the MetaMazeDiscrete3D pose cache (the replaced tasks' region rebuilt in place on the stream).

(1) GPU time of update_tasks on the cache for K = 1, 8 and 64 replaced slots (CUDA events around the call, which enqueues
    the whole rebuild), and the host time per call.
(2) Meta-batch loop, 1024 envs = 64 tasks x 16 envs, 128x128 uint8, SURVIVAL, max_steps = 200, in env-steps/s:
    (a) 8 slots replaced every 25 steps on the cache, (b) the same loop on the direct renderer (cache=False),
    (c) set_task + reset of the whole table every 200 steps on the cache.
The arms alternate over --rounds rounds; medians and ranges are printed as one JSON line with the card and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                     # reporting only
        return "unknown (%s)" % e


def tasks(k, seed):
    from metagym_b200 import MazeTaskSampler
    rs = np.random.RandomState(seed)
    return [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=rs) for _ in range(k)]


def free_cells(t):
    w = np.asarray(t.cell_walls) == 0
    w[t.start[0], t.start[1]] = True
    return int(w.sum())


def stats(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs)), "n": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=400)
    args = ap.parse_args()
    import torch
    from metagym_b200 import BatchedMetaMazeDiscrete3D
    from metagym_b200.textures import synthetic_textures
    N, K, H = 1024, 64, 128
    table = tasks(K, 0)
    most = max(free_cells(t) for t in table)
    foods = max(int((np.asarray(t.food_rewards) > 0).sum()) for t in table)
    fresh = [t for t in tasks(1024, 1) if free_cells(t) <= most and int((np.asarray(t.food_rewards) > 0).sum()) <= foods]
    e2t = np.repeat(np.arange(K), N // K)
    tex = synthetic_textures(seed=0)

    def make(cache):
        env = BatchedMetaMazeDiscrete3D(resolution=(H, H), max_steps=200, task_type="SURVIVAL", num_envs=N, squeeze=False,
                                        textures=tex, obs_dtype="uint8", auto_reset=True, cache=cache)
        env.set_task(table, env2task=e2t)
        env.reset()
        return env

    envs = {"cache": make(True), "direct": make(False)}
    info = envs["cache"].cache_info()
    acts = torch.randint(0, 4, (64, N), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(1))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rs = np.random.RandomState(7)

    def pick(k):
        return rs.choice(K, size=k, replace=False), [fresh[int(rs.randint(len(fresh)))] for _ in range(k)]

    # (1) update_tasks alone, K = 1, 8, 64
    upd = {k: {"gpu_ms": [], "host_ms": []} for k in (1, 8, 64)}
    env = envs["cache"]
    for k in upd:                                             # warm-up: staging of every size
        env.update_tasks(*pick(k))
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k in upd:
            g, h = [], []
            for _ in range(5):
                slots, new = pick(k)
                e0.record()
                t0 = time.perf_counter()
                env.update_tasks(slots, new)
                h.append((time.perf_counter() - t0) * 1e3)
                e1.record()
                torch.cuda.synchronize()
                g.append(e0.elapsed_time(e1))
            upd[k]["gpu_ms"].append(float(np.median(g)))
            upd[k]["host_ms"].append(float(np.median(h)))

    # (2) meta-batch loops
    def loop(arm):
        env = envs["direct" if arm == "b_direct" else "cache"]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for t in range(args.steps):
            if arm == "c_set_task" and t % 200 == 199:
                env.set_task([fresh[int(rs.randint(len(fresh)))] for _ in range(K)], env2task=e2t)
                env.reset()
            elif arm != "c_set_task" and t % 25 == 24:
                env.update_tasks(*pick(8))
            env.step(acts[t % 64])
        torch.cuda.synchronize()
        return N * args.steps / (time.perf_counter() - t0)

    arms = ["a_update_cache", "b_direct", "c_set_task"]
    for arm in arms:
        loop(arm)
    rates = {arm: [] for arm in arms}
    for _ in range(args.rounds):
        for arm in arms:
            rates[arm].append(loop(arm))
    print(json.dumps({"card": card(), "cache_info": info,
                      "update_tasks": {str(k): {"gpu_ms": stats(v["gpu_ms"]), "host_ms": stats(v["host_ms"])} for k, v in upd.items()},
                      "meta_batch_env_steps_per_s": {arm: stats(v) for arm, v in rates.items()},
                      "steps_per_round": args.steps, "rounds": args.rounds}))


if __name__ == "__main__":
    main()
