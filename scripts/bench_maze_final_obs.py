"""Cost of terminal observations (final_obs=True: the optional outputs of mgb_maze_step) on auto-reset maze steps.

Both arms replay T step() calls from a CUDA graph, like bench.py; one handle has final_obs off, the other on, with the
same tasks and actions.  Cases: config 4 (1024 envs, 64 tasks, 15x15, 128x128 uint8, SURVIVAL, max_steps=200; the fused
pose-cache step), the same with max_steps=10 (high done rate), the direct renderer (cache=False) and the continuous env.
The arms alternate for --runs runs; medians and ranges in microseconds per batch step, the done fraction per step measured
on the same actions, and the card's name and power limit.  One JSON line per case."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from metagym_b200 import BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D, MazeTaskSampler


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=60).stdout
        return float(out.strip())
    except Exception:
        return None


def timed_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def run_case(name, cls, kw, tasks, n, T, K, runs, cont):
    envs, graphs = {}, {}
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    if cont:
        acts = torch.rand((T, n, 2), device="cuda", dtype=torch.float32, generator=g) * 2 - 1
    else:
        acts = torch.randint(0, 4, (T, n), device="cuda", dtype=torch.int32, generator=g)
    for arm in ("off", "on"):
        env = cls(resolution=(128, 128), task_type="SURVIVAL", num_envs=n, squeeze=False, auto_reset=True,
                  obs_dtype="uint8", final_obs=(arm == "on"), **kw)
        env.set_task(tasks)
        env.reset()
        done = 0
        for t in range(T):                   # warm-up outside the capture (pose cache, scratch); counts the done rate
            done += int(env.step(acts[t])[2].sum())
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for t in range(T):
                env.step(acts[t])
        envs[arm], graphs[arm] = env, graph

    def runner(arm):
        def run():
            for _ in range(K // T):
                graphs[arm].replay()
        return run

    for arm in ("off", "on"):
        runner(arm)()
    us = {"off": [], "on": []}
    for _ in range(runs):
        for arm in ("off", "on"):
            us[arm].append(timed_ms(runner(arm)) * 1e3 / K)
    # done fraction of the timed regime: the same action sequence, stepped eagerly on the "on" handle
    env = envs["on"]
    done = 0
    for k in range(K):
        done += int(env.step(acts[k % T])[2].sum())
    med = {k: statistics.median(v) for k, v in us.items()}
    print(json.dumps({
        "case": name, "envs": n, "steps_per_run": K, "runs": runs, "gpu": torch.cuda.get_device_name(),
        "power_limit_w": power_limit_w(), "done_fraction_per_step": done / float(K * n),
        "us_per_step_off": med["off"], "us_per_step_on": med["on"],
        "range_off": [min(us["off"]), max(us["off"])], "range_on": [min(us["on"]), max(us["on"])],
        "overhead_us": med["on"] - med["off"]}), flush=True)
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--T", type=int, default=32, help="steps per captured graph")
    ap.add_argument("--steps", type=int, default=512, help="timed steps per run (a multiple of T)")
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--cases", default="config4,config4_max10,direct,continuous")
    args = ap.parse_args()
    assert args.steps % args.T == 0, "--steps must be a multiple of --T"
    assert torch.cuda.is_available(), "needs a CUDA device"
    rs = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=rs) for _ in range(64)]
    cases = {
        "config4": (BatchedMetaMazeDiscrete3D, {"max_steps": 200}, False),
        "config4_max10": (BatchedMetaMazeDiscrete3D, {"max_steps": 10}, False),
        "direct": (BatchedMetaMazeDiscrete3D, {"max_steps": 200, "cache": False}, False),
        "continuous": (BatchedMetaMazeContinuous3D, {"max_steps": 200}, True),
    }
    for name in args.cases.split(","):
        cls, kw, cont = cases[name]
        run_case(name, cls, kw, tasks, args.envs, args.T, args.steps, args.runs, cont)


if __name__ == "__main__":
    main()
