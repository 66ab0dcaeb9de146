"""MetaMazeContinuous3D: T steps as one fused rollout launch (mgb_maze_rollout, device-drawn actions) against
the same T steps as single step() launches replayed from a CUDA graph (pre-drawn actions).  Both run the direct renderer;
the rollout saves the per-step launch and the step logic's round trip through a separate launch.

Shape: 1024 envs, 64 tasks, 15x15 mazes, 128x128 uint8 frames, SURVIVAL, auto-reset, T = 32.  Each run times K steps
(K / T rollout launches, or K graph-replayed steps) with CUDA events after a warm-up of every path; the two paths
alternate for --runs runs each and the medians are reported in microseconds per batch step, with the card's name and power
limit.  Prints one JSON line.  Development aid: bench.py carries the contract metric."""
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
from metagym_b200 import BatchedMetaMazeContinuous3D, MazeTaskSampler


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--steps", type=int, default=256, help="K timed steps per run (a multiple of T)")
    ap.add_argument("--runs", type=int, default=7)
    args = ap.parse_args()
    n, T, K = args.envs, args.T, args.steps
    assert K % T == 0, "--steps must be a multiple of --T"
    assert torch.cuda.is_available(), "needs a CUDA device"
    rs = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=rs) for _ in range(64)]
    envs = {}
    for name in ("step_graph", "rollout"):
        env = BatchedMetaMazeContinuous3D(resolution=(128, 128), max_steps=200, task_type="SURVIVAL", num_envs=n,
                                          squeeze=False, auto_reset=True, obs_dtype="uint8")
        env.set_task(tasks)
        env.reset()
        envs[name] = env

    # single steps: T step() launches captured once, the graph replayed K / T times; actions drawn beforehand
    se = envs["step_graph"]
    acts = torch.rand((T, n, 2), device="cuda", dtype=torch.float32) * 2 - 1
    for t in range(T):                       # warm-up outside the capture (module load, renderer scratch)
        se.step(acts[t])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for t in range(T):
            se.step(acts[t])

    # fused: K / T rollout launches with device-drawn actions into preallocated buffers
    re = envs["rollout"]
    out = re.rollout(T, act_seed=3)

    def run_steps():
        for _ in range(K // T):
            graph.replay()

    def run_rollout():
        for _ in range(K // T):
            re.rollout(T, act_seed=3, out=out)

    run_steps()
    run_rollout()
    us = {"step_graph": [], "rollout": []}
    for _ in range(args.runs):
        us["step_graph"].append(timed_ms(run_steps) * 1e3 / K)
        us["rollout"].append(timed_ms(run_rollout) * 1e3 / K)
    med = {k: statistics.median(v) for k, v in us.items()}
    print(json.dumps({
        "case": "maze_continuous_%d_envs_128x128_u8_T%d" % (n, T), "envs": n, "T": T, "steps_per_run": K,
        "runs": args.runs, "gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(),
        "us_per_step_step_graph": med["step_graph"], "us_per_step_rollout": med["rollout"],
        "range_step_graph": [min(us["step_graph"]), max(us["step_graph"])],
        "range_rollout": [min(us["rollout"]), max(us["rollout"])],
        "rollout_speedup": med["step_graph"] / med["rollout"]}), flush=True)
    for env in envs.values():
        env.close()


if __name__ == "__main__":
    main()
