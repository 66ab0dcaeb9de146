"""Cost of the terminal observations and truncation flags of the fused rollouts (mgb_quad_rollout_ex,
and mgb_maze_rollout of the three maze kinds) and of the quadrotor step's truncation
flag (mgb_quad_step_ex).

Two handles per case, final_obs off and on, same configuration and seeds.  Each arm replays a CUDA graph, like bench.py:
one rollout of T steps (device-drawn actions), or T single steps for the step case.  The arms alternate for --runs runs
of --steps timed steps; the script prints medians and ranges in microseconds per batch step, the done fraction per
step of the "on" arm, and the card's name and power limit.  One JSON line per case.  Cases:
  quad_hover_nt1000 / quad_hover_nt50   hovering_control, 65 536 envs, rollout T = 32, nt = 1000 / 50
  quad_velocity                          velocity_control, dt = 0.005, 65 536 envs, rollout T = 32
  quad_step                              the 65 536-env velocity_control step (dt = 0.005), without / with truncated
  maze2d_max200 / maze2d_max10           MetaMaze2D, 16 384 envs, view_grid = 1, ESCAPE, rollout T = 32
  maze3d_max200 / maze3d_max10           MetaMazeDiscrete3D (pose cache), 1024 envs, 64 tasks, 128x128 uint8, SURVIVAL,
                                         rollout T = 32 (the shape of bench.py --workload maze3d)
  cont3d_max200 / cont3d_max10           MetaMazeContinuous3D, the same shape (direct renderer)
For the 3-D cases both arms are the same kind of handle; "on" calls rollout(..., final_obs=True)."""
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
from metagym_b200 import (BatchedMetaMaze2D, BatchedMetaMazeContinuous3D, BatchedMetaMazeDiscrete3D, BatchedQuadrotor,
                          MazeTaskSampler)


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


def make(case, final_obs, tasks):
    kind, kw = CASES[case]
    if kind == "maze":
        env = BatchedMetaMaze2D(view_grid=1, task_type="ESCAPE", num_envs=16384, squeeze=False, auto_reset=True,
                                final_obs=final_obs, **kw)
        env.set_task(tasks)
    elif kind in ("maze3d", "cont3d"):
        cls = BatchedMetaMazeDiscrete3D if kind == "maze3d" else BatchedMetaMazeContinuous3D
        env = cls(resolution=(128, 128), obs_dtype="uint8", task_type="SURVIVAL", num_envs=1024, squeeze=False,
                  auto_reset=True, **kw)
        env.set_task(tasks)
    else:
        env = BatchedQuadrotor(num_envs=65536, squeeze=False, auto_reset=True, rng_seed=3, final_obs=final_obs, **kw)
    env.reset()
    return env


def capture(case, env, T, final_obs):
    """-> (graph, count): count() = number of done flags over the T steps of the graph's last replay (the step case
    counts them on T eager steps, so that its graph holds nothing but the steps)."""
    if case == "quad_step":
        g = torch.Generator(device="cuda").manual_seed(0)
        acts = torch.rand((T, env.num_envs, 4), device="cuda", generator=g) * 14.9 + 0.1
        for t in range(T):                                   # warm-up outside the capture
            env.step(acts[t])
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for t in range(T):
                env.step(acts[t])
        return graph, lambda: sum(int(env.step(acts[t])[2].sum()) for t in range(T))
    kw = {"final_obs": True} if final_obs and CASES[case][0] in ("maze3d", "cont3d") else {}
    out = env.rollout(T, act_seed=7, **kw)                   # warm-up; its buffers are the graph's
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        env.rollout(T, act_seed=7, out=out, **kw)
    return graph, lambda: int(out["done"].sum())


CASES = {
    "quad_hover_nt1000": ("quad", {"task": "hovering_control", "nt": 1000}),
    "quad_hover_nt50": ("quad", {"task": "hovering_control", "nt": 50}),
    "quad_velocity": ("quad", {"task": "velocity_control", "dt": 0.005, "seed": list(range(64))}),
    "quad_step": ("quad", {"task": "velocity_control", "dt": 0.005, "seed": list(range(64))}),
    "maze2d_max200": ("maze", {"max_steps": 200}),
    "maze2d_max10": ("maze", {"max_steps": 10}),
    "maze3d_max200": ("maze3d", {"max_steps": 200}),
    "maze3d_max10": ("maze3d", {"max_steps": 10}),
    "cont3d_max200": ("cont3d", {"max_steps": 200}),
    "cont3d_max10": ("cont3d", {"max_steps": 10}),
}


def run_case(case, T, K, runs, tasks):
    envs, graphs, dones = {}, {}, {}
    for arm in ("off", "on"):
        env = make(case, arm == "on", tasks)
        graphs[arm], dones[arm] = capture(case, env, T, arm == "on")
        envs[arm] = env

    def runner(arm):
        def run():
            for _ in range(K // T):
                graphs[arm].replay()
        return run

    for arm in ("off", "on"):
        runner(arm)()
    us = {"off": [], "on": []}
    done = 0
    for _ in range(runs):
        for arm in ("off", "on"):
            us[arm].append(timed_ms(runner(arm)) * 1e3 / K)
        done += dones["on"]()
    n = envs["on"].num_envs
    med = {k: statistics.median(v) for k, v in us.items()}
    print(json.dumps({
        "case": case, "envs": n, "T": T, "steps_per_run": K, "runs": runs, "gpu": torch.cuda.get_device_name(),
        "power_limit_w": power_limit_w(), "done_fraction_per_step": done / float(runs * T * n),
        "us_per_step_off": med["off"], "us_per_step_on": med["on"],
        "range_off": [min(us["off"]), max(us["off"])], "range_on": [min(us["on"]), max(us["on"])],
        "overhead_us": med["on"] - med["off"], "overhead_pct": 100.0 * (med["on"] / med["off"] - 1.0)}), flush=True)
    for e in envs.values():
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=32, help="rollout length / steps per captured step graph")
    ap.add_argument("--steps", type=int, default=1024, help="timed steps per run (a multiple of T)")
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--cases", default=",".join(CASES))
    args = ap.parse_args()
    assert args.steps % args.T == 0, "--steps must be a multiple of --T"
    assert torch.cuda.is_available(), "needs a CUDA device"
    rs = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=rs) for _ in range(64)]
    for name in args.cases.split(","):
        run_case(name, args.T, args.steps, args.runs, tasks)


if __name__ == "__main__":
    main()
