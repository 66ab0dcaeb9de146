"""What trials of k episodes per maze (episodes_per_task=k) cost in the resampling rollouts and in step().

Shapes (those of scripts/bench_maze2d_resample_rollout.py, bench_maze_resample_rollout.py and
bench_rnn_policy_rollout.py): MetaMaze2D 16 384 envs, 15x15, view_grid 1, SURVIVAL, max_steps=200, T = 32;
MetaMazeDiscrete3D 1024 envs, 128x128 uint8, direct renderer, T = 32; one task-table slot per env, auto-reset, every
slot a different maze.  For each workload three handles -- no trials, k = 1 and k = 4 -- are alternated round by round in
one process:
  maze2d      rollout(32, resample=...) with device-drawn actions;
  maze2d_gru  rollout(32, policy=GRUPolicy(GRUCell(14, 64), Linear(64, 4), hidden_reset="task"), resample=...);
  maze3d      rollout(32, resample=...) on the direct raycaster;
  step2d / step3d  step(a) without resampling (a trial handle adds one counting kernel per step).
k = 1 must give the outputs of the handle without trials: before timing, each workload runs one block on both from the
same state and compares obs, rew and done.  Each round times a window of at least --window-ms per handle with CUDA
events; one JSON line per (workload, handle) with the median and range over --rounds rounds in microseconds per
env-step, and the card's name and power limit read in the same run."""
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
from torch import nn

from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, MazeTaskSampler
from metagym_b200.policy import GRUPolicy

CFG = dict(allow_loops=True, crowd_ratio=0.35)
VARIANTS = (("plain", None), ("k1", 1), ("k4", 4))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=60).stdout
        return float(out.strip())
    except Exception:
        return None


def make(kind, n, k, seed=1):
    if kind == "2d":
        env = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=n, squeeze=False,
                                auto_reset=True, episodes_per_task=k)
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=(128, 128), max_steps=200, task_type="SURVIVAL", num_envs=n,
                                        squeeze=False, auto_reset=True, obs_dtype="uint8", cache=False,
                                        episodes_per_task=k)
    task = MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=np.random.RandomState(0))
    env.set_task([task] * n, env2task=np.arange(n))
    env.resample_tasks(None, seed=seed, **CFG)        # a different maze in every slot
    env.reset()
    return env


def gru_policy(env):
    g = torch.Generator().manual_seed(0)
    cell, head = nn.GRUCell(9 + 5, 64), nn.Linear(64, 4)
    with torch.no_grad():
        for p in list(cell.parameters()) + list(head.parameters()):
            p.copy_(torch.randn(p.shape, generator=g) * (1.5 / p.shape[-1] ** 0.5 if p.dim() == 2 else 0.3))
    return GRUPolicy(cell, head, feedback=True, hidden_reset="task", device=env.device)


def workload(name, T):
    """-> (envs per handle, {handle: one timed block of T steps})"""
    kind = "3d" if name in ("maze3d", "step3d") else "2d"
    n = 1024 if kind == "3d" else 16384
    blocks = {}
    for v, k in VARIANTS:
        env = make(kind, n, k)
        if name.startswith("step"):
            act = torch.randint(0, 4, (n,), dtype=torch.int32, device="cuda")
            def steps(env=env, act=act):
                for _ in range(T):
                    env.step(act)
            blocks[v] = steps
            continue
        out = {"obs": torch.empty((T, n) + tuple(env._obs.shape[1:]), dtype=env._obs.dtype, device="cuda"),
               "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
               "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"), "act": None}
        if k is not None:
            out["task_episodes0"] = torch.empty(n, dtype=torch.int32, device="cuda")
        if name == "maze2d_gru":
            pol = gru_policy(env)
            out.update(act=torch.empty((T, n), dtype=torch.int32, device="cuda"),
                       logp=torch.empty((T, n), dtype=torch.float32, device="cuda"),
                       obs0=torch.empty((n, 3, 3), dtype=torch.float32, device="cuda"),
                       state0=torch.empty((n, pol.state_dim), dtype=torch.float32, device="cuda"))
            state = pol.initial_state(n)
            blocks[v] = (lambda env=env, out=out, pol=pol, state=state:
                         env.rollout(T, policy=pol, state=state, act_seed=3, out=out, resample=dict(seed=9, **CFG)))
        elif kind == "2d":
            blocks[v] = lambda env=env, out=out: env.rollout(T, act_seed=3, out=out, resample=dict(seed=9, **CFG))
        else:
            blocks[v] = lambda env=env, out=out: env.rollout(T, act_seed=3, out=out, final_obs=False,
                                                             resample=dict(seed=9, **CFG))
    return n, blocks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window-ms", type=float, default=50.0)
    ap.add_argument("--workloads", default="maze2d,maze2d_gru,maze3d,step2d,step3d")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_maze_trials.py measures on a CUDA device; none is present")
    T = args.T
    gpu = dict(gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w())
    for name in args.workloads.split(","):
        n, blocks = workload(name, T)
        if not name.startswith("step"):                # k = 1 equals no trials, from the same state
            a, b = blocks["plain"](), blocks["k1"]()
            same = all(torch.equal(a[key], b[key]) for key in ("obs", "rew", "done"))
            print(json.dumps(dict(workload=name, check="k1 == plain: obs, rew, done", equal=bool(same))), flush=True)
        torch.cuda.synchronize()
        reps = {}
        for v in blocks:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); blocks[v](); e1.record(); torch.cuda.synchronize()
            reps[v] = max(1, int(np.ceil(args.window_ms / e0.elapsed_time(e1))))
        us = {v: [] for v in blocks}
        for _ in range(args.rounds):
            for v in blocks:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(reps[v]):
                    blocks[v]()
                e1.record()
                torch.cuda.synchronize()
                us[v].append(e0.elapsed_time(e1) * 1000.0 / (reps[v] * T * n))
        for v in blocks:
            print(json.dumps(dict(workload=name, handle=v, envs=n, T=T, us_per_env_step=statistics.median(us[v]),
                                  range=[min(us[v]), max(us[v])], **gpu)), flush=True)


if __name__ == "__main__":
    main()
