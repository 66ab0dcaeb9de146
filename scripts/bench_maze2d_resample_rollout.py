"""Per-episode task churn in MetaMaze2D: what a fresh maze for every finished env costs per env-step.

Shape: 16 384 envs of MetaMaze2D, 15x15, view_grid 1, SURVIVAL, max_steps=200, one task-table slot per env, auto-reset.
Legs, each on its own handle, alternated round by round in one process:
  (a) step(a) + resample_tasks(done) per step (obs of a re-tasked env still shows its old maze);
  (b) (a) + reset(mask=done), the loop whose obs shows the new maze (three launches per step);
  (c) rollout(32, resample=...): step, resample and the window on the new maze in one launch per 32 steps;
  (d) rollout(32) without resampling.
Before timing, (b) and (c) run the same 32 steps from the same state, over the steps where the first episodes end, and
must give identical obs, rew and done.
Each round times one window of at least --window-ms per leg with CUDA events; the medians and ranges over --rounds rounds
are printed as env-steps/s and microseconds per env-step, with the launches per step and the card's name and power limit
read in the same run.  One JSON line per leg, then one line with the check and the done fraction per step (over the checked steps and over the last timed (c) block), and
one line with the sampler on its own: resample_tasks of a single env (the latency of one carve, one warp busy) and of
every env, in microseconds per call."""
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
from metagym_b200 import BatchedMetaMaze2D, MazeTaskSampler

CFG = dict(allow_loops=True, crowd_ratio=0.35)


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=60).stdout
        return float(out.strip())
    except Exception:
        return None


def make(n, seed):
    env = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=n, squeeze=False, auto_reset=True)
    task = MazeTaskSampler(n=15, allow_loops=True, crowd_ratio=0.35, rng=np.random.RandomState(0))
    env.set_task([task] * n, env2task=np.arange(n))
    env.resample_tasks(None, seed=seed, **CFG)        # a different maze in every slot
    env.reset()
    return env


def launches(env):
    return int(env._lib.mgb_maze_launch_count(env._h))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=16384)
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--window-ms", type=float, default=50.0)
    args = ap.parse_args()
    n, T = args.envs, args.T
    assert torch.cuda.is_available(), "needs a CUDA device"
    g = torch.Generator(device="cuda")
    g.manual_seed(0)
    acts = torch.randint(0, 4, (T, n), device="cuda", dtype=torch.int32, generator=g)
    rs = dict(seed=5, **CFG)
    envs = {leg: make(n, 1) for leg in "abcd"}
    outs = {leg: {"obs": torch.empty((T, n, 3, 3), dtype=torch.float32, device="cuda"),
                  "rew": torch.empty((T, n), dtype=torch.float64, device="cuda"),
                  "done": torch.empty((T, n), dtype=torch.uint8, device="cuda"), "act": None} for leg in "cd"}

    def block(leg):
        env = envs[leg]
        if leg in "ab":
            for t in range(T):
                _, _, done, _ = env.step(acts[t])
                env.resample_tasks(done, **rs)
                if leg == "b":
                    env.reset(mask=done)
        else:
            env.rollout(T, actions=acts, out=outs[leg], resample=rs if leg == "c" else None)

    # ---- the check: (b) and (c) from the same state, the same actions, over the steps where the first episodes end
    # (life 1.0 at -0.01 per step runs out near step 100 unless food is eaten)
    for _ in range(3):
        for leg in "bc":
            envs[leg].rollout(T, actions=acts, out=outs["c"])
    b_obs, b_rew, b_done = [], [], []
    env = envs["b"]
    for t in range(T):
        _, r, d, _ = env.step(acts[t])
        b_rew.append(r.clone()); b_done.append(d.clone())
        env.resample_tasks(d, **rs)
        b_obs.append(env.reset(mask=d).clone())
    envs["c"].rollout(T, actions=acts, out=outs["c"], resample=rs)
    torch.cuda.synchronize()
    same = (torch.equal(torch.stack(b_obs), outs["c"]["obs"]) and torch.equal(torch.stack(b_rew), outs["c"]["rew"]) and
            torch.equal(torch.stack(b_done).to(torch.uint8), outs["c"]["done"]))
    done_frac = float(torch.stack(b_done).float().mean())
    del b_obs

    # ---- launches per step, then warm-up
    per_step = {}
    for leg in "abcd":
        l0 = launches(envs[leg])
        block(leg)
        per_step[leg] = (launches(envs[leg]) - l0) / T
    torch.cuda.synchronize()
    reps = {}
    for leg in "abcd":                                   # blocks per window of >= window_ms
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); block(leg); e1.record(); torch.cuda.synchronize()
        reps[leg] = max(1, int(np.ceil(args.window_ms / e0.elapsed_time(e1))))
    us = {leg: [] for leg in "abcd"}
    for _ in range(args.rounds):
        for leg in "abcd":
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps[leg]):
                block(leg)
            e1.record()
            torch.cuda.synchronize()
            us[leg].append(e0.elapsed_time(e1) * 1000.0 / (reps[leg] * T * n))
    # ---- the sampler alone, on leg (a)'s handle: one env (mask with one entry) and every env
    one = torch.zeros(n, dtype=torch.uint8, device="cuda")
    one[n // 2] = 1
    sampler_us = {}
    for what, mask in (("one_env", one), ("all_envs", None)):
        envs["a"].resample_tasks(mask, **rs)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(50):
            envs["a"].resample_tasks(mask, **rs)
        e1.record()
        torch.cuda.synchronize()
        sampler_us[what] = e0.elapsed_time(e1) * 1000.0 / 50
    card = {"card": torch.cuda.get_device_name(), "power_limit_w": power_limit_w()}
    names = {"a": "step+resample_tasks", "b": "step+resample_tasks+reset(mask=done)", "c": "rollout(T, resample)",
             "d": "rollout(T)"}
    for leg in "abcd":
        med = statistics.median(us[leg])
        print(json.dumps(dict(leg=leg, what=names[leg], envs=n, T=T, env_steps_per_s=1e6 / med, us_per_env_step=med,
                              us_per_env_step_range=[min(us[leg]), max(us[leg])], launches_per_step=per_step[leg],
                              window_ms_min=args.window_ms, rounds=args.rounds, **card)))
    print(json.dumps(dict(check="(b) == (c): obs, rew, done", equal=bool(same), done_fraction_per_step=done_frac,
                          done_fraction_per_step_timed_c=float(outs["c"]["done"].float().mean()),
                          speedup_c_over_a=statistics.median(us["a"]) / statistics.median(us["c"]),
                          speedup_c_over_b=statistics.median(us["b"]) / statistics.median(us["c"]), **card)))
    print(json.dumps(dict(sampler="resample_tasks, 15x15", us_per_call_one_env=sampler_us["one_env"],
                          us_per_call_all_envs=sampler_us["all_envs"], envs=n, **card)))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
