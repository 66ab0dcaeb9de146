"""Policy-driven rollouts: the fused rollout with the MLP evaluated in the launch, against what a user does without it.
Shapes:
  quadrotor  velocity_control, 65 536 envs, dt 0.005, nt 1000, auto-reset, T = 32, 19 -> 64 -> 64 -> 4 tanh, Gaussian head
  maze2d     MetaMaze2D SURVIVAL 15x15, 16 384 envs, view_grid 1, auto-reset, T = 32, 9 -> 64 -> 64 -> 4 tanh, categorical
             head; without and with in-launch task resampling (one table slot per env)
Three arms per shape, each timed with CUDA events as a median over alternating rounds after warm-up:
  (a) policy   rollout(T, policy=...[, resample=...])                   one launch
  (b) torch    T x (step() + the same module in torch + the same sampling and log-prob [+ resample_tasks(done) +
               reset(mask=done)]), one CUDA graph, allow_tf32 off (float32 GEMMs)
  (c) open     rollout(T[, resample=...]) with device-drawn actions     the ceiling: the env alone
Writes JSON (card name and power limit read in the same run) to --out and prints it.

usage: python scripts/bench_policy_rollout.py [--T 32] [--rounds 7] [--iters 20] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        info["power_limit_w"] = float(out.strip().splitlines()[0])
    except Exception:       # noqa: BLE001 -- reported as unknown
        pass
    return info


def graph_of(torch, steps):
    """steps() warmed up on a side stream (cuBLAS picks its kernels outside the capture), then captured in one graph."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        steps()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        steps()
    return g.replay


def time_arms(torch, args, arms, env_steps, shape):
    for f in arms.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for r in range(args.rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(list(arms)))
        for k in order:
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.iters):
                arms[k]()
            e.record()
            e.synchronize()
            times[k].append(s.elapsed_time(e) / 1e3 / args.iters)
    out = {"shape": shape, "arms": {}}
    for k, v in times.items():
        v = sorted(v)
        med = v[len(v) // 2]
        out["arms"][k] = {"median_s_per_call": med, "min_s": v[0], "max_s": v[-1], "env_steps_per_s": env_steps / med}
    out["speedup_a_over_b"] = out["arms"]["b_torch_graph"]["median_s_per_call"] / out["arms"]["a_policy_rollout"]["median_s_per_call"]
    return out


def maze_shape(torch, nn, args, resample):
    from metagym_b200 import BatchedMetaMaze2D, MazeTaskSampler
    from metagym_b200.policy import MLPPolicy
    import numpy as np
    N, T, dev = 16384, args.T, torch.device("cuda", 0)
    rs = dict(seed=5, food_density=0.05, food_interval=4) if resample else None
    rng = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, food_density=0.05, food_interval=4, rng=rng) for _ in range(64)]

    def make_env():
        env = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=N, device=0, squeeze=False,
                                auto_reset=True)
        if resample:       # one table slot per env, each drawn on the device
            env.set_task([tasks[0]] * N, env2task=np.arange(N))
            env.resample_tasks(None, **rs)
        else:
            env.set_task(tasks)
        env.reset()
        return env

    torch.manual_seed(1)
    module = nn.Sequential(nn.Linear(9, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 4)).to(dev)
    policy = MLPPolicy(module, device=dev)
    env_a, env_b, env_c = make_env(), make_env(), make_env()
    f = lambda *s, **k: torch.empty(s, device=dev, **k)          # noqa: E731
    out_a = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8),
             "act": f(T, N, dtype=torch.int32), "logp": f(T, N), "obs0": f(N, 3, 3)}
    out_c = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8), "act": None}
    buf = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8),
           "act": f(T, N, dtype=torch.int32), "logp": f(T, N)}
    cur = env_b._obs.clone()

    def steps_b():
        x = cur
        for t in range(T):
            with torch.no_grad():
                logits = module(x.reshape(N, 9))
                lsm = torch.log_softmax(logits, -1)
                u = torch.rand((N, 1), device=dev)
                a = (u >= lsm.exp().cumsum(-1)[:, :3]).sum(-1).to(torch.int32)       # inverse CDF
                buf["act"][t].copy_(a)
                buf["logp"][t].copy_(lsm.gather(-1, a.long()[:, None])[:, 0])
            o, r, d, _ = env_b.step(a)
            if resample:
                env_b.resample_tasks(d, **rs)
                o = env_b.reset(mask=d)
            buf["obs"][t].copy_(o)
            buf["rew"][t].copy_(r)
            buf["done"][t].copy_(d)
            x = buf["obs"][t]
        cur.copy_(x)

    arms = {"a_policy_rollout": lambda: env_a.rollout(T, policy=policy, act_seed=1, out=out_a, resample=rs),
            "b_torch_graph": graph_of(torch, steps_b),
            "c_open_loop_rollout": lambda: env_c.rollout(T, act_seed=2, out=out_c, resample=rs)}
    return time_arms(torch, args, arms, N * T, {"env": "MetaMaze2D SURVIVAL 15x15", "envs": N, "view_grid": 1, "T": T,
                                               "resample": resample, "policy": "9-64-64-4 tanh, categorical"})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import torch.nn as nn
    from metagym_b200 import BatchedQuadrotor
    from metagym_b200.policy import MLPPolicy
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    N, T, dev = 65536, args.T, torch.device("cuda", 0)

    def make_env():
        return BatchedQuadrotor(task="velocity_control", dt=0.005, nt=1000, seed=list(range(64)), num_envs=N, device=0,
                                squeeze=False, auto_reset=True, rng_seed=0)

    torch.manual_seed(0)
    module = nn.Sequential(nn.Linear(19, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 4)).to(dev)
    with torch.no_grad():
        module[-1].bias.add_(7.5)
    log_std = torch.full((4,), -0.5, device=dev)
    policy = MLPPolicy(module, log_std=log_std, device=dev)

    # (a) fused policy rollout, preallocated outputs
    env_a = make_env()
    env_a.reset()
    D = env_a.obs_dim
    out_a = {"obs": torch.empty((T, N, D), device=dev), "rew": torch.empty((T, N), device=dev),
             "done": torch.empty((T, N), dtype=torch.uint8, device=dev), "act": torch.empty((T, N, 4), device=dev),
             "logp": torch.empty((T, N), device=dev), "obs0": torch.empty((N, D), device=dev)}

    def arm_a():
        env_a.rollout(T, policy=policy, act_seed=1, out=out_a)

    # (b) step + torch MLP + sampling, T steps in one graph
    env_b = make_env()
    obs_b = env_b.reset()
    buf_b = {"obs": torch.empty((T, N, D), device=dev), "rew": torch.empty((T, N), device=dev),
             "done": torch.empty((T, N), dtype=torch.uint8, device=dev), "act": torch.empty((T, N, 4), device=dev),
             "logp": torch.empty((T, N), device=dev)}
    cur = obs_b.clone()
    std = torch.exp(log_std)
    half_log_2pi = 0.5 * torch.log(torch.tensor(2 * torch.pi, device=dev))

    def steps_b():
        x = cur
        for t in range(T):
            with torch.no_grad():
                mean = module(x)
                z = torch.randn_like(mean)
                a = mean + std * z
                buf_b["act"][t].copy_(a)
                buf_b["logp"][t].copy_((-0.5 * z * z - log_std - half_log_2pi).sum(-1))
            env_b.step(a, out=(buf_b["obs"][t], buf_b["rew"][t], buf_b["done"][t]))
            x = buf_b["obs"][t]
        cur.copy_(x)

    # (c) open-loop rollout
    env_c = make_env()
    env_c.reset()
    out_c = {"obs": torch.empty((T, N, D), device=dev), "rew": torch.empty((T, N), device=dev),
             "done": torch.empty((T, N), dtype=torch.uint8, device=dev), "act": None}

    def arm_c():
        env_c.rollout(T, act_seed=2, out=out_c)

    res = {"card": card(), "rounds": args.rounds, "iters_per_round": args.iters, "shapes": []}
    res["shapes"].append(time_arms(torch, args, {"a_policy_rollout": arm_a, "b_torch_graph": graph_of(torch, steps_b),
                                                 "c_open_loop_rollout": arm_c}, N * T,
                                   {"env": "quadrotor velocity_control", "envs": N, "dt": 0.005, "nt": 1000, "T": T,
                                    "policy": "19-64-64-4 tanh, Gaussian"}))
    for resample in (False, True):
        try:
            res["shapes"].append(maze_shape(torch, nn, args, resample))
        except Exception as e:      # noqa: BLE001 -- reported in the JSON, the other shapes stand
            res["shapes"].append({"shape": "maze2d resample=%s" % resample, "error": repr(e)})
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
