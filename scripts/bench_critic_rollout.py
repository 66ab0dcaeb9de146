"""Value heads and GAE in the policy rollouts: the critic rollout against the same policy without a value head, and
against what a PPO user computes after the rollout today.

ns per env-step, T = 32, medians of alternating rounds (each timed over 20 replays of a CUDA graph), on:
- quadrotor velocity_control, 65 536 envs, MLP 19-64-64-4 tanh, value head Linear(64, 1);
- MetaMaze2D, 16 384 envs: MLP 9-64-64-4 tanh, GRUCell(14, 64) + Linear(64, 4) and LSTMCell(14, 64) + Linear(64, 4),
  value head Linear(64, 1), the recurrent ones with and without in-launch resampling.
Arms:
  (a) critic   rollout(T, policy=<with value head>, gae=(0.99, 0.95))            one launch
  (b) plain    rollout(T, policy=<the same policy without value head>)          one launch
  (c) torch    (b), then V through MLPPolicy.evaluate (obs0, obs and final_obs) or unroll(value=True) under no_grad, and
               a torch GAE loop over T, all in one CUDA graph with TF32 off.  The recurrent arm evaluates no terminal
               values and no V(s_T) (both need memory the launch has wiped or carried on), so it is a lower bound.
Prints one JSON line per workload with the GPU name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

nn = torch.nn
T = 32
GAMMA, LAM = 0.99, 0.95


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                 # noqa: BLE001
        return torch.cuda.get_device_name(0)


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps * 1e6       # ns per call


def graph_of(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def seeded(m, seed, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * scale)
    return m.cuda()


def torch_gae(rew, cut, trunc, v, v_next_last, fv):
    """adv [T, N] by the GAE recursion in torch: what a user runs after the rollout."""
    adv = torch.empty_like(v)
    A = torch.zeros_like(v[0])
    nv = v_next_last
    zero = torch.zeros_like(A)
    for t in range(T - 1, -1, -1):
        boot = torch.where(cut[t], torch.where(trunc[t], fv[t], zero), nv)
        delta = rew[t] + GAMMA * boot - v[t]
        A = delta + torch.where(cut[t], zero, GAMMA * LAM * A)
        adv[t] = A
        nv = v[t]
    return adv, adv + v


def make_env(workload, resample):
    from metagym_b200 import BatchedMetaMaze2D, BatchedQuadrotor, MazeTaskSampler
    if workload == "quad":
        env = BatchedQuadrotor(task="velocity_control", dt=0.01, nt=1000, seed=list(range(8)), num_envs=65536, device=0,
                               squeeze=False, auto_reset=True, final_obs=True)
        env.reset()
        return env, None
    N = 16384
    rng = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, food_density=0.05, food_interval=4, rng=rng) for _ in range(64)]
    rs = dict(seed=5, food_density=0.05, food_interval=4) if resample else None
    env = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=N, device=0, squeeze=False,
                            auto_reset=True, final_obs=True)
    if resample:                   # one table slot per env, each drawn on the device
        env.set_task([tasks[0]] * N, env2task=np.arange(N))
        env.resample_tasks(None, **rs)
    else:
        env.set_task(tasks)
    env.reset()
    return env, rs


def policies(workload, dev):
    from metagym_b200 import GRUPolicy, LSTMPolicy, MLPPolicy
    value = seeded(nn.Linear(64, 1), 9)
    if workload in ("quad", "maze"):
        D = 19 if workload == "quad" else 9
        m = seeded(nn.Sequential(nn.Linear(D, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 4)), 1)
        kw = dict(log_std=[-1.0] * 4) if workload == "quad" else {}
        return MLPPolicy(m, device=dev, **kw), MLPPolicy(m, device=dev, value=value, **kw)
    cls, cell = (GRUPolicy, nn.GRUCell) if workload == "gru" else (LSTMPolicy, nn.LSTMCell)
    c, head = seeded(cell(14, 64), 1, 0.2), seeded(nn.Linear(64, 4), 2, 0.2)
    return cls(c, head, device=dev), cls(c, head, device=dev, value=value)


def bench(workload, resample, rounds):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    env_a, rs = make_env(workload, resample)
    env_b, _ = make_env(workload, resample)
    env_c, _ = make_env(workload, resample)
    N, dev = env_a.num_envs, env_a.device
    plain, critic = policies(workload, dev)
    recurrent = workload in ("gru", "lstm")
    kw = {} if workload == "quad" else dict(resample=rs)
    st = {k: (plain.initial_state(N) if recurrent else None) for k in "abc"}

    def run(env, pol, key, out=None, **extra):
        s = dict(state=st[key]) if recurrent else {}
        return env.rollout(T, policy=pol, out=out, **kw, **s, **extra)
    out_a = run(env_a, critic, "a", gae=(GAMMA, LAM))
    out_b = run(env_b, plain, "b")
    out_c = run(env_c, plain, "c")

    def arm_c():
        out = run(env_c, plain, "c", out=out_c)
        with torch.no_grad():
            cut = out["done"].bool()
            trunc = out["truncated"].bool()
            rew = out["rew"].float()
            if recurrent:
                _, _, v = critic.unroll(out, value=True)
                v_last = torch.zeros_like(v[0])
                fv = torch.zeros_like(v)
            else:
                obs = torch.cat([out["obs0"].reshape(1, N, -1), out["obs"].reshape(T, N, -1)], 0)
                _, vv = critic.evaluate(obs)
                v, v_last = vv[:T], vv[T]
                _, fv = critic.evaluate(out["final_obs"].reshape(T, N, -1))
            torch_gae(rew, cut, trunc, v, v_last, fv)

    arms = {"a_critic_gae": graph_of(lambda: run(env_a, critic, "a", out=out_a, gae=(GAMMA, LAM))),
            "b_plain": graph_of(lambda: run(env_b, plain, "b", out=out_b)),
            "c_plain_then_torch": graph_of(arm_c)}
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, 20) / (T * N))
    med = {k: float(np.median(v)) for k, v in res.items()}
    print(json.dumps({"workload": workload, "resample": bool(resample), "envs": N, "T": T,
                      "ns_per_env_step": {k: round(v, 3) for k, v in med.items()},
                      "range": {k: [round(min(v), 3), round(max(v), 3)] for k, v in res.items()},
                      "a_over_b": round(med["a_critic_gae"] / med["b_plain"], 4),
                      "c_over_a": round(med["c_plain_then_torch"] / med["a_critic_gae"], 3),
                      "gpu": gpu_info()}), flush=True)
    for e in (env_a, env_b, env_c):
        e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--workload", choices=["quad", "maze", "gru", "lstm", "all"], default="all")
    args = ap.parse_args()
    plan = [("quad", False), ("maze", False), ("gru", False), ("gru", True), ("lstm", False), ("lstm", True)]
    for w, rs in plan:
        if args.workload in ("all", w):
            bench(w, rs, args.rounds)


if __name__ == "__main__":
    main()
