"""Whole-episode evaluation: one evaluate() launch against the same episodes collected by chained rollouts.

Arms, per workload:
  (a) evaluate(policy, episodes): every env stops at its own last done;
  (b) ceil(B / 32) chained T = 32 policy rollouts that output rew / done / truncated, plus torch ops that split each
      chunk into per-episode returns, lengths and truncation flags; all captured in one CUDA graph.  B = episodes x the
      time limit, the bound (a) also runs to.
Both arms start from the same snapshot in every round (the restore is outside the timed window).  The two arms'
lengths and truncation flags are compared exactly and their returns to 1e-9 relative (the graph's scatter_add sums
each episode in another order): "arms_agree".  Reports ms per evaluation and env-steps taken (the sum of length) per
second, medians of alternating rounds, one JSON line per workload, with the GPU name and power limit.

Workloads:
  - quadrotor velocity_control, 65 536 envs, nt = 1000, dt = 0.005, MLP 19-64-64-4, episodes = 1 after reset():
    "fresh" (torch's default init) and "bias7.5" (output bias 7.5 V, small output weights);
  - the same two with a 1024-member population;
  - MetaMaze2D, 16 384 envs, GRUCell(14, 64) + Linear(64, 4), trials of k = 4 with resampling, episodes = 4, with
    step rewards -0.01 and -0.05 (life runs out after about 100 and 20 steps without food; max_steps is 200).
"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

nn = torch.nn
CHUNK = 32
SEED = 0x9E3779B97F4A7C15
CFG = dict(allow_loops=True, crowd_ratio=0.35, food_density=0.08, food_interval=3)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                 # noqa: BLE001
        return torch.cuda.get_device_name(0)


def quad_env(n, nt):
    from metagym_b200 import BatchedQuadrotor
    e = BatchedQuadrotor(task="velocity_control", dt=0.005, nt=nt, seed=list(range(8)), num_envs=n, device=0,
                         squeeze=False, auto_reset=True, rng_seed=3)
    e.reset()
    return e


def quad_policy(env, seed, bias=None):
    from metagym_b200.policy import MLPPolicy
    torch.manual_seed(seed)
    m = nn.Sequential(nn.Linear(env.obs_dim, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 4))
    if bias is not None:
        with torch.no_grad():
            m[-1].weight.mul_(0.05)
            m[-1].bias.fill_(bias)
    return MLPPolicy(m, log_std=torch.full((4,), -2.0), device=env.device)


def maze_env(n, k, step_reward):
    from metagym_b200 import BatchedMetaMaze2D
    from metagym_b200.metamaze import MazeTaskSampler
    e = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=n, squeeze=False,
                          auto_reset=True, episodes_per_task=k)
    rs = np.random.RandomState(0)
    e.set_task([MazeTaskSampler(n=9, food_density=0.08, food_interval=3, step_reward=step_reward, rng=rs)
                for _ in range(n)], env2task=np.arange(n))
    e.reset()
    return e


def maze_policy(env):
    from metagym_b200 import GRUPolicy
    torch.manual_seed(0)
    return GRUPolicy(nn.GRUCell(14, 64), nn.Linear(64, 4), hidden_reset="task", device=env.device)


def chained_arm(env, pol, episodes, limit, state, resample, reset):
    """(b): the rollouts and the stitching as one graph replay, and the outputs it fills.  reset() puts the handle back
    at the snapshot before the capture, so that the captured launches use the step counter evaluate() starts from."""
    n, dev = env.num_envs, env.device
    B = episodes * limit
    chunks = math.ceil(B / CHUNK)
    rew_t = torch.float32 if hasattr(env, "nt") else torch.float64
    buf = {"rew": torch.empty((CHUNK, n), dtype=rew_t, device=dev),
           "done": torch.empty((CHUNK, n), dtype=torch.uint8, device=dev),
           "truncated": torch.empty((CHUNK, n), dtype=torch.uint8, device=dev)}
    res = {"return": torch.zeros((episodes, n), dtype=torch.float64, device=dev),
           "length": torch.zeros((episodes, n), dtype=torch.int64, device=dev),
           "truncated": torch.zeros((episodes, n), dtype=torch.int64, device=dev)}
    ep = torch.zeros(n, dtype=torch.int64, device=dev)
    cols = torch.arange(n, device=dev)
    kw = {} if hasattr(env, "nt") else dict(resample=resample)

    def run():
        for r in res.values():
            r.zero_()
        ep.zero_()
        for _ in range(chunks):
            env.rollout(CHUNK, policy=pol, act_seed=SEED, state=state, out=buf, **kw)
            done = buf["done"].to(torch.int64)
            before = ep + torch.cumsum(done, 0) - done           # the episode each step belongs to
            live = before < episodes
            idx = (before.clamp(max=episodes - 1) * n + cols).reshape(-1)
            res["return"].view(-1).scatter_add_(0, idx, torch.where(live, buf["rew"].double(), 0.0).reshape(-1))
            res["length"].view(-1).scatter_add_(0, idx, live.to(torch.int64).reshape(-1))
            res["truncated"].view(-1).scatter_add_(0, idx, (live & (done != 0)).to(torch.int64).reshape(-1)
                                                  * buf["truncated"].to(torch.int64).reshape(-1))
            ep.add_((done * live).sum(0))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    reset()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()

    def replay():
        g.replay()
    replay.keep = (buf, ep, cols)       # the graph reads and writes these: they must live as long as it does
    return replay, res


def measure(name, env, pol, episodes, limit, rounds, state=None, resample=None, extra=None):
    snap = env.snapshot()
    state0 = state.clone() if state is not None else None
    kw = {} if hasattr(env, "nt") else dict(resample=resample)

    def reset():
        env.restore(snap)
        if state is not None:
            state.copy_(state0)

    replay_b, res_b = chained_arm(env, pol, episodes, limit, state, resample, reset)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    times = {"a": [], "b": []}
    res_a = None
    for r in range(rounds + 1):               # round 0 warms both arms up
        for arm in (("a", "b") if r % 2 == 0 else ("b", "a")):
            reset()
            torch.cuda.synchronize()
            start.record()
            if arm == "a":
                res_a = env.evaluate(pol, episodes, act_seed=SEED, state=state, **kw)
            else:
                replay_b()
            end.record()
            torch.cuda.synchronize()
            if r:
                times[arm].append(start.elapsed_time(end))
    agree = (torch.equal(res_a["length"].to(torch.int64), res_b["length"])
             and torch.equal(res_a["truncated"].to(torch.int64), res_b["truncated"])
             and torch.allclose(res_a["return"], res_b["return"], rtol=1e-9, atol=1e-9))
    steps = int(res_a["length"].sum().item())
    ms_a, ms_b = float(np.median(times["a"])), float(np.median(times["b"]))
    line = {"workload": name, "gpu": gpu_info(), "num_envs": env.num_envs, "episodes": episodes, "bound_steps":
            episodes * limit, "env_steps_taken": steps, "mean_length": steps / (episodes * env.num_envs),
            "evaluate_ms": round(ms_a, 3), "chained_ms": round(ms_b, 3), "speedup": round(ms_b / ms_a, 2),
            "evaluate_env_steps_per_s": steps / ms_a * 1e3, "chained_env_steps_per_s": steps / ms_b * 1e3,
            "rounds": rounds, "arms_agree": agree}
    line.update(extra or {})
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--quick", action="store_true", help="small shapes (a rehearsal, not a measurement)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_evaluate.py measures on the GPU"
    from metagym_b200 import PolicyPopulation
    n, nt = (2048, 100) if args.quick else (65536, 1000)
    for pop in (1, 1024):
        for kind, bias in (("fresh", None), ("bias7.5", 7.5)):
            env = quad_env(n, nt)
            pols = [quad_policy(env, s, bias) for s in range(pop)]
            pol = pols[0] if pop == 1 else PolicyPopulation(pols)
            measure("quad-%s-M%d" % (kind, pop), env, pol, 1, nt, args.rounds)
            env.close()
    mn, k = (1024, 4) if args.quick else (16384, 4)
    for step_reward in (-0.01, -0.05):      # life lasts about 100 and 20 steps without food; max_steps is 200
        env = maze_env(mn, k, step_reward)
        pol = maze_policy(env)
        state = pol.initial_state(mn)
        measure("maze2d-gru64-k%d-resample-step_reward%g" % (k, step_reward), env, pol, k, env.max_steps, args.rounds,
                state=state, resample=dict(seed=5, step_reward=step_reward, **CFG))


if __name__ == "__main__":
    main()
