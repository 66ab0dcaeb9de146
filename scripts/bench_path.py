"""Cost of path recording (record_path=True) and of the trajectory view (god_view(trajectory=True)).

    python scripts/bench_path.py [--rounds 5]

Prints the card's name and power limit, then one JSON line per measurement:
  * maze3d: MetaMazeDiscrete3D SURVIVAL, 15x15 tasks (64), 1024 envs, 128x128 uint8 frames, the pose-cache fused step
    (bench.py --workload maze3d's shape): ms per step() with recording off and on, in alternating rounds of 200 steps.
  * maze2d_rollout: MetaMaze2D ESCAPE, view_grid 1, 15x15 tasks, 16 384 envs, rollout(T=32) with device-drawn actions
    (bench.py --workload mixed's maze half): ms per rollout with recording off and on, alternating rounds of 20 rollouts.
  * trajectory_view: 1024 MetaMaze2D envs whose paths are full (max_steps = 5000, auto_reset off, 5000 steps taken), one
    god_view(trajectory=True) at S = 480 against one live god_view() of the same envs.
Times are medians over rounds of CUDA-event windows; the range over rounds is printed beside them.
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


def window(torch, fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def alternate(torch, fns, iters, rounds):
    """{name: [ms per call of each round]}, the variants interleaved round by round."""
    for fn in fns.values():
        window(torch, fn, max(2, iters // 10))
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            out[k].append(window(torch, fn, iters))
    return out


def report(workload, times, **extra):
    import numpy as np
    row = {"workload": workload}
    for k, v in times.items():
        row[k + "_ms"] = round(float(np.median(v)), 4)
        row[k + "_ms_range"] = [round(min(v), 4), round(max(v), 4)]
    row.update(extra)
    print(json.dumps(row), flush=True)


def main():
    import numpy as np
    import torch
    from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D, MazeTaskSampler
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    rs = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, food_density=0.1, rng=rs) for _ in range(64)]

    # ---- maze3d fused step
    N = 1024
    envs = {}
    for rec in (False, True):
        e = BatchedMetaMazeDiscrete3D(num_envs=N, squeeze=False, resolution=(128, 128), obs_dtype="uint8",
                                      task_type="SURVIVAL", auto_reset=True, record_path=rec)
        e.set_task(tasks)
        e.reset()
        envs["on" if rec else "off"] = e
    acts = torch.randint(0, 4, (64, N), dtype=torch.int32, device="cuda")
    ctr = {"off": 0, "on": 0}

    def stepper(k):
        def fn():
            envs[k].step(acts[ctr[k] % 64])
            ctr[k] += 1
        return fn
    times = alternate(torch, {"off": stepper("off"), "on": stepper("on")}, 200, args.rounds)
    same = all(torch.equal(x, y) for x, y in zip(envs["off"].agent_state(), envs["on"].agent_state()))
    report("maze3d_fused_step", times, envs=N, frame="128x128 uint8", state_equal=same,
           fused_kernel=envs["on"].cache_info()["in_use"])
    for e in envs.values():
        e.close()

    # ---- maze2d rollout, T = 32
    N2, T = 16384, 32
    envs = {}
    for rec in (False, True):
        e = BatchedMetaMaze2D(num_envs=N2, squeeze=False, view_grid=1, task_type="ESCAPE", auto_reset=True,
                              record_path=rec)
        e.set_task(tasks)
        e.reset()
        envs["on" if rec else "off"] = e
    outs = {k: None for k in envs}

    def roller(k):
        def fn():
            outs[k] = envs[k].rollout(T, out=outs[k])
        return fn
    times = alternate(torch, {"off": roller("off"), "on": roller("on")}, 20, args.rounds)
    same = all(torch.equal(x, y) for x, y in zip(envs["off"].agent_state(), envs["on"].agent_state()))
    report("maze2d_rollout_T32", times, envs=N2, state_equal=same)
    for e in envs.values():
        e.close()

    # ---- trajectory view of full-length paths
    K, S = 1024, 480
    env = BatchedMetaMaze2D(num_envs=K, squeeze=False, task_type="ESCAPE", max_steps=5000, auto_reset=False,
                            render_scale=S, record_path=True)
    env.set_task(tasks)
    env.reset()
    for _ in range(5):
        env.rollout(1000, out={"obs": None})
    _, lens = env.trajectory()
    out = torch.empty((K, S, S, 3), dtype=torch.uint8, device="cuda")
    times = alternate(torch, {"live": lambda: env.god_view(out=out),
                              "trajectory": lambda: env.god_view(out=out, trajectory=True)}, 20, args.rounds)
    report("god_view_1024x480", times, path_len_min=int(lens.min()), path_len_max=int(lens.max()))
    env.close()


if __name__ == "__main__":
    main()
