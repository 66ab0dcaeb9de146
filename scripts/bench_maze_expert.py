"""ESCAPE expert: what the tables cost to build and what the expert adds to a rollout and a step.

Prints one JSON line per measurement with the GPU name and power limit.  Each comparison times its arms in alternation,
one block of calls per arm per round after a warm-up, and reports per arm the median and the range over the rounds
(CUDA events around each block).
  - table build: the kernel time of maze_expert_kernel itself (torch.profiler, CUDA activity, in a pass of its own)
    under update_tasks of all 64 slots of a 15x15 table and under resample_tasks on every env of 1024 (one slot per
    env, direct renderer) at 15x15 and at 31x31; and resample_tasks on an expert handle against a plain one;
  - rollout T = 32: expert (eps = 0.3) against open-loop device-drawn actions, MetaMaze2D at 16 384 envs and
    MetaMazeDiscrete3D at 1024 envs, 128x128 uint8, on the pose cache and on the direct renderer;
  - step: step(a, want_expert=True) against step(a), 1024 discrete-3D envs on the pose cache;
  - the same labels from torch: step + snapshot() + a gather from expert_table(), 32 steps captured in one CUDA graph,
    against 32 step(want_expert=True) captured the same way.
"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from metagym_b200 import BatchedMetaMaze2D, BatchedMetaMazeDiscrete3D  # noqa: E402
from metagym_b200.metamaze import MazeTaskSampler  # noqa: E402
from metagym_b200.textures import synthetic_textures  # noqa: E402

T = 32


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                 # noqa: BLE001
        return torch.cuda.get_device_name(0)


def paired(arms, calls=10, rounds=11):
    """{name: fn} -> {name_ms: median, name_range: [min, max]}, ms per call; the arms alternate within every round."""
    for fn in arms.values():
        fn()
    torch.cuda.synchronize()
    per = {k: [] for k in arms}
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(arms)[::-1]
        for k in order:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                arms[k]()
            b.record()
            torch.cuda.synchronize()
            per[k].append(a.elapsed_time(b) / calls)
    out = {}
    for k, v in per.items():
        out[k + "_ms"] = float(np.median(v))
        out[k + "_range"] = [float(min(v)), float(max(v))]
    return out


def build_kernel_us(fn, calls=20):
    """Mean device time of maze_expert_kernel per launch under fn (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if "maze_expert_kernel" in e.key:
            total = getattr(e, "device_time_total", None)
            if total is None:
                total = e.cuda_time_total
            return total / e.count, e.count
    raise RuntimeError("maze_expert_kernel was not launched")


def tasks(K, n=15):
    rng = np.random.RandomState(0)
    return [MazeTaskSampler(n=n, rng=rng) for _ in range(K)]


def make(kind, N, expert, K=64, env2task=None, cache=None, max_steps=200, n=15):
    kw = dict(num_envs=N, squeeze=False, auto_reset=True, task_type="ESCAPE", max_steps=max_steps, expert=expert)
    if kind == "2D":
        env = BatchedMetaMaze2D(view_grid=2, **kw)
    else:
        env = BatchedMetaMazeDiscrete3D(resolution=(128, 128), obs_dtype="uint8", textures=synthetic_textures(seed=0),
                                        cache=cache, **kw)
    env.set_task(tasks(K, n), env2task=env2task)
    env.reset()
    return env


def emit(**kw):
    print(json.dumps(dict(kw, gpu=gpu_info())), flush=True)


def main():
    table = tasks(64)
    env = make("3D", 1024, True)
    us, k = build_kernel_us(lambda: env.update_tasks(np.arange(64), table))
    emit(what="build_kernel", under="update_tasks", slots=64, n=15, us_per_launch=us, launches=k)
    for n in (15, 31):
        env = make("3D", 1024, True, K=1024, env2task=np.arange(1024), cache=False, n=n)
        us, k = build_kernel_us(lambda: env.resample_tasks(None, seed=1))
        emit(what="build_kernel", under="resample_tasks", slots=1024, n=n, us_per_launch=us, launches=k)
    envs = {x: make("3D", 1024, x, K=1024, env2task=np.arange(1024), cache=False) for x in (True, False)}
    emit(what="resample_tasks_1024x15x15", **paired({"expert": lambda: envs[True].resample_tasks(None, seed=1),
                                                    "plain": lambda: envs[False].resample_tasks(None, seed=1)}))
    for kind, N, cache in (("2D", 16384, None), ("3D", 1024, True), ("3D", 1024, False)):
        env = make(kind, N, True, cache=cache)
        out = env.rollout(T, expert=0.3, act_seed=1)
        out0 = env.rollout(T, act_seed=1, want_actions=True)
        emit(what="rollout_T32", kind=kind, envs=N, cache=cache,
             **paired({"expert": lambda: env.rollout(T, expert=0.3, act_seed=1, out=out),
                       "open_loop": lambda: env.rollout(T, act_seed=1, out=out0)}))
    env = make("3D", 1024, True, cache=True)
    a = torch.randint(0, 4, (1024,), dtype=torch.int32, device="cuda")
    emit(what="step", kind="3D", envs=1024, **paired({"step_expert": lambda: env.step(a, want_expert=True),
                                                      "step": lambda: env.step(a)}, calls=50))

    mask_tab, _ = env.expert_table()
    snap = env.snapshot()
    acts = torch.randint(0, 4, (T, 1024), dtype=torch.int32, device="cuda")
    lab = torch.empty((T, 1024), dtype=torch.uint8, device="cuda")

    def torch_labels():
        for t in range(T):
            env.step(acts[t])
            rec = env.snapshot(out=snap)["records"].view(torch.int32)
            lab[t] = mask_tab[rec[:, 7].long(), rec[:, 2].long(), rec[:, 0].long(), rec[:, 1].long()]

    def native_labels():
        for t in range(T):
            _, _, _, info = env.step(acts[t], want_expert=True)
            lab[t] = info["expert"]

    graphs = {}
    for name, fn in (("torch_snapshot", torch_labels), ("step_expert", native_labels)):
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        graphs[name] = g
    emit(what="labels_T32_graph", kind="3D", envs=1024, **paired({k: g.replay for k, g in graphs.items()}, calls=5))


if __name__ == "__main__":
    main()
