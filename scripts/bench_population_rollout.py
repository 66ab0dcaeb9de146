"""Policy populations: one fused launch for M policies against the single-policy launch and the step() + bmm path.

ns per env-step, T = 32, medians of 7 alternating rounds, on three workloads:
- quadrotor velocity_control, 65 536 envs, MLP 19-64-64-4 tanh, M in {1, 64, 1024, 2048};
- MetaMaze2D, 16 384 envs, MLP 9-64-64-4, M in {128, 512};
- MetaMaze2D, 16 384 envs, GRUCell(14, 64) + Linear(64, 4), M = 128.
Arms: (a) the population rollout; (b) the single-policy rollout of the same shape; (c) T x (step() + per-member
torch.bmm forward + sampling), captured in one CUDA graph with TF32 off.  Prints one JSON line per workload and M, with
the GPU name and power limit.
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


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:                 # noqa: BLE001
        q = torch.cuda.get_device_name(0)
    return q


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


def mlp(D, seed):
    g = torch.Generator().manual_seed(seed)
    m = nn.Sequential(nn.Linear(D, 64), nn.Tanh(), nn.Linear(64, 64), nn.Tanh(), nn.Linear(64, 4))
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return m


def bmm_arm(env, pop, N, kind):
    """T x (step + per-member bmm forward + sampling) as one replayable graph."""
    M, E = pop.members, N // pop.members
    if kind == "gru":
        cells = pop.policies[0]._cell
        Wi = cells.weight_ih.detach().cuda().expand(M, -1, -1).contiguous()
        Wh = cells.weight_hh.detach().cuda().expand(M, -1, -1).contiguous()
        bi = cells.bias_ih.detach().cuda().expand(M, -1).contiguous()
        bh = cells.bias_hh.detach().cuda().expand(M, -1).contiguous()
        hd = pop.policies[0]._head
        Wo = hd.weight.detach().cuda().expand(M, -1, -1).contiguous()
        bo = hd.bias.detach().cuda().expand(M, -1).contiguous()
        h = torch.zeros(M, E, 64, device="cuda")
        fb = torch.zeros(M, E, 5, device="cuda")
    else:
        lins = [m for m in pop.policies[0]._module if isinstance(m, nn.Linear)]
        Ws = [lin.weight.detach().cuda().expand(M, -1, -1).contiguous() for lin in lins]
        bs = [lin.bias.detach().cuda().expand(M, -1).contiguous() for lin in lins]
    obs = env._obs
    quad = kind == "quad"
    log_std = torch.zeros(4, device="cuda")

    def fwd(x):
        x = x.reshape(M, E, -1).float()
        if kind == "gru":
            xi = torch.cat([x, fb], -1)
            gi = torch.baddbmm(bi[:, None], xi, Wi.transpose(1, 2))
            gh = torch.baddbmm(bh[:, None], h, Wh.transpose(1, 2))
            r, z, n_ = gi.chunk(3, -1)
            rh, zh, nh = gh.chunk(3, -1)
            r, z = torch.sigmoid(r + rh), torch.sigmoid(z + zh)
            n_ = torch.tanh(n_ + r * nh)
            h.copy_((1 - z) * n_ + z * h)
            return torch.baddbmm(bo[:, None], h, Wo.transpose(1, 2))
        for k, (w, b) in enumerate(zip(Ws, bs)):
            x = torch.baddbmm(b[:, None], x, w.transpose(1, 2))
            if k < len(Ws) - 1:
                x = torch.tanh(x)
        return x

    def run():
        for _ in range(T):
            out = fwd(obs).reshape(N, 4)
            if quad:
                a = out + torch.exp(log_std) * torch.randn_like(out)
            else:
                a = torch.multinomial(torch.softmax(out, -1), 1)[:, 0].to(torch.int32)
            env.step(a)
    return graph_of(run)


def bench(workload, Ms, rounds):
    from metagym_b200 import BatchedMetaMaze2D, BatchedQuadrotor, GRUPolicy, MLPPolicy, PolicyPopulation
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    if workload == "quad":
        N = 65536
        env = BatchedQuadrotor(task="velocity_control", dt=0.01, nt=1000, seed=list(range(8)), num_envs=N, device=0,
                               squeeze=False, auto_reset=True)
        env.reset()
        make = lambda s: MLPPolicy(mlp(19, s), log_std=[-1.0] * 4, device=env.device)   # noqa: E731
    else:
        from metagym_b200 import MazeTaskSampler
        N = 16384
        env = BatchedMetaMaze2D(max_steps=200, view_grid=1, num_envs=N, squeeze=False, auto_reset=True)
        env.set_task([MazeTaskSampler(n=9, rng=np.random.RandomState(k)) for k in range(64)],
                     env2task=np.arange(N) % 64)
        env.reset()
        if workload == "gru":
            def make(s):
                g = torch.Generator().manual_seed(s)
                cell, head = nn.GRUCell(14, 64), nn.Linear(64, 4)
                with torch.no_grad():
                    for p in list(cell.parameters()) + list(head.parameters()):
                        p.copy_(torch.randn(p.shape, generator=g) * 0.2)
                return GRUPolicy(cell, head, device=env.device)
        else:
            make = lambda s: MLPPolicy(mlp(9, s), device=env.device)    # noqa: E731
    single = make(0)
    for M in Ms:
        pop = PolicyPopulation([single] + [make(s + 1) for s in range(M - 1)]) if M > 1 else PolicyPopulation([single])
        state = pop.initial_state(N) if workload == "gru" else None
        kw = dict(state=state) if state is not None else {}
        out_a = env.rollout(T, policy=pop, **kw)
        out_b = env.rollout(T, policy=single, **kw)
        arms = {"population": graph_of(lambda: env.rollout(T, policy=pop, out=out_a, **kw)),
                "single": graph_of(lambda: env.rollout(T, policy=single, out=out_b, **kw)),
                "step_bmm": bmm_arm(env, pop, N, workload)}
        res = {k: [] for k in arms}
        for _ in range(rounds):
            for k, fn in arms.items():
                res[k].append(timed(fn, 5) / (T * N))
        print(json.dumps({"workload": workload, "envs": N, "members": M, "envs_per_member": N // M,
                          "ns_per_env_step": {k: round(float(np.median(v)), 3) for k, v in res.items()},
                          "range": {k: [round(min(v), 3), round(max(v), 3)] for k, v in res.items()},
                          "gpu": gpu_info()}), flush=True)
    env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--workload", choices=["quad", "maze", "gru", "all"], default="all")
    args = ap.parse_args()
    plan = {"quad": [1, 64, 1024, 2048], "maze": [128, 512], "gru": [128]}
    for w in (plan if args.workload == "all" else [args.workload]):
        bench(w, plan[w], args.rounds)


if __name__ == "__main__":
    main()
