"""Recurrent policy-driven rollouts: the fused MetaMaze2D rollout with a GRU or an LSTM evaluated in the launch, against
what a user does without it.
Shape: MetaMaze2D SURVIVAL 15x15, 16 384 envs, view_grid 1, auto-reset, T = 32, GRUCell(9 + 5, 64) (--cell gru, the
default) or LSTMCell(9 + 5, 64) (--cell lstm) with feedback (onehot prev action, prev reward), head Linear(64, 4),
categorical, hidden_reset "task"; without and with in-launch task resampling (one table slot per env).
Three arms, timed as scripts/bench_policy_rollout.py times them (CUDA events, median over alternating rounds):
  (a) fused    rollout(T, policy=GRUPolicy|LSTMPolicy, state=s[, resample=...])    one launch, hid not recorded
  (b) torch    T x (step() + the same cell and head in torch + the same sampling and log-prob + the carried state's
               feedback and reset masking [+ resample_tasks(done) + reset(mask=done)]), one CUDA graph, allow_tf32 off
  (c) open     rollout(T[, resample=...]) with device-drawn actions     the ceiling: the env alone
Achieved FLOP/s of (a) counts 2 flops per multiply-add of the cell and head, from the shapes.  Writes JSON (card name
and power limit read in the same run) to --out and prints it.

usage: python scripts/bench_rnn_policy_rollout.py [--cell gru|lstm] [--T 32] [--rounds 7] [--iters 20] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_policy_rollout import card, graph_of, time_arms  # noqa: E402

D, H = 9, 64


def fma_per_env_step(obs_dim, hidden, feedback=True, head_width=0, gates=3):
    """Multiply-adds of one cell step and its head: gates H (in + H) for the cell (3 for the GRU, 4 for the LSTM), then
    the head's layers."""
    n_in = obs_dim + 5 * feedback
    head = hidden * head_width + head_width * 4 if head_width else hidden * 4
    return gates * hidden * (n_in + hidden) + head


def maze_shape(torch, nn, args, resample):
    from metagym_b200 import BatchedMetaMaze2D, MazeTaskSampler
    from metagym_b200.policy import GRUPolicy, LSTMPolicy
    import numpy as np
    lstm = args.cell == "lstm"
    M = 2 * H if lstm else H            # state entries before the feedback: [h, c] or [h]
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
    cell = (nn.LSTMCell if lstm else nn.GRUCell)(D + 5, H).to(dev)
    head = nn.Linear(H, 4).to(dev)
    policy = (LSTMPolicy if lstm else GRUPolicy)(cell, head, feedback=True, hidden_reset="task", device=dev)
    env_a, env_b, env_c = make_env(), make_env(), make_env()
    f = lambda *s, **k: torch.empty(s, device=dev, **k)          # noqa: E731
    state_a = policy.initial_state(N)
    out_a = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8),
             "act": f(T, N, dtype=torch.int32), "logp": f(T, N), "obs0": f(N, 3, 3), "state0": f(N, M + 5)}
    out_c = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8), "act": None}
    buf = {"obs": f(T, N, 3, 3), "rew": f(T, N, dtype=torch.float64), "done": f(T, N, dtype=torch.uint8),
           "act": f(T, N, dtype=torch.int32), "logp": f(T, N)}
    cur = env_b._obs.clone()
    state_b = policy.initial_state(N)
    eye = torch.eye(4, device=dev)

    def steps_b():
        x, s = cur, state_b
        for t in range(T):
            with torch.no_grad():
                xin = torch.cat([x.reshape(N, D), s[:, M:]], 1)
                if lstm:
                    h, c = cell(xin, (s[:, :H], s[:, H:M]))
                else:
                    h = cell(xin, s[:, :H])
                lsm = torch.log_softmax(head(h), -1)
                u = torch.rand((N, 1), device=dev)
                a = (u >= lsm.exp().cumsum(-1)[:, :3]).sum(-1).to(torch.int32)       # inverse CDF
                buf["act"][t].copy_(a)
                buf["logp"][t].copy_(lsm.gather(-1, a.long()[:, None])[:, 0])
            o, r, d, _ = env_b.step(a)
            with torch.no_grad():
                s = torch.cat([h, c, eye[a.long()], r.float()[:, None]] if lstm else
                              [h, eye[a.long()], r.float()[:, None]], 1)
                if resample:             # the task rule: a done env drew a new maze, its memory starts over
                    s = s * (d == 0)[:, None]
            if resample:
                env_b.resample_tasks(d, **rs)
                o = env_b.reset(mask=d)
            buf["obs"][t].copy_(o)
            buf["rew"][t].copy_(r)
            buf["done"][t].copy_(d)
            x = buf["obs"][t]
        cur.copy_(x)
        state_b.copy_(s)

    arms = {"a_policy_rollout": lambda: env_a.rollout(T, policy=policy, state=state_a, act_seed=1, out=out_a,
                                                      resample=rs),
            "b_torch_graph": graph_of(torch, steps_b),
            "c_open_loop_rollout": lambda: env_c.rollout(T, act_seed=2, out=out_c, resample=rs)}
    res = time_arms(torch, args, arms, N * T, {"env": "MetaMaze2D SURVIVAL 15x15", "envs": N, "view_grid": 1, "T": T,
                                               "resample": resample,
                                               "policy": "%s(14, 64) + Linear(64, 4), feedback, task reset"
                                                         % ("LSTMCell" if lstm else "GRUCell")})
    fma = fma_per_env_step(D, H, gates=4 if lstm else 3)
    res["fma_per_env_step"] = fma
    res["a_achieved_flop_per_s"] = 2.0 * fma * N * T / res["arms"]["a_policy_rollout"]["median_s_per_call"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cell", choices=("gru", "lstm"), default="gru")
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import torch.nn as nn
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    res = {"card": card(), "cell": args.cell, "rounds": args.rounds, "iters_per_round": args.iters, "shapes": []}
    for resample in (False, True):
        res["shapes"].append(maze_shape(torch, nn, args, resample))
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
