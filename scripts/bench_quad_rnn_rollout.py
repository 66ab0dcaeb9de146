"""Recurrent quadrotor policy rollouts: the fused rollout with a GRU or an LSTM and a Gaussian head evaluated in the
launch, against what a user does without it.
Shape: velocity_control, dt 0.005, nt 1000, 64 velocity tasks, auto-reset, T = 32; N = 16 384 and 65 536 envs (--envs);
policies GRUCell(19 + 5, 64), LSTMCell(19 + 5, 64) and GRUCell(19 + 5, 32) (--cells), each with feedback (the raw
previous action and reward), head Linear(H, 4) and log_std.
Three arms, timed as scripts/bench_policy_rollout.py times them (CUDA events, median over alternating rounds):
  (a) fused    rollout(T, policy=GRUPolicy|LSTMPolicy(dist="gaussian"), state=s)    one launch, hid not recorded
  (b) torch    T x (step() + the same cell and head in torch + Gaussian sampling and log-prob + the carried state's
               feedback and masking), one CUDA graph, allow_tf32 off
  (c) open     rollout(T) with device-drawn actions     the ceiling: the env alone
Achieved FLOP/s counts 2 flops per multiply-add of the cell and head, from the shapes, over the arm's time.  Writes
JSON (card name and power limit read in the same run) to --out and prints it.

usage: python scripts/bench_quad_rnn_rollout.py [--envs 16384,65536] [--cells gru64,lstm64,gru32] [--T 32]
                                                [--rounds 7] [--iters 20] [--out FILE]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_policy_rollout import card, graph_of, time_arms  # noqa: E402
from bench_rnn_policy_rollout import fma_per_env_step  # noqa: E402

D = 19
CELLS = {"gru64": ("gru", 64), "lstm64": ("lstm", 64), "gru32": ("gru", 32)}
LOG_STD = (-1.0, -1.0, -1.0, -1.0)


def quad_shape(torch, nn, args, N, name):
    from metagym_b200 import BatchedQuadrotor
    from metagym_b200.policy import LOG_2PI_2, GRUPolicy, LSTMPolicy
    kind, H = CELLS[name]
    lstm = kind == "lstm"
    M = 2 * H if lstm else H            # state entries before the feedback: [h, c] or [h]
    T, dev = args.T, torch.device("cuda", 0)

    def make_env():
        env = BatchedQuadrotor(task="velocity_control", dt=0.005, nt=1000, seed=list(range(64)), num_envs=N, device=0,
                               squeeze=False, auto_reset=True)
        env.reset()
        return env

    torch.manual_seed(1)
    cell = (nn.LSTMCell if lstm else nn.GRUCell)(D + 5, H).to(dev)
    head = nn.Linear(H, 4).to(dev)
    with torch.no_grad():
        head.bias.add_(7.5)             # mid-range voltages
    log_std = torch.tensor(LOG_STD, device=dev)
    policy = (LSTMPolicy if lstm else GRUPolicy)(cell, head, log_std=log_std, dist="gaussian", device=dev)
    env_a, env_b, env_c = make_env(), make_env(), make_env()
    f = lambda *s, **k: torch.empty(s, device=dev, **k)          # noqa: E731
    state_a = policy.initial_state(N)
    out_a = {"obs": f(T, N, D), "rew": f(T, N), "done": f(T, N, dtype=torch.uint8), "act": f(T, N, 4),
             "logp": f(T, N), "obs0": f(N, D), "state0": f(N, M + 5)}
    out_c = {"obs": f(T, N, D), "rew": f(T, N), "done": f(T, N, dtype=torch.uint8), "act": None}
    buf = {"obs": f(T, N, D), "rew": f(T, N), "done": f(T, N, dtype=torch.uint8), "act": f(T, N, 4), "logp": f(T, N)}
    cur = env_b._obs.clone()
    state_b = policy.initial_state(N)
    std = log_std.exp()

    def steps_b():
        x, s = cur, state_b
        for t in range(T):
            with torch.no_grad():
                xin = torch.cat([x, s[:, M:]], 1)
                if lstm:
                    h, c = cell(xin, (s[:, :H], s[:, H:M]))
                else:
                    h = cell(xin, s[:, :H])
                z = torch.randn((N, 4), device=dev)
                a = head(h) + std * z
                buf["act"][t].copy_(a)
                buf["logp"][t].copy_((-0.5 * z * z - log_std).sum(-1) - LOG_2PI_2)
            o, r, d, _ = env_b.step(a)
            with torch.no_grad():
                s = torch.cat([h, c, a, r[:, None]] if lstm else [h, a, r[:, None]], 1) * (~d)[:, None]
            buf["obs"][t].copy_(o)
            buf["rew"][t].copy_(r)
            buf["done"][t].copy_(d)
            x = buf["obs"][t]
        cur.copy_(x)
        state_b.copy_(s)

    arms = {"a_policy_rollout": lambda: env_a.rollout(T, policy=policy, state=state_a, act_seed=1, out=out_a),
            "b_torch_graph": graph_of(torch, steps_b),
            "c_open_loop_rollout": lambda: env_c.rollout(T, act_seed=2, out=out_c)}
    res = time_arms(torch, args, arms, N * T, {"env": "quadrotor velocity_control dt 0.005 nt 1000", "envs": N, "T": T,
                                               "policy": "%s(24, %d) + Linear(%d, 4), feedback, log_std"
                                                         % ("LSTMCell" if lstm else "GRUCell", H, H)})
    fma = fma_per_env_step(D, H, gates=4 if lstm else 3)
    res["fma_per_env_step"] = fma
    for k in ("a_policy_rollout", "b_torch_graph"):
        res[k[:1] + "_achieved_flop_per_s"] = 2.0 * fma * N * T / res["arms"][k]["median_s_per_call"]
    for e in (env_a, env_b, env_c):
        e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="16384,65536")
    ap.add_argument("--cells", default="gru64,lstm64,gru32")
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
    from metagym_b200 import _lib
    res = {"card": card(), "cta_envs": _lib.QUAD_RNN_CTA_ENVS, "rounds": args.rounds, "iters_per_round": args.iters,
           "shapes": []}
    for N in (int(v) for v in args.envs.split(",")):
        for name in args.cells.split(","):
            res["shapes"].append(quad_shape(torch, nn, args, N, name))
            torch.cuda.empty_cache()
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
