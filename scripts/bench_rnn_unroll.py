"""The learner's recompute of a recurrent rollout: GRUPolicy / LSTMPolicy.unroll through the fused cell sequence against
the torch step loop it replaces (DESIGN.md "Fused unroll").

MetaMaze2D SURVIVAL 15x15, 16 384 envs, T = 32, GRUCell(14, 64) or LSTMCell(14, 64), Linear(64, 4) and a value head
Linear(64, 1), on one collected chunk.  ms per chunk, medians of alternating rounds (each timed over `reps` calls with
CUDA events), TF32 off:
  (a) fused      unroll(out, value=True) + backward of a fixed linear loss over logits, logp and value, eager
  (a_graph)      (a) captured in one CUDA graph
  (b) loop       _unroll_reference(out, value=True) + the same backward, eager
  (c) loop_graph (b) captured in one CUDA graph
  and each of them forward-only under no_grad (*_fwd), and the fused rollout that collected the chunk, for scale.
Also each kernel alone (mgb_rnn_seq_forward saving the gates, mgb_rnn_seq_backward) with its achieved FLOP/s, from the
cell's multiply-adds: forward 2 G H (in + H) per env-step (both gate GEMVs), backward 2 G H H (W_hh^T dG).
Prints one JSON line per cell with the GPU name and power limit read in the same run.
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
T, N, H = 32, 16384, 64


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
    return start.elapsed_time(end) / reps          # ms per call


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


def seeded(m, seed, scale=0.2):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * scale)
    return m.cuda()


def make_env():
    from metagym_b200 import BatchedMetaMaze2D, MazeTaskSampler
    rng = np.random.RandomState(0)
    tasks = [MazeTaskSampler(n=15, food_density=0.05, food_interval=4, rng=rng) for _ in range(64)]
    env = BatchedMetaMaze2D(max_steps=200, task_type="SURVIVAL", view_grid=1, num_envs=N, device=0, squeeze=False,
                            auto_reset=True)
    env.set_task(tasks)
    env.reset()
    return env


def bench(kind, rounds, reps):
    from metagym_b200 import GRUPolicy, LSTMPolicy, _lib, cell_seq
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    env = make_env()
    cls, cell = (GRUPolicy, nn.GRUCell) if kind == "gru" else (LSTMPolicy, nn.LSTMCell)
    c, head, value = seeded(cell(14, 64), 1), seeded(nn.Linear(64, 4), 2), seeded(nn.Linear(64, 1), 3)
    pol = cls(c, head, device=env.device, value=value)
    assert cell_seq.fits(c)
    st = pol.initial_state(N)
    env.rollout(T, policy=pol, state=st)                 # a chunk from a carried, non-zero state
    out = env.rollout(T, policy=pol, state=st)
    params = [p for m in (c, head, value) for p in m.parameters()]
    g = torch.Generator(device="cuda").manual_seed(4)
    w = [torch.randn((T, N, 4), generator=g, device="cuda"), torch.randn((T, N), generator=g, device="cuda"),
         torch.randn((T, N), generator=g, device="cuda")]

    def train(fn):
        def step():
            res = fn(out, True)
            torch.autograd.grad(sum((r * x).sum() for r, x in zip(res, w)), params)
        return step

    def infer(fn):
        def step():
            with torch.no_grad():
                fn(out, True)
        return step

    st_r = pol.initial_state(N)
    out_r = env.rollout(T, policy=pol, state=st_r)
    arms = {"a_fused": train(pol.unroll), "a_fused_graph": graph_of(train(pol.unroll)),
            "b_loop": train(pol._unroll_reference), "c_loop_graph": graph_of(train(pol._unroll_reference)),
            "a_fused_fwd": infer(pol.unroll), "a_fused_graph_fwd": graph_of(infer(pol.unroll)),
            "b_loop_fwd": infer(pol._unroll_reference), "c_loop_graph_fwd": graph_of(infer(pol._unroll_reference)),
            "rollout_graph": graph_of(lambda: env.rollout(T, policy=pol, state=st_r, out=out_r))}

    # the two kernels alone, on the chunk's inputs
    obs, act, rew, wipe, state0 = pol._unroll_inputs(out)
    X = pol._cell_input(obs, act, rew, wipe, state0).transpose(1, 2).contiguous()
    wipe = wipe.contiguous()
    HC = pol._memory * H
    s0 = state0[:, :HC].contiguous()
    params_c = cell_seq._packed(c.weight_ih, c.weight_hh, c.bias_ih, c.bias_hh).detach()
    code = pol._cell_code
    h, gates = cell_seq.forward(code, H, params_c, X, wipe, s0, save=True)
    G = 3 if kind == "gru" else 4
    dh = torch.randn((T, N, H), generator=g, device="cuda")
    dgi = torch.empty((T, G * H, N), device="cuda")
    dghn = torch.empty((T, H, N), device="cuda") if kind == "gru" else None
    ds0 = torch.empty_like(s0)
    seq = cell_seq._struct(code, H, params_c, X, wipe, s0, h, gates)
    seq.dh_dev, seq.dgi_dev, seq.dghn_dev, seq.dstate0_dev = dh.data_ptr(), dgi.data_ptr(), _lib.ptr(dghn), ds0.data_ptr()
    arms["kernel_forward"] = lambda: cell_seq.forward(code, H, params_c, X, wipe, s0, save=True)
    arms["kernel_backward"] = lambda: cell_seq._call(_lib.load().mgb_rnn_seq_backward, seq, X.device)

    for fn in arms.values():          # warm-up of every shape the timed window uses
        fn()
    torch.cuda.synchronize()
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            res[k].append(timed(fn, reps))
    med = {k: float(np.median(v)) for k, v in res.items()}
    n_in = 14
    flops = {"kernel_forward": 2.0 * G * H * (n_in + H) * T * N, "kernel_backward": 2.0 * G * H * H * T * N}
    saved = (T * (4 if kind == "gru" else 5) * H * N + T * N * H) * 4
    print(json.dumps({"cell": kind, "envs": N, "T": T, "H": H, "in": n_in,
                      "ms_per_chunk": {k: round(v, 4) for k, v in med.items()},
                      "range": {k: [round(min(v), 4), round(max(v), 4)] for k, v in res.items()},
                      "tflops": {k: round(f / (med[k] * 1e-3) / 1e12, 3) for k, f in flops.items()},
                      "c_over_a": round(med["c_loop_graph"] / med["a_fused"], 3),
                      "c_over_a_graph": round(med["c_loop_graph"] / med["a_fused_graph"], 3),
                      "a_over_rollout": round(med["a_fused"] / med["rollout_graph"], 3),
                      "saved_bytes_h_and_gates": saved, "fwd_bwd_smem_bytes": cell_seq.smem_bytes(G, H, n_in),
                      "gpu": gpu_info()}), flush=True)
    env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cell", choices=["gru", "lstm", "all"], default="all")
    args = ap.parse_args()
    for kind in ("gru", "lstm"):
        if args.cell in ("all", kind):
            bench(kind, args.rounds, args.reps)


if __name__ == "__main__":
    main()
