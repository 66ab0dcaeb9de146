"""Measure (on an H100) how fast the GPU quadrotor drifts from the reference's golden free-running
episodes, and write the running-max curve tests/test_quadrotor_gpu.py asserts against (x2).

    python tests/golden/measure_free_run_envelope.py          # rewrites tests/golden/free_run_envelope.json

Error metric = tests/util.py group_rel_err over the 16 sensor observations (per physical vector, angles against 1 rad,
z against its 5 m offset).  curve[j] = max over the recorded episodes of the error at step j of an episode, made
monotone (running max): a free run can only be asserted as tightly as its worst earlier step.
Also records the same curve for the CPU oracle in float64 (the reference's own float32 noise: SURVEY.md 8c).
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import numpy as np
import torch
from metagym_b200 import BatchedQuadrotor
from util import OBS_GROUPS, golden_run, group_rel_err

g = np.load(os.path.join(HERE, "quadrotor_golden.npz"))
RUNS = ["hover_a", "hover_fall", "nocol_a", "vel_a", "vel_c"]
curve = np.zeros(0)
per_run = {}
for name in RUNS:
    r = golden_run(g, name)
    kw = dict(dt=r["dt"], nt=r["nt"])
    if r["task"] == "velocity_control":
        kw["seed"] = r["seed"]
    env = BatchedQuadrotor(task=r["task"], num_envs=1, device=0, squeeze=False, **kw)
    ep = r["ep"]
    errs = []
    for k in range(int(ep.max()) + 1):
        idx = np.nonzero(ep == k)[0]
        env.reset(noise=r["reset_noise"][k][None])
        for j, i in enumerate(idx):
            obs, rew, done, _ = env.step(torch.as_tensor(r["act"][i][None]).cuda())
            e = group_rel_err(obs.cpu().numpy()[:, :16], r["obs"][i][None, :16], OBS_GROUPS)
            if j >= len(errs):
                errs.append(e)
            else:
                errs[j] = max(errs[j], e)
    env.close()
    per_run[name] = errs
    if len(errs) > len(curve):
        curve = np.concatenate([curve, np.zeros(len(errs) - len(curve))])
    curve[:len(errs)] = np.maximum(curve[:len(errs)], errs)
mono = np.maximum.accumulate(curve)
# ---- the same for test_random_batch_vs_oracle: 4096 envs, 20 free steps, actions U(-1, 16), vs the CPU oracle (mix mode)
from oracle import quad_oracle as qo
cfg = qo.make_cfg()
batch = np.zeros(20)
for task, dt in (("hovering_control", 0.01), ("velocity_control", 0.005), ("no_collision", 0.01)):
    for n in (1, 127, 129, 4096):
        rng = np.random.RandomState(1234 + n)
        nt = 30
        env = BatchedQuadrotor(task=task, num_envs=n, device=0, squeeze=False, dt=dt, nt=nt, seed=[0, 1, 2])
        noise = rng.random_sample((n, 12))
        env.reset(noise=noise)
        state = qo.reset_state(None, noise)
        ct = np.zeros(n, np.int32)
        kw = {}
        if task == "velocity_control":
            kw = dict(targets=env.velocity_targets.cpu().numpy(), env2task=env.env2task.cpu().numpy())
        for t in range(20):
            act = rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32)
            obs, rew, done, _ = env.step(torch.as_tensor(act).cuda())
            o_ref = qo.env_step(cfg, state, ct, act, task, dt, nt, mode="mix", **kw)[0]
            batch[t] = max(batch[t], group_rel_err(obs.cpu().numpy()[:, :16], o_ref[:, :16], OBS_GROUPS))
        env.close()
batch = np.maximum.accumulate(batch)
# ---- the same for test_path_matrix_vs_oracle, indexed by steps since an env's last reset: its batches exactly (sizes,
# seeds, edge states, actions; every path computes the same bits, so the default kernel stands for all), observations
# and terminal observations of the followed envs
import tempfile  # noqa: E402
import test_quadrotor_gpu as tq  # noqa: E402
from util import group_rel_err_rows  # noqa: E402
matrix = np.zeros(20)
tmp = tempfile.mkdtemp()
for n in (4099, 9473, tq._stream_size()):
    for task, terrain in tq.MATRIX_TASKS:
        for config in ("default", "general"):
            for drawn in ((False, True) if n == 4099 else (False,)):
                env, ob, rng = tq._matrix_batch(n, task, terrain, config, g["map_obst"], tmp)
                rows, since = ob.idx, np.zeros(ob.idx.size, np.int64)
                acts = [rng.uniform(-1.0, 16.0, (n, 4)).astype(np.float32) for _ in range(20)]
                outs = []
                if drawn:
                    for t0 in (0, 10):
                        o = env.rollout(10, act_seed=tq.MATRIX_ACT_SEED, want_actions=True)
                        for t in range(10):
                            acts[t0 + t] = o["act"][t].cpu().numpy()
                            outs.append((o["obs"][t].cpu().numpy(), o["done"][t].cpu().numpy(), None))
                for t in range(20):
                    if not drawn:
                        obs, _, done, _ = env.step(torch.as_tensor(acts[t]).cuda())
                        outs.append((obs.cpu().numpy(), done.cpu().numpy(), env.final_observation.cpu().numpy()))
                    r = ob.step(acts[t])
                    o, d, f = outs[t]
                    o, d = o[rows], d[rows].astype(bool)
                    assert np.array_equal(d, r.done), (n, task, terrain, config, t)
                    e = group_rel_err_rows(o[~d, :16], r.obs[~d, :16], OBS_GROUPS)
                    np.maximum.at(matrix, since[~d], e)
                    if f is not None:
                        np.maximum.at(matrix, since[d], group_rel_err_rows(f[rows][d, :16], r.final_obs[d, :16],
                                                                           OBS_GROUPS))
                    since = np.where(d, 0, since + 1)
                env.close()
matrix = np.maximum.accumulate(matrix)
out = {"random_batch_vs_oracle_running_max": [float(x) for x in batch],
       "path_matrix_running_max": [float(x) for x in matrix], "metric": "group_rel_err over obs[:16] (tests/util.py), GPU free run vs reference golden episodes",
       "runs": RUNS, "curve_running_max": [float(x) for x in mono], "per_run_max": {k: float(max(v)) for k, v in per_run.items()},
       "per_run_len": {k: len(v) for k, v in per_run.items()}, "device": torch.cuda.get_device_name(0)}
with open(os.path.join(HERE, "free_run_envelope.json"), "w") as f:
    json.dump(out, f)
print("steps", len(mono), "err@1,10,50,100,end:", [float(mono[min(i, len(mono) - 1)]) for i in (0, 9, 49, 99, len(mono) - 1)])
print(out["per_run_max"])
print("random batch vs oracle, err@1,5,10,20:", [float(batch[i]) for i in (0, 4, 9, 19)])
print("path matrix, err by steps since reset:", [float(x) for x in matrix[:7]])
