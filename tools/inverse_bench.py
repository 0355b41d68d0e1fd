"""Time and throughput of smplsim_inverse (HumanoidBatchB200.inverse) on the H100.  Cases:

  smpl-4096     SMPL, 4 096 rows on a 4 096-env handle: one launch
  smpl-4096-cw  the same with the per-body contact wrench output
  smpl-131072   SMPL, 131 072 rows on a 4 096-env handle: 32 launches of 4 096 rows on the stream
  smplx-4096    SMPL-X, 4 096 rows: one launch

Inputs are states with floor contacts and joint-limit rows: each handle resets (Default init, speed task, stable PD) and takes 10 env
steps; its (qpos, qvel, aux.qacc) rows are then repeated, with seeded noise on the joint angles and accelerations, up to the row count.
Each case warms up 3 calls, then times 20 calls with CUDA events, each after a 256 MiB L2 flush (as bench.py), and reports the mean ms
per call and rows/s.  Prints one JSON line per case and a summary line with the card name and power limit, read in the same process.
Needs a CUDA device.

    python tools/inverse_bench.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

CASES = [("smpl-4096", "smpl_humanoid", 4096, False), ("smpl-4096-cw", "smpl_humanoid", 4096, True),
         ("smpl-131072", "smpl_humanoid", 131072, False), ("smplx-4096", "smplx_humanoid", 4096, False)]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def inputs(env, rows, gen):
    dev = env.device
    env.reset()
    for _ in range(10):
        env.step(torch.clamp(torch.randn(env.num_envs, env.num_actions, generator=gen, device=dev) * 0.3, -1, 1))
        env.reset_done()
    rep = (rows + env.num_envs - 1) // env.num_envs
    q = env.qpos.repeat(rep, 1)[:rows].clone()
    v = env.qvel.repeat(rep, 1)[:rows].clone()
    a = env.qacc.repeat(rep, 1)[:rows].clone()
    q[env.num_envs:, 7:] += torch.randn(rows - env.num_envs, env.num_actions, generator=gen, device=dev) * 0.05
    a += torch.randn(a.shape, generator=gen, device=dev) * 2.0
    return q, v, a


def run(name, robot, rows, cw, reps, gen, flush):
    env = HumanoidBatchB200(make_cfg(env="speed", robot=robot), num_envs=4096, device="cuda:0", seed=0)
    q, v, a = inputs(env, rows, gen)
    for _ in range(3):
        env.inverse(q, v, a, contact_wrench=cw)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = env.inverse(q, v, a, contact_wrench=cw); e1.record()
    torch.cuda.synchronize()
    ms = [e0.elapsed_time(e1) for e0, e1 in ev]
    res = out[0] if cw else out
    wt = float(np.sum(env.model.body_mass)) * 9.81
    return dict(case=name, rows=rows, launches=(rows + 4095) // 4096, ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)),
                ms_max=float(np.max(ms)), rows_per_s=rows / (float(np.mean(ms)) / 1e3), finite=bool(torch.isfinite(res).all().item()),
                median_root_residual_over_weight=float(res[:, :6].abs().amax(1).median().item() / wt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/inverse_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inverse_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    rows = []
    for name, robot, n, cw in CASES:
        r = run(name, robot, n, cw, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), rows_per_s=round(r["rows_per_s"])) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "inverse_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
