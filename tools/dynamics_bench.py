"""Time and write bandwidth of smplsim_dynamics (HumanoidBatchB200.dynamics) on the H100.  Cases:

  smpl-4096-all     SMPL, 4 096 rows on a 4 096-env handle: M, qfrc_bias and the Jacobians of 5 bodies, one launch
  smpl-4096-M       the same, M only
  smpl-4096-bias    the same, qfrc_bias only
  smpl-4096-jac5    the same, Jacobians only: both hands, both feet (toes) and the head
  smpl-131072-all   SMPL, 131 072 rows on a 4 096-env handle, all outputs: 32 launches of 4 096 rows on the stream
  smplx-4096-all    SMPL-X, 4 096 rows, all outputs (wrists instead of hands)

Inputs are states with floor contact: each handle resets (Default init, speed task, stable PD) and takes 10 env steps; its (qpos, qvel)
rows are then repeated, with seeded noise on the joint angles, up to the row count.  Each case warms up 3 calls, then times 20 calls
with CUDA events, each after a 256 MiB L2 flush (as bench.py), and reports the mean ms per call, rows/s, the bytes the call must write
(outputs only) over its time, and that rate's share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  Prints one JSON line per
case and a summary line with the card name and power limit, read in the same process.  Needs a CUDA device.

    python tools/dynamics_bench.py [--reps 20] [--out DIR]
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

HBM_BPS = 3.35e12
BODIES = {"smpl_humanoid": ["L_Hand", "R_Hand", "L_Toe", "R_Toe", "Head"],
          "smplx_humanoid": ["L_Wrist", "R_Wrist", "L_Toe", "R_Toe", "Head"]}     # SMPL-X: the wrist bodies carry the fingers
# name, robot, rows, (mass_matrix, bias, jacobians)
CASES = [("smpl-4096-all", "smpl_humanoid", 4096, (True, True, True)), ("smpl-4096-M", "smpl_humanoid", 4096, (True, False, False)),
         ("smpl-4096-bias", "smpl_humanoid", 4096, (False, True, False)), ("smpl-4096-jac5", "smpl_humanoid", 4096, (False, False, True)),
         ("smpl-131072-all", "smpl_humanoid", 131072, (True, True, True)), ("smplx-4096-all", "smplx_humanoid", 4096, (True, True, True))]


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
    q[env.num_envs:, 7:] += torch.randn(rows - env.num_envs, env.num_actions, generator=gen, device=dev) * 0.05
    return q, v


def run(name, robot, rows, what, reps, gen, flush):
    env = HumanoidBatchB200(make_cfg(env="speed", robot=robot), num_envs=4096, device="cuda:0", seed=0)
    q, v = inputs(env, rows, gen)
    mm, bias, jac = what
    kw = dict(mass_matrix=mm, bias=bias, jac_bodies=BODIES[robot] if jac else None)
    for _ in range(3):
        env.dynamics(q, v, **kw)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = env.dynamics(q, v, **kw); e1.record()
    torch.cuda.synchronize()
    ms = [e0.elapsed_time(e1) for e0, e1 in ev]
    nv = env.model.nv
    wbytes = 4 * rows * ((nv * nv if mm else 0) + (nv if bias else 0) + (len(BODIES[robot]) * 6 * nv if jac else 0))
    t = float(np.mean(ms)) / 1e3
    return dict(case=name, rows=rows, launches=(rows + 4095) // 4096, ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)),
                ms_max=float(np.max(ms)), rows_per_s=rows / t, write_bytes=wbytes, write_GBps=wbytes / t / 1e9,
                write_share_of_hbm_peak=wbytes / t / HBM_BPS, finite=all(bool(torch.isfinite(x).all().item()) for x in out.values()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/dynamics_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("dynamics_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    rows = []
    for name, robot, n, what in CASES:
        r = run(name, robot, n, what, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), write_share=round(r["write_share_of_hbm_peak"], 3)) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dynamics_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
