"""Time of smplsim_forward (HumanoidBatchB200.forward) and smplsim_transition_fd (HumanoidBatchB200.transition_fd) on the H100.  Cases:

  fwd-smpl-4096       SMPL forward, 4 096 rows on a 4 096-env handle: one launch
  fwd-smpl-131072     SMPL forward, 131 072 rows: 32 launches of 4 096 rows on the stream
  fwd-smplx-4096      SMPL-X forward, 4 096 rows
  fwd-smplx-131072    SMPL-X forward, 131 072 rows
  fd-smpl-{1,64,4096} SMPL transition_fd (centered, defaults): 1 + 438 forward passes per row, in launches of 4 096 slots
  fd-smplx-{1,256}    SMPL-X transition_fd: 1 + 942 forward passes per row

Inputs are states with floor contacts and joint-limit rows: each handle resets (Default init, speed task, stable PD) and takes 10 env
steps; its (qpos, qvel, aux.ctrl) rows are then repeated, with seeded noise on the joint angles, up to the row count.  Each case warms up,
then times its calls with CUDA events, each after a 256 MiB L2 flush (as bench.py), and reports the mean ms per call, rows/s and forward
passes/s.  Prints one JSON line per case and a summary line with the card name and power limit, read in the same process.  Needs a
CUDA device.

    python tools/fd_bench.py [--reps 10] [--out DIR]
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

CASES = [("fwd-smpl-4096", "smpl_humanoid", "forward", 4096), ("fwd-smpl-131072", "smpl_humanoid", "forward", 131072),
         ("fwd-smplx-4096", "smplx_humanoid", "forward", 4096), ("fwd-smplx-131072", "smplx_humanoid", "forward", 131072),
         ("fd-smpl-1", "smpl_humanoid", "fd", 1), ("fd-smpl-64", "smpl_humanoid", "fd", 64), ("fd-smpl-4096", "smpl_humanoid", "fd", 4096),
         ("fd-smplx-1", "smplx_humanoid", "fd", 1), ("fd-smplx-256", "smplx_humanoid", "fd", 256)]


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
    u = env.ctrl.repeat(rep, 1)[:rows].clone()
    if rows > env.num_envs:
        q[env.num_envs:, 7:] += torch.randn(rows - env.num_envs, env.num_actions, generator=gen, device=dev) * 0.05
    return q, v, u


def run(env, name, kind, rows, reps, gen, flush):
    q, v, u = inputs(env, rows, gen)
    call = (lambda: env.forward(q, v, u)) if kind == "forward" else (lambda: env.transition_fd(q, v, u))
    for _ in range(2):
        out = call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = call(); e1.record()
    torch.cuda.synchronize()
    ms = [e0.elapsed_time(e1) for e0, e1 in ev]
    m = env.model
    passes = rows if kind == "forward" else rows * (1 + 2 * (2 * m.nv + m.nu))
    r = dict(case=name, rows=rows, forward_passes=passes, ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)),
             rows_per_s=rows / (float(np.mean(ms)) / 1e3), passes_per_s=passes / (float(np.mean(ms)) / 1e3),
             finite=bool(torch.isfinite(out["qacc"]).all().item()))
    if kind == "fd":
        f = out["flags"]
        r.update(finite=r["finite"] and bool(torch.isfinite(out["A"]).all().item()), kink_columns=float((f & 1).float().mean().item()),
                 solver_columns=float((f & 2).float().mean().item()))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/fd_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fd_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    envs = {r: HumanoidBatchB200(make_cfg(env="speed", robot=r), num_envs=4096, device="cuda:0", seed=0) for r in ("smpl_humanoid", "smplx_humanoid")}
    rows = []
    for name, robot, kind, n in CASES:
        r = run(envs[robot], name, kind, n, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), rows_per_s=round(r["rows_per_s"], 1)) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fd_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
