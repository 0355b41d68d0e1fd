"""Time of smplsim_rne_post (HumanoidBatchB200.rne_post) on the H100, against smplsim_inverse with contact_wrench on the same rows.
Both run S1 (kinematics, velocities, floor contacts and joint-limit rows) and the outward acceleration sweep; the inverse then runs
its inward force sweep, rne_post its per-body subtree sums and outputs.  Cases:

  smpl-4096-all     SMPL, 4 096 rows on a 4 096-env handle: body_acc, joint_wrench and one IMU site at every body frame
                    (imu_sites="bodies": accelerometer, gyro, force, torque)
  smpl-4096-jw      the same rows, joint_wrench only
  smplx-4096-all    SMPL-X, 4 096 rows, all outputs as smpl-4096-all
  smplx-4096-jw     the same rows, joint_wrench only

Baseline per case: inverse(qpos, qvel, qacc, contact_wrench=True) on the same rows.

Inputs are states with floor contact: each handle resets (Default init, speed task, stable PD) and takes 10 env steps; its (qpos, qvel,
qacc) rows are those of the last step.  Each case warms up 3 calls, then times 20 calls with CUDA events, each after a 256 MiB L2
flush (as bench.py), and reports the mean ms per call and rows/s.  Prints one JSON line per case and a summary line with the card name,
power limit and SM clock cap, read in the same process.  Needs a CUDA device.

    python tools/rne_post_bench.py [--reps 20] [--out DIR]
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

# name, robot, rne_post keywords
CASES = [("smpl-4096-all", "smpl_humanoid", dict(imu_sites="bodies")), ("smpl-4096-jw", "smpl_humanoid", dict(acc=False)),
         ("smplx-4096-all", "smplx_humanoid", dict(imu_sites="bodies")), ("smplx-4096-jw", "smplx_humanoid", dict(acc=False))]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def inputs(env, gen):
    dev = env.device
    env.reset()
    for _ in range(10):
        env.step(torch.clamp(torch.randn(env.num_envs, env.num_actions, generator=gen, device=dev) * 0.3, -1, 1))
        env.reset_done()
    return env.qpos_fwd.clone(), env.qvel_fwd.clone(), env.qacc.clone()


def timed(fn, reps, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = fn(); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev], out


def run(name, robot, kw, reps, gen, flush):
    env = HumanoidBatchB200(make_cfg(env="speed", robot=robot), num_envs=4096, device="cuda:0", seed=0)
    q, v, a = inputs(env, gen)
    rows = q.shape[0]
    ms, out = timed(lambda: env.rne_post(q, v, a, **kw), reps, flush)
    bms, _ = timed(lambda: env.inverse(q, v, a, contact_wrench=True), reps, flush)
    return dict(case=name, rows=rows, outputs=list(out), ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)),
                rows_per_s=rows / (float(np.mean(ms)) / 1e3), inverse_ms_mean=float(np.mean(bms)),
                ratio_to_inverse=float(np.mean(ms)) / float(np.mean(bms)),
                finite=all(bool(torch.isfinite(x).all().item()) for x in out.values()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/rne_post_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rne_post_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    rows = []
    for name, robot, kw in CASES:
        r = run(name, robot, kw, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), inverse_ms=round(r["inverse_ms_mean"], 4),
                                           ratio=round(r["ratio_to_inverse"], 2)) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rne_post_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
