"""Time of smplsim_rollout (HumanoidBatchB200.rollout) against the host-loop workaround it replaces, on the H100.  Cases:

  mppi-smpl         MPPI / predictive sampling: 1 start state x 1 024 action sequences x 30 action steps (1 s), SMPL
  mjroll-smpl       MuJoCo's rollout shape: 256 rows x 450 ctrl substeps (mode "ctrl", nsub = 1: one mj_step per control row), SMPL
  batch-smpl        4 096 rows x 30 action steps, SMPL
  mppi-smplx        1 start state x 1 024 action sequences x 30 action steps, SMPL-X

The host loop is what a user could do before: a scratch batch with one env per row, set_state + qacc_warm, then one step / mj_step
launch per control row, copying qpos / qvel out after each.  Start states come from a handle that resets (Default init, speed task,
stable PD) and takes 10 env steps; action sequences are seeded normal noise (sigma 0.3, clamped), ctrl sequences the PD torques of the
start state plus seeded noise.  Each case first checks that the rollout's qpos / qvel are bit-identical with the host loop's on a fresh
scratch batch (empty working-set memory, as the rollout starts), then times both with CUDA events, each call after a 256 MiB L2 flush,
and reports the mean ms per call, row-steps/s and the speed-up.  The timed host loop reuses its scratch batch, whose working-set
memory then carries over from the previous repetition.  Prints one JSON line per case and a summary line with the card name and power
limit, read in the same process.  Needs a CUDA device.

    python tools/rollout_bench.py [--reps 5] [--out DIR]
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

# (name, robot, mode, start states, rows, steps)
CASES = [("mppi-smpl", "smpl_humanoid", "action", 1, 1024, 30), ("mjroll-smpl", "smpl_humanoid", "ctrl", 256, 256, 450),
         ("batch-smpl", "smpl_humanoid", "action", 4096, 4096, 30), ("mppi-smplx", "smplx_humanoid", "action", 1, 1024, 30)]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def inputs(robot, mode, starts, rows, T, gen):
    cfg = make_cfg(env="speed", robot=robot)
    src = HumanoidBatchB200(cfg, num_envs=starts, device="cuda:0", seed=0)
    dev = src.device
    src.reset()
    for _ in range(10):
        src.step(torch.clamp(torch.randn(starts, src.num_actions, generator=gen, device=dev) * 0.3, -1, 1))
        src.reset_done()
    rep = rows // starts
    q, v, w = (x.repeat_interleave(rep, 0).contiguous() for x in (src.qpos, src.qvel, src.qacc_warm))
    if mode == "action":
        u = torch.clamp(torch.randn(rows, T, src.num_actions, generator=gen, device=dev) * 0.3, -1, 1)
    else:
        u = src.ctrl.repeat_interleave(rep, 0)[:, None] + torch.randn(rows, T, src.num_actions, generator=gen, device=dev) * 5.0
    return cfg, q, v, w, u.contiguous()


def host_loop(env, q, v, w, u, mode, out):
    env.set_state(q, v)
    env.qacc_warm.copy_(w)
    for t in range(u.shape[1]):
        if mode == "action":
            env.step(u[:, t])
        else:
            env.mj_step(u[:, t], 1)
        out[0][:, t].copy_(env.qpos)
        out[1][:, t].copy_(env.qvel)


def timed(call, reps, flush):
    call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); call(); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def run(name, robot, mode, starts, rows, T, reps, gen, flush):
    cfg, q, v, w, u = inputs(robot, mode, starts, rows, T, gen)
    env = HumanoidBatchB200(cfg, num_envs=rows, device="cuda:0", seed=0)
    kw = dict(mode=mode, nsub=1 if mode == "ctrl" else None, qacc_warmstart=w)
    got = env.rollout(q, v, u, **kw)
    out = (torch.empty_like(got["qpos"]), torch.empty_like(got["qvel"]))
    host_loop(HumanoidBatchB200(cfg, num_envs=rows, device="cuda:0", seed=0), q, v, w, u, mode, out)   # a fresh scratch batch
    torch.cuda.synchronize()
    same = bool(torch.equal(got["qpos"], out[0]) and torch.equal(got["qvel"], out[1]))
    ms_roll = timed(lambda: env.rollout(q, v, u, **kw), reps, flush)
    scratch = HumanoidBatchB200(cfg, num_envs=rows, device="cuda:0", seed=0)
    ms_loop = timed(lambda: host_loop(scratch, q, v, w, u, mode, out), reps, flush)
    r, lp = float(np.mean(ms_roll)), float(np.mean(ms_loop))
    st = got["status"]
    return dict(case=name, robot=robot, mode=mode, rows=rows, steps=T, substeps_per_step=1 if mode == "ctrl" else int(env.envcfg.nsubsteps),
                rollout_ms=r, rollout_ms_min=float(np.min(ms_roll)), host_loop_ms=lp, host_loop_ms_min=float(np.min(ms_loop)),
                row_steps_per_s=rows * T / (r / 1e3), host_loop_row_steps_per_s=rows * T / (lp / 1e3), speedup=lp / r,
                bit_identical=same, status_rows=int((st != 0).any(1).sum().item()), finite=bool(torch.isfinite(got["qpos"]).all().item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/rollout_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rollout_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    rows = []
    for case in CASES:
        r = run(*case, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(rollout_ms=round(r["rollout_ms"], 3), host_loop_ms=round(r["host_loop_ms"], 3),
                                           speedup=round(r["speedup"], 2), bit_identical=r["bit_identical"]) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rollout_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
