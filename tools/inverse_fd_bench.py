"""Time of smplsim_inverse_fd (HumanoidBatchB200.inverse_fd) on the H100, against the same derivatives composed in torch from one
inverse() call on all perturbed rows.  Cases:

  invfd-smpl-{1,64,4096}  SMPL inverse_fd (centered, defaults): 1 + 450 inverse passes per row, in launches of 4 096 slots
  invfd-smplx-{1,256}     SMPL-X inverse_fd: 1 + 954 inverse passes per row

The torch baseline builds the 2 * 3nv perturbed rows of every state (the root rotation as q (x) exp(+-eps e_k)), calls inverse() once on
all of them (in launches of 4 096 rows), and divides the differences by the fp32 differences of the inputs.  Inputs are states with
floor contacts and joint-limit rows: each handle resets (Default init, speed task, stable PD) and takes 10 env steps; its (qpos, qvel,
aux.qacc) rows are then repeated, with seeded noise on the joint angles, up to the row count.  Each call is timed with CUDA events after
a 256 MiB L2 flush (as bench.py); reported: mean ms per call, rows/s and inverse passes/s of both, whether every column but the
root-rotation ones is bit-identical in both (same inputs, same pass), and the median difference of the root-rotation columns the kernel
does not flag, |k - t| / max(1, max |t|) (the two build the rotated quaternion with different fp32 roundings).  Prints one JSON line per case and a summary
line with the card name and power limit, read in the same process.  Needs a CUDA device.

    python tools/inverse_fd_bench.py [--reps 10] [--out DIR]
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

CASES = [("invfd-smpl-1", "smpl_humanoid", 1), ("invfd-smpl-64", "smpl_humanoid", 64), ("invfd-smpl-4096", "smpl_humanoid", 4096),
         ("invfd-smplx-1", "smplx_humanoid", 1), ("invfd-smplx-256", "smplx_humanoid", 256)]
EPS = HumanoidBatchB200.INVFD_EPS


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
    if rows > env.num_envs:
        q[env.num_envs:, 7:] += torch.randn(rows - env.num_envs, env.num_actions, generator=gen, device=dev) * 0.05
    return q, v, a


def qmul(a, b):
    w1, x1, y1, z1 = a.unbind(-1)
    w2, x2, y2, z2 = b.unbind(-1)
    return torch.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                        w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)


def composed(env, q, v, a):
    """dfrc [n, nv, 3nv] from one inverse() call on the 2 * 3nv perturbed rows of every state."""
    n, nv = v.shape
    nq, ncol, dev = nv + 1, 3 * nv, v.device
    Q = q[:, None, None].repeat(1, 2, ncol, 1)            # [n, sign, column, nq]
    V = v[:, None, None].repeat(1, 2, ncol, 1)
    A = a[:, None, None].repeat(1, 2, ncol, 1)
    sg = torch.tensor([1.0, -1.0], device=dev)
    lin = [j for j in range(nv) if not 3 <= j < 6]
    qi = torch.tensor([j if j < 3 else j + 1 for j in lin], device=dev)
    lj = torch.tensor(lin, device=dev)
    for s in range(2):
        Q[:, s, lj, qi] = Q[:, s, lj, qi] + sg[s] * EPS[0]
        k = torch.arange(nv, device=dev)
        V[:, s, nv + k, k] = V[:, s, nv + k, k] + sg[s] * EPS[1]
        A[:, s, 2 * nv + k, k] = A[:, s, 2 * nv + k, k] + sg[s] * EPS[2]
        for r in range(3):
            half = torch.tensor(0.5 * float(sg[s]) * EPS[0], device=dev)
            d = torch.zeros(4, device=dev); d[0] = torch.cos(half); d[1 + r] = torch.sin(half)
            qr = qmul(Q[:, s, 3 + r, 3:7], d.expand(n, 4))
            Q[:, s, 3 + r, 3:7] = qr / qr.norm(dim=-1, keepdim=True)
    f = env.inverse(Q.reshape(-1, nq), V.reshape(-1, nv), A.reshape(-1, nv)).reshape(n, 2, ncol, nv)
    den = torch.empty(n, ncol, device=dev)                 # the fp32 differences of the inputs loaded; 2 eps for the root rotation
    den[:, lj] = Q[:, 0, lj, qi] - Q[:, 1, lj, qi]
    den[:, 3:6] = 2 * torch.tensor(EPS[0], dtype=torch.float32)
    den[:, nv:2 * nv] = V[:, 0, nv:].diagonal(dim1=1, dim2=2) - V[:, 1, nv:].diagonal(dim1=1, dim2=2)
    den[:, 2 * nv:] = A[:, 0, 2 * nv:].diagonal(dim1=1, dim2=2) - A[:, 1, 2 * nv:].diagonal(dim1=1, dim2=2)
    return ((f[:, 0] - f[:, 1]) / den[:, :, None]).transpose(1, 2)


def timed(call, reps, flush):
    for _ in range(2):
        out = call()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = call(); e1.record()
    torch.cuda.synchronize()
    return out, [e0.elapsed_time(e1) for e0, e1 in ev]


def run(env, name, rows, reps, gen, flush):
    q, v, a = inputs(env, rows, gen)
    nv = env.model.nv
    out, ms = timed(lambda: env.inverse_fd(q, v, a), reps, flush)
    ref, tms = timed(lambda: composed(env, q, v, a), reps, flush)
    passes = rows * (1 + 2 * 3 * nv)
    lin = torch.ones(3 * nv, dtype=torch.bool, device=q.device)
    lin[3:6] = False
    exact = bool(torch.equal(out["dfrc"][:, :, lin], ref[:, :, lin]))    # the same inputs and the same inverse pass, bit for bit
    keep = (out["flags"] == 0)[:, None, 3:6]
    scale = ref[:, :, 3:6].abs().amax(dim=1, keepdim=True).clamp_min(1.0)
    d = (out["dfrc"][:, :, 3:6] - ref[:, :, 3:6]).abs() / scale
    rot = float(d[keep.expand_as(d)].median().item()) if bool(keep.any()) else 0.0
    km, tm = float(np.mean(ms)), float(np.mean(tms))
    return dict(case=name, rows=rows, inverse_passes=passes, ms_mean=km, ms_min=float(np.min(ms)), ms_max=float(np.max(ms)),
                rows_per_s=rows / (km / 1e3), passes_per_s=passes / (km / 1e3), torch_ms_mean=tm, torch_rows_per_s=rows / (tm / 1e3),
                speedup=tm / km, exact_non_rotation=exact, median_diff_rotation=rot, finite=bool(torch.isfinite(out["dfrc"]).all().item()),
                kink_columns=float((out["flags"] & 1).float().mean().item()), solver_columns=float((out["flags"] & 2).float().mean().item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/inverse_fd_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inverse_fd_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    envs = {r: HumanoidBatchB200(make_cfg(env="speed", robot=r), num_envs=4096, device="cuda:0", seed=0) for r in ("smpl_humanoid", "smplx_humanoid")}
    rows = []
    for name, robot, n in CASES:
        r = run(envs[robot], name, n, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), torch_ms=round(r["torch_ms_mean"], 4), exact=r["exact_non_rotation"]) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "inverse_fd_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
