"""Cost of the per-body contact wrench output (HumanoidBatchB200(contact_wrench=True)) on the cfg2 workload: 4 096 SMPL envs, speed
task, uhc_pd, 15 substeps per env step, autoreset.  Two modes:

  off  contact_wrench=False: the output pointer is NULL and the step kernel skips it
  on   contact_wrench=True: after the last substep the kernel writes [N, nbody, 6] from the contact list of that forward pass

The modes alternate three times in one process.  Each run: fresh batch, reset, warm-up steps, then the timed steps (CUDA events around
step + autoreset, a 256 MiB L2 flush after every step as in bench.py), then the mean k_step5 launch time over 50 steps (events around
`step`).  Prints one JSON line per run and a summary line with the card name and power limit, read in the same process.  Needs a
CUDA device.

    python tools/contact_wrench_bench.py [--envs 4096] [--steps 200] [--warmup 20] [--out DIR]
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

SIGMA = float(np.exp(-2.5))          # the action noise of bench.py (learning/simple_mlp.yaml fixed log_std)


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def run(mode, N, K, W):
    dev = torch.device("cuda:0")
    env = HumanoidBatchB200(make_cfg(env="speed"), num_envs=N, device="cuda:0", seed=0, with_aux=False, contact_wrench=(mode == "on"))
    nu = env.num_actions
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2

    def one(a):
        env.step(a)
        env.reset_done()

    env.reset()
    acts = torch.clamp(torch.randn(W, N, nu, generator=gen, device=dev) * SIGMA, -1, 1)
    for i in range(W):
        one(acts[i]); flush.zero_()
    acts = torch.clamp(torch.randn(K, N, nu, generator=gen, device=dev) * SIGMA, -1, 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K):
        one(acts[i]); flush.zero_()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(50)]
    for i, (a, b) in enumerate(kev):
        flush.zero_()
        a.record(); env.step(acts[i % K]); b.record()
        env.reset_done()
    torch.cuda.synchronize()
    k_ms = float(np.mean([a.elapsed_time(b) for a, b in kev]))
    r = dict(mode=mode, envs=N, steps=K, env_steps_per_s=N * K / (ms / 1e3), ms_per_step=ms / K, k_step5_ms=k_ms,
             status_nonzero=int((env.status != 0).sum().item()))
    if env.contact_wrench is not None:      # plausibility: mean vertical contact force per env over the humanoid's weight
        fz = env.contact_wrench[:, :, 2].sum(1)
        r["mean_fz_over_weight"] = float(fz.mean().item() / (float(np.sum(env.model.body_mass)) * 9.81))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/contact_wrench_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("contact_wrench_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    rows = []
    for mode in ["off", "on"] * 3:
        r = run(mode, args.envs, args.steps, args.warmup)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu}
    for mode in ("off", "on"):
        rs = [r for r in rows if r["mode"] == mode]
        summ[mode] = dict(env_steps_per_s=[round(r["env_steps_per_s"]) for r in rs], k_step5_ms=[round(r["k_step5_ms"], 4) for r in rs])
    a = np.median([r["k_step5_ms"] for r in rows if r["mode"] == "off"])
    b = np.median([r["k_step5_ms"] for r in rows if r["mode"] == "on"])
    summ["on_over_off_k_step5"] = round(float(b / a), 4)
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "contact_wrench_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
