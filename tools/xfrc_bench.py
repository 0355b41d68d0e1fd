"""Cost of external body wrenches (HumanoidBatchB200.xfrc_applied) on the cfg2 workload: 4 096 SMPL envs, speed task, uhc_pd,
15 substeps per env step, autoreset.  Three modes:

  none  xfrc_applied = None (the kernel without the wrench code)
  zero  an all-zero [N, nbody, 6] tensor: the mechanism's own cost (the wrench instance of the kernel, loads of zeros)
  push  a push schedule: every env gets a 300 N horizontal force on the pelvis for one env step every 60 steps, phases and
        directions from a seeded RNG (this changes the physics: pushed humanoids stumble and touch the floor more)

`none` and `zero` alternate three times in one process; `push` runs once.  Each run: fresh batch, reset, warm-up steps, then the
timed steps (CUDA events around step + autoreset), then the mean k_step5 launch time over 50 steps (events around `step`).  Prints
one JSON line per run and a summary line with the card name and power limit, read in the same process.  Needs a CUDA device.

    python tools/xfrc_bench.py [--envs 4096] [--steps 200] [--warmup 20] [--out DIR]
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
PUSH_N, PUSH_EVERY = 300.0, 60


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def run(mode, N, K, W):
    dev = torch.device("cuda:0")
    env = HumanoidBatchB200(make_cfg(env="speed"), num_envs=N, device="cuda:0", seed=0, with_aux=False)
    nb, nu = env.model.nbody, env.num_actions
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    xf = None
    if mode != "none":
        xf = torch.zeros(N, nb, 6, dtype=torch.float32, device=dev)
        env.xfrc_applied = xf
    rng = np.random.default_rng(0)
    phase = torch.as_tensor(rng.integers(0, PUSH_EVERY, N), device=dev)
    ang = rng.uniform(0, 2 * np.pi, N)
    push = torch.as_tensor(np.stack([np.cos(ang), np.sin(ang)], 1) * PUSH_N, dtype=torch.float32, device=dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2

    def one(t, a):
        if mode == "push":
            on = ((phase + t) % PUSH_EVERY == 0).to(torch.float32)[:, None]
            xf[:, 0, 0:2] = push * on
        env.step(a)
        env.reset_done()

    env.reset()
    acts = torch.clamp(torch.randn(W, N, nu, generator=gen, device=dev) * SIGMA, -1, 1)
    for i in range(W):
        one(i, acts[i]); flush.zero_()
    acts = torch.clamp(torch.randn(K, N, nu, generator=gen, device=dev) * SIGMA, -1, 1)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(K):
        one(W + i, acts[i]); flush.zero_()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(50)]
    for i, (a, b) in enumerate(kev):
        if mode == "push":
            xf[:, 0, 0:2] = push * ((phase + W + K + i) % PUSH_EVERY == 0).to(torch.float32)[:, None]
        flush.zero_()
        a.record(); env.step(acts[i % K]); b.record()
        env.reset_done()
    torch.cuda.synchronize()
    k_ms = float(np.mean([a.elapsed_time(b) for a, b in kev]))
    return dict(mode=mode, envs=N, steps=K, env_steps_per_s=N * K / (ms / 1e3), ms_per_step=ms / K, k_step5_ms=k_ms,
                status_nonzero=int((env.status != 0).sum().item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/xfrc_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("xfrc_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    rows = []
    for mode in ["none", "zero"] * 3 + ["push"]:
        r = run(mode, args.envs, args.steps, args.warmup)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu}
    for mode in ("none", "zero", "push"):
        rs = [r for r in rows if r["mode"] == mode]
        summ[mode] = dict(env_steps_per_s=[round(r["env_steps_per_s"]) for r in rs], k_step5_ms=[round(r["k_step5_ms"], 4) for r in rs])
    a = np.median([r["k_step5_ms"] for r in rows if r["mode"] == "none"])
    b = np.median([r["k_step5_ms"] for r in rows if r["mode"] == "zero"])
    summ["zero_over_none_k_step5"] = round(float(b / a), 4)
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "xfrc_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
