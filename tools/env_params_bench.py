"""Cost of per-env physics parameters (HumanoidBatchB200.set_env_params).  Step-kernel time of

  cfg2  4 096 SMPL envs, speed task, uhc_pd (stable PD, stale inertia), 15 substeps per env step, autoreset
  cfg5  4 096 SMPL-X envs, getup task (Fall init), uhc_pd

in these modes, alternated three times for cfg2 and once for cfg5 in one process:

  none  no records: the kernels without the parameter reads (what every batch ran before records existed)
  nominal  records holding the model's values: the parameter instances on the same physics as `none` (bit-identical results), so
        nominal / none is the mechanism's own cost
  xfrc0  no records, an all-zero xfrc_applied: the wrench instance the records' step instance is built on, for attribution
  rand  every env with its own draws: friction U(0.4, 1.6), kp / kd / torque limit x U(0.6, 1.4), mass scale U(0.7, 1.3) per body,
        gravity + U(-0.5, 0.5) per component (this changes the physics, so the contact work differs a little from `none`)

Each run: fresh batch, reset, warm-up steps, then the mean step time over 50 env steps (CUDA events around `step`, an L2 flush
between steps).  Also times one set_env_params over all envs: the whole Python call (validation with its host sync) and the
record-writing kernel alone.  Prints one JSON line per run and a summary with the card name and power limit, read in the same
process.  Needs a CUDA device.

    python tools/env_params_bench.py [--steps 50] [--warmup 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

SIGMA = float(np.exp(-2.5))          # the action noise of bench.py (learning/simple_mlp.yaml fixed log_std)
CFGS = {"cfg2": dict(env="speed", robot="smpl_humanoid"), "cfg5": dict(env="getup", robot="smplx_humanoid")}


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def draws(env, dev, seed=0):
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    m, N = env.model, env.num_envs
    u = lambda lo, hi, *s: lo + (hi - lo) * torch.rand(*s, generator=g, device=dev)  # noqa: E731
    f32 = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device=dev)  # noqa: E731
    return {"friction": u(0.4, 1.6, N), "gravity": f32(m.gravity)[None] + u(-0.5, 0.5, N, 3),
            "kp": f32(m.act_kp)[None] * u(0.6, 1.4, N, m.nu), "kd": f32(m.act_kd)[None] * u(0.6, 1.4, N, m.nu),
            "torque_limit": f32(m.act_torque_lim)[None] * u(0.6, 1.4, N, m.nu), "body_mass_scale": u(0.7, 1.3, N, m.nbody)}


def run(wl, mode, N, K, W):
    dev = torch.device("cuda:0")
    env = HumanoidBatchB200(make_cfg(**CFGS[wl]), num_envs=N, device="cuda:0", seed=0, with_aux=False)
    nu = env.num_actions
    out = dict(workload=wl, mode=mode, envs=N, steps=K)
    if mode == "nominal":
        env.set_env_params(**env.env_params)
    if mode == "xfrc0":
        env.xfrc_applied = torch.zeros(N, env.model.nbody, 6, dtype=torch.float32, device=dev)
    if mode == "rand":
        P = draws(env, dev)
        env.set_env_params(**P)       # first call: allocates the records
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        env.set_env_params(**P)
        torch.cuda.synchronize()
        out["set_env_params_call_ms"] = (time.perf_counter() - t0) * 1e3
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        from smplsim_b200.abi import SmplsimEnvParamsC
        import ctypes as C
        p = SmplsimEnvParamsC(**{k: v.data_ptr() for k, v in P.items()})
        a.record()
        env._check(env._L().smplsim_set_env_params(env._h, C.byref(p), None, env._stream()))
        b.record()
        torch.cuda.synchronize()
        out["set_env_params_kernel_ms"] = a.elapsed_time(b)
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    env.reset()
    acts = torch.clamp(torch.randn(W + K, N, nu, generator=gen, device=dev) * SIGMA, -1, 1)
    for i in range(W):
        env.step(acts[i]); env.reset_done(); flush.zero_()
    kev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
    for i, (a, b) in enumerate(kev):
        flush.zero_()
        a.record(); env.step(acts[W + i]); b.record()
        env.reset_done()
    torch.cuda.synchronize()
    out["k_step5_ms"] = float(np.mean([a.elapsed_time(b) for a, b in kev]))
    out["status_nonzero"] = int((env.status != 0).sum().item())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("env_params_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    rows = []
    for wl, mode in [("cfg2", "none"), ("cfg2", "xfrc0"), ("cfg2", "nominal"), ("cfg2", "rand")] * 3 + [("cfg5", "none"), ("cfg5", "nominal"), ("cfg5", "rand")]:
        r = run(wl, mode, args.envs, args.steps, args.warmup)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu}
    for wl in CFGS:
        med = {md: float(np.median([r["k_step5_ms"] for r in rows if r["workload"] == wl and r["mode"] == md]))
               for md in ("none", "xfrc0", "nominal", "rand") if any(r["workload"] == wl and r["mode"] == md for r in rows)}
        summ[wl] = dict({f"{md}_ms": round(x, 4) for md, x in med.items()}, nominal_over_none=round(med["nominal"] / med["none"], 4),
                        rand_over_none=round(med["rand"] / med["none"], 4))
    print(json.dumps({"summary": summ}), flush=True)


if __name__ == "__main__":
    main()
