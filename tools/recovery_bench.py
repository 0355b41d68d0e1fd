"""Cost of fail-state recovery in the imitation task on the H100: 4 096 SMPL envs, obs v2, all bodies tracked, 64 synthetic clips of 300
frames.
  k_imitation_ms / k_imitation_rec_ms   the task kernel alone (full mode) in its base instance (make_cfg(env="im")) and in its recovery
                   instance (make_cfg(env="im_recovery"): zero-out-far, point goal, recovery window, power), same env, same state;
                   CUDA events around each call, each after a 256 MiB L2 flush and a ~1 ms GPU spin (as tools/imitation_bench.py)
  im_steps_per_s / im_recovery_steps_per_s   HumanoidImB200.step + reset_done for the two cfgs, alternated in one process over
                   --rounds rounds of --steps steps (N(0, 0.3) actions, so envs fall, terminate and are reset), median of the rounds
  bank_build_ms    the one-off fall-state bank of the im_recovery constructor (8 Fall resets over all envs and the copies)
  resets           per kind (mocap / fall / recovery) over the im_recovery rounds
Prints one JSON line with the card's name, power limit and maximum SM clock read in the same process.  Needs a CUDA device.
    python tools/recovery_bench.py [--steps 60] [--warmup 10] [--rounds 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from imitation_bench import card, events  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402

N = 4096


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("recovery_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu, dev = card(), torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    envs = {}
    bank_ms = 0.0
    for name in ("im", "im_recovery"):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        envs[name] = HumanoidImB200(make_cfg(env=name), lambda b: synthetic_tables(b, num_clips=64, frames=300), num_envs=N,
                                    device="cuda:0", seed=0)
        torch.cuda.synchronize()
        if name == "im_recovery":   # time the bank build on its own, on the env just built
            env = envs[name]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for r in range(env.fall_qpos.shape[0]):
                env.batch.reset(None, init_mode=1)
                env.fall_qpos[r].copy_(env.batch.qpos)
                env.fall_qvel[r].copy_(env.batch.qvel)
            torch.cuda.synchronize()
            bank_ms = (time.perf_counter() - t0) * 1e3
        envs[name].reset()
    nu = envs["im"].num_actions
    K, W = args.steps, args.warmup

    def run(env, steps):
        acts = torch.clamp(torch.randn(steps, N, nu, generator=gen, device=dev) * 0.3, -1, 1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(steps):
            env.step(acts[i])
            env.reset_done()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for env in envs.values():
        run(env, W)
    rate = {k: [] for k in envs}
    rec = envs["im_recovery"]
    c0 = rec.reset_counts.clone()
    for _ in range(args.rounds):
        for k, env in envs.items():
            rate[k].append(N * K / run(env, K))
    counts = (rec.reset_counts - c0).tolist()
    # the kernels alone, base and recovery instance, on the state the im_recovery loop left
    base = events(lambda i: rec._task(None, obs_only=False, recovery=False), 30, flush)
    saved = rec.recovery.clone()
    krec = events(lambda i: rec._task(None, obs_only=False), 30, flush)
    rec.recovery.copy_(saved)
    r = dict(envs=N, steps=K, rounds=args.rounds, k_imitation_ms=float(np.mean(base)), k_imitation_rec_ms=float(np.mean(krec)),
             k_imitation_ms_min=float(np.min(base)), k_imitation_rec_ms_min=float(np.min(krec)),
             im_steps_per_s=float(np.median(rate["im"])), im_recovery_steps_per_s=float(np.median(rate["im_recovery"])),
             im_rounds=[round(x) for x in rate["im"]], im_recovery_rounds=[round(x) for x in rate["im_recovery"]],
             bank_build_ms=bank_ms, resets=dict(mocap=counts[1], fall=counts[2], recovery=counts[3]), gpu=gpu)
    print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
