"""Cost of the AMP observation kernel (smplsim_amp_obs / smplsim_amp_demo) and of the AMP pieces around it on the H100.  K = 10 frames,
the reference's key bodies, root height and local root observation (F = 232 for SMPL, 484 for SMPL-X).  Cases:

  push       PUSH per call (shift 9 frames, write the new one; medians of 30 calls) on 4 096 and 8 192 SMPL envs and 4 096 SMPL-X envs, CUDA events around
             each call, with the step kernel of the same env (k_step5, obs v2) for scale
  demo       DEMO for 4 096 and 65 536 rows (SMPL, 64 synthetic clips of 300 frames)
  reward     the discriminator reward forward ([1024, 512] relu) on 4 096 SMPL rows
  update     one AMPLearner.update on 16 steps x 4 096 envs of agent rows (16 minibatches of 4 096: demo rows generated per minibatch)
  env_step   a full HumanoidAmpB200(HumanoidImB200) step with the discriminator reward, and reset_done, 4 096 SMPL envs; beside it the
             HumanoidImB200 loop alone

Every timed call follows a 256 MiB L2 flush; the per-kernel timings also follow a ~1 ms GPU spin that keeps the host's enqueue out of
the event window.  Prints one JSON line per case and a summary with the card's name, power limit and maximum SM clock read in the same
process.  Needs a CUDA device.

    python tools/amp_bench.py [--steps 40] [--warmup 10] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from imitation_bench import card, events, loop_ms  # noqa: E402
from smplsim_b200.abi import AMP_PUSH  # noqa: E402
from smplsim_b200.amp import HumanoidAmpB200  # noqa: E402
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402

PUSH_CASES = [("smpl-4096", "smpl_humanoid", 4096), ("smpl-8192", "smpl_humanoid", 8192), ("smplx-4096", "smplx_humanoid", 4096)]
V2 = {"env.self_obs_v": 2, "robot.create_vel_sensors": True}


def stats(x):
    return dict(ms=float(np.mean(x)), ms_median=float(np.median(x)), ms_min=float(np.min(x)), ms_max=float(np.max(x)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/amp_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("amp_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu, dev = card(), torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    torch.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    rows = []

    def emit(r):
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    for name, robot, N in PUSH_CASES:
        b = HumanoidBatchB200(make_cfg(env="speed", robot=robot, overrides=V2), num_envs=N, device="cuda:0", seed=0)
        amp = HumanoidAmpB200(b)
        b.reset(); amp.reset()
        acts = torch.clamp(torch.randn(30, N, b.num_actions, generator=gen, device=dev) * 0.3, -1, 1)
        kstep, kpush = [], []
        for i in range(30):
            kstep += events(lambda _: b.step(acts[i]), 1, flush)
            kpush += events(lambda _: amp._amp(None, AMP_PUSH), 1, flush)
            b.reset_done()
        F = amp.amp_frame_dim
        # bytes per env: 9 frames read and written, 1 written; qpos, qvel, the root and key-body positions and the root quaternion read
        moved = N * (19 * F + b.model.nq + b.model.nv + 3 * (1 + amp._keys.size) + 4) * 4
        emit(dict(case=f"push-{name}", envs=N, frame_dim=F, k_amp_push=stats(kpush), k_step5=stats(kstep),
                  push_over_step=float(np.median(kpush) / np.median(kstep)), push_GBps=moved / (np.median(kpush) * 1e-3) / 1e9,
                  bytes_per_env=moved / N))
        del amp, b
    # DEMO rows and the discriminator / learner on SMPL
    env = HumanoidImB200(make_cfg(env="im"), lambda bb: synthetic_tables(bb, num_clips=64, frames=300), num_envs=4096, device="cuda:0", seed=0)
    amp = HumanoidAmpB200(env)
    lib = env.lib
    for n in (4096, 65536):
        ids = lib.sample_motions(n)
        span = 9 * env.dt
        tm = lib.sample_time(ids, truncate_time=span) + span
        out = torch.empty(n, 10, amp.amp_frame_dim, device=dev)
        kd = events(lambda _: lib.amp_obs_demo(motion_ids=ids, motion_times=tm, out=out), 30, flush)
        emit(dict(case=f"demo-{n}", rows=n, k_amp_demo=stats(kd), demo_GBps=n * 10 * amp.amp_frame_dim * 4 / (np.mean(kd) * 1e-3) / 1e9))
    learner = amp.make_learner(generator=gen)
    x = torch.randn(4096, amp.num_amp_obs, device=dev)
    learner.update(torch.randn(4, 4096, amp.num_amp_obs, device=dev))      # warm up (and fill the input moments)
    kr = events(lambda _: amp.discriminator.reward(x, 2.0), 30, flush)
    emit(dict(case="disc-reward-4096", rows=4096, ms=stats(kr)))
    agent = torch.randn(16, 4096, amp.num_amp_obs, device=dev)
    ku = []
    for _ in range(5):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); learner.update(agent); e1.record()
        torch.cuda.synchronize()
        ku.append(e0.elapsed_time(e1))
    emit(dict(case="amp-update-16x4096", rows=16 * 4096, minibatches=16, ms=stats(ku)))
    # full env steps: AMP wrapper with the discriminator reward vs the imitation env alone
    K, W, N = args.steps, args.warmup, env.num_envs
    acts = torch.clamp(torch.randn(W + K, N, env.num_actions, generator=gen, device=dev) * 0.3, -1, 1)
    amp.reset()

    def amp_step(a):
        amp.step(a); amp.reset_done()
        if len(amp._rows) > 16:
            amp.drain_amp_obs()

    am = loop_ms(amp_step, acts, W, flush)
    env.reset()

    def im_step(a):
        env.step(a); env.reset_done()

    im = loop_ms(im_step, acts, W, flush)
    emit(dict(case="env-step-smpl-4096", envs=N, steps=K, amp_steps_per_s=N * K / (am * 1e-3), amp_ms_per_step=am / K,
              im_steps_per_s=N * K / (im * 1e-3), im_ms_per_step=im / K))
    print(json.dumps({"summary": {r["case"]: {k: v for k, v in r.items() if k != "gpu"} for r in rows}, "gpu": gpu}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "amp_bench.jsonl"), "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
