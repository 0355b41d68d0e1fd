"""Cost of the motion-imitation task (smplsim_imitation, HumanoidImB200) on the H100.  Cases: 4 096 and 8 192 SMPL envs, 4 096 SMPL-X
envs (obs v2, all bodies tracked, 64 synthetic clips of 300 frames).  Per case:

  k_imitation_ms   the task kernel alone (full mode), CUDA events around each call
  k_step5_ms       the step kernel of the same env, for scale
  im_steps_per_s   a full imitation env step: HumanoidImB200.step (step kernel + task kernel + per-clip counters) and reset_done (clip
                   draw, two-table gather, masked MoCap reset, observation-only task call), env-steps per second over the timed loop
  cfg4_steps_per_s the same loop written as bench.py's cfg4 does it: get_motion_state_intervaled (nine-table gather) + speed-task step +
                   masked MoCap reset; it computes no tracking observation or reward

Every timed call follows a 256 MiB L2 flush (as bench.py); the per-kernel timings also follow a ~1 ms GPU spin that keeps the host's
enqueue out of the event window; the loops are timed end to end with the flushes inside and the flush time alone is reported beside
them.  Actions are N(0, 0.3) clipped, so envs fall, terminate and are reset during the loop, as in training.  Prints one JSON line per
case and a summary with the card's name, power limit and maximum SM clock read in the same process.  Needs a CUDA device.

    python tools/imitation_bench.py [--steps 60] [--warmup 10] [--out DIR]
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
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables  # noqa: E402

HEADROOM = 2_000_000     # GPU spin (cycles, ~1 ms) queued before a timed kernel
CASES = [("smpl-4096", "smpl_humanoid", 4096), ("smpl-8192", "smpl_humanoid", 8192), ("smplx-4096", "smplx_humanoid", 4096)]
V2 = {"env.self_obs_v": 2, "robot.create_vel_sensors": True}


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def events(fn, reps, flush):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i, (e0, e1) in enumerate(ev):
        flush.zero_()
        torch.cuda._sleep(HEADROOM)
        e0.record(); fn(i); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def loop_ms(one_step, acts, warmup, flush):
    for i in range(warmup):
        one_step(acts[i]); flush.zero_()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(warmup, acts.shape[0]):
        one_step(acts[i]); flush.zero_()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/imitation_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("imitation_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu, dev = card(), torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    flush.zero_(); torch.cuda.synchronize()
    f0.record()
    for _ in range(10):
        flush.zero_()
    f1.record(); torch.cuda.synchronize()
    flush_ms = f0.elapsed_time(f1) / 10
    K, W = args.steps, args.warmup
    rows = []
    for name, robot, N in CASES:
        tabs = None

        def tables(b):
            nonlocal tabs
            tabs = synthetic_tables(b, num_clips=64, frames=300)
            return tabs

        env = HumanoidImB200(make_cfg(env="im", robot=robot), tables, num_envs=N, device="cuda:0", seed=0)
        nu = env.num_actions
        acts = torch.clamp(torch.randn(W + K, N, nu, generator=gen, device=dev) * 0.3, -1, 1)
        env.reset()

        def im_step(a):
            env.step(a); env.reset_done()

        im_ms = loop_ms(im_step, acts, W, flush)
        resets = float(env.clip_episodes.sum().item())
        # the kernels alone, on the state the loop left
        kim = events(lambda i: env._task(None, obs_only=False), 30, flush)
        kstep = []
        for i in range(30):
            kstep += events(lambda _: env.batch.step(acts[i]), 1, flush)
            env._task(None, obs_only=False); torch.bitwise_or(env.terminate_buf, env.truncate_buf, out=env.reset_buf); env.reset_done()
        # bytes the task kernel needs per env: two reference rows and the simulated body state (13 floats a body each), the self
        # observation read, the observation row written
        kernel_bytes = (3 * 13 * env.model.nbody + env.batch.num_obs + env.num_obs) * 4
        del env
        # the cfg4 loop of bench.py: nine-table gather, speed-task step, masked MoCap reset
        b4 = HumanoidBatchB200(make_cfg(env="speed", robot=robot, overrides=V2), num_envs=N, device="cuda:0", seed=0, with_aux=False)
        lib = MotionLibB200(b4, tabs)
        ids = (torch.arange(N, device=dev) % 64).to(torch.int32)
        t_env = torch.rand(N, generator=gen, device=dev) * 8.0
        dt = float(b4.dt)

        def cfg4_step(a):
            st = lib.get_motion_state_intervaled(ids, t_env)
            b4.step(a)
            b4.reset(b4.reset_buf, init_mode=2, qpos0=st["qpos"], qvel0=st["qvel"])
            t_env.add_(dt)
            t_env.masked_fill_(t_env > 9.0, 0.0)

        st0 = lib.get_motion_state_intervaled(ids, t_env)
        b4.reset(None, init_mode=2, qpos0=st0["qpos"], qvel0=st0["qvel"])
        c4_ms = loop_ms(cfg4_step, acts, W, flush)
        del b4, lib
        r = dict(case=name, robot=robot, envs=N, steps=K, k_imitation_ms=float(np.mean(kim)), k_imitation_ms_min=float(np.min(kim)),
                 k_imitation_ms_max=float(np.max(kim)), k_step5_ms=float(np.mean(kstep)), task_over_step=float(np.mean(kim) / np.mean(kstep)),
                 k_imitation_GBps=N * kernel_bytes / (np.mean(kim) * 1e-3) / 1e9,
                 im_steps_per_s=N * K / (im_ms * 1e-3), im_ms_per_step=im_ms / K, cfg4_steps_per_s=N * K / (c4_ms * 1e-3), cfg4_ms_per_step=c4_ms / K,
                 flush_ms=flush_ms, episodes_ended_per_step=resets / (W + K), gpu=gpu)
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, "flush_ms": round(flush_ms, 4),
            **{r["case"]: dict(k_imitation_ms=round(r["k_imitation_ms"], 4), k_step5_ms=round(r["k_step5_ms"], 4),
                               task_over_step=round(r["task_over_step"], 4), im_ksteps_per_s=round(r["im_steps_per_s"] / 1e3, 1),
                               cfg4_ksteps_per_s=round(r["cfg4_steps_per_s"] / 1e3, 1)) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "imitation_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
