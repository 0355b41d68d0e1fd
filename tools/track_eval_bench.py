"""Cost of tracking evaluation (smplsim_track_eval, HumanoidImB200.evaluate) on the H100.  Cases: 4 096 SMPL and 4 096 SMPL-X envs
(obs v2, all bodies evaluated, 64 synthetic clips of 300 frames).  Per case:

  k_track_eval_ms  the evaluation kernel alone, every env active, CUDA events around each call
  k_imitation_ms   the task kernel of the same env (full mode), for scale
  k_step5_ms       the step kernel, for scale

Then a whole evaluation: ``evaluate`` of a random linear policy on a synthetic library of 9 000 clips of 60 frames (64 synthetic clips
repeated; three waves of 4 096 SMPL envs), termination distance 100 m so every clip runs to its end; scored clip-frames per second over the call (host clock
around it, ended by a device synchronise).

Every per-kernel timing follows a 256 MiB L2 flush and a ~1 ms GPU spin that keeps the host's enqueue out of the event window, as
tools/imitation_bench.py.  Prints one JSON line per case and a summary with the card's name, power limit and maximum SM clock read in
the same process.  Needs a CUDA device.

    python tools/track_eval_bench.py [--reps 30] [--eval-clips 9000] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.abi import SmplsimTrackEvalCfgC, SmplsimTrackEvalStateC  # noqa: E402
from smplsim_b200.batched import _ptr  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402
from imitation_bench import HEADROOM, card  # noqa: E402

CASES = [("smpl-4096", "smpl_humanoid", 4096), ("smplx-4096", "smplx_humanoid", 4096)]


def tiled(tabs, K):
    """The synthetic library ``tabs`` repeated to K clips (frame tables tiled, clip rows and keys extended)."""
    k0 = len(tabs["motion_num_frames"])
    reps = (K + k0 - 1) // k0
    F = int(tabs["motion_num_frames"][0])
    out = {k: np.tile(v, (reps, 1))[:K * F] for k, v in tabs.items() if v.ndim == 2 and v.shape[0] == k0 * F}
    for k in ("motion_num_frames", "motion_dt", "motion_lengths", "motion_fps"):
        out[k] = np.tile(tabs[k], reps)[:K]
    out["length_starts"] = (np.arange(K) * F).astype(np.int32)
    out["motion_bodies"] = np.zeros((K, 17), np.float32)
    out["motion_keys"] = np.array([f"synthetic_{k:05d}" for k in range(K)])
    return out


def events(fn, reps, flush):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i, (e0, e1) in enumerate(ev):
        flush.zero_()
        torch.cuda._sleep(HEADROOM)
        e0.record(); fn(i); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--eval-clips", type=int, default=9000)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/track_eval_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("track_eval_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu, dev = card(), torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    rows = []
    for name, robot, N in CASES:
        env = HumanoidImB200(make_cfg(env="im", robot=robot), lambda b: synthetic_tables(b, num_clips=64, frames=300), num_envs=N,
                             device="cuda:0", seed=0)
        b, nb = env.batch, env.model.nbody
        env.reset()
        acts = torch.clamp(torch.randn(args.reps, N, env.num_actions, generator=gen, device=dev) * 0.3, -1, 1)
        env.step(acts[0])
        active = torch.ones(N, dtype=torch.uint8, device=dev)
        frames = torch.zeros(N, dtype=torch.int32, device=dev)
        success = torch.zeros(N, dtype=torch.uint8, device=dev)
        sums = torch.zeros(N, 6, dtype=torch.float64, device=dev)
        prev = torch.zeros(N, 2, nb, 3, device=dev)
        fm = torch.zeros(N, 6, device=dev)
        zero = torch.zeros(N, dtype=torch.uint8, device=dev)
        tcfg = SmplsimTrackEvalCfgC(num_bodies=nb, bodies=None, interpolate=0, dt=0.0)
        st = SmplsimTrackEvalStateC(active=_ptr(active), prev_diff=_ptr(prev), frames=_ptr(frames), sums=_ptr(sums), success=_ptr(success),
                                    frame_metrics=_ptr(fm))
        L = b._L()

        def track(_):
            b._check(L.smplsim_track_eval(b._h, C.byref(tcfg), C.byref(env._tab), _ptr(env.motion_ids), _ptr(env.motion_start_times),
                                          _ptr(b.progress_buf), C.byref(b._aux), _ptr(zero), _ptr(zero), C.byref(st), b._stream()))

        track(0)
        kte = events(track, args.reps, flush)
        kim = events(lambda i: env._task(None, obs_only=False), args.reps, flush)
        kstep = []
        for i in range(args.reps):
            kstep += events(lambda _: b.step(acts[i]), 1, flush)
            env._task(None, obs_only=False); torch.bitwise_or(env.terminate_buf, env.truncate_buf, out=env.reset_buf); env.reset_done()
        assert bool(active.all()) and torch.isfinite(fm).all()
        r = dict(case=name, robot=robot, envs=N, k_track_eval_ms=float(np.mean(kte)), k_track_eval_ms_min=float(np.min(kte)),
                 k_imitation_ms=float(np.mean(kim)), k_step5_ms=float(np.mean(kstep)), eval_over_step=float(np.mean(kte) / np.mean(kstep)), gpu=gpu)
        rows.append(r)
        print(json.dumps(r), flush=True)
        del env
    # a whole evaluation over more clips than envs
    N, K = 4096, args.eval_clips
    env = HumanoidImB200(make_cfg(env="im"), lambda b: tiled(synthetic_tables(b, num_clips=64, frames=60), K), num_envs=N, device="cuda:0", seed=0)
    print(f"library: {env.lib.num_motions()} clips", flush=True)
    W = torch.randn(env.num_obs, env.num_actions, generator=gen, device=dev) * 0.002
    pol = lambda obs: torch.tanh(obs @ W)  # noqa: E731
    env.evaluate(pol, motion_ids=list(range(min(N, K))), termination_distance=100.0)     # warm-up: one wave
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = env.evaluate(pol, termination_distance=100.0)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    steps = int(sum(env.clip_steps(list(range(w, min(w + N, K)))).max() for w in range(0, K, N)))
    ev = dict(case="evaluate-smpl-4096", clips=K, waves=(K + N - 1) // N, env_steps=steps, frames_scored=int(res.frames.sum()), seconds=sec,
              clip_frames_per_s=float(res.frames.sum()) / sec, env_steps_per_s=steps * N / sec, success_rate=res.summary()["success_rate"], gpu=gpu)
    rows.append(ev)
    print(json.dumps(ev), flush=True)
    summ = {"gpu": gpu, **{r["case"]: {k: round(v, 4) if isinstance(v, float) else v for k, v in r.items() if k not in ("case", "gpu", "robot")}
                           for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "track_eval_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
