"""Cost of blended motion-library states on the H100: smplsim_motion_blend against the nearest-frame gather, the imitation task with
interpolated and future targets, and blended AMP demonstration rows.  Cases:

  blend_<rows>      k_motion_blend against k_motion_gather over the eight library tables (qpos QPOS, qvel, xpos POS, xquat SLERP,
                    body_vel, body_ang_vel, dof_pos, dof_vel), 4 096 and 65 536 rows of SMPL tables (64 synthetic clips of 300 frames)
  im_<case>         k_imitation for the options (interpolate, T): (0, 1) as before, (1, 1), (1, 3) and (0, 3), on 4 096 / 8 192 SMPL
                    envs and 4 096 SMPL-X envs (obs v2, all bodies tracked), the state an env step left
  amp_demo          AMP_DEMO rows (K = 10 frames each) with and without blending, 65 536 rows

Every timed call follows a 256 MiB L2 flush and a ~1 ms GPU spin (the rules of tools/imitation_bench.py), CUDA events around each
call.  Prints one JSON line per case and the card's name, power limit and maximum SM clock read in the same process.  Needs a CUDA
device.

    python tools/motion_state_bench.py [--reps 30] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from imitation_bench import card, events  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import TABLE_KEYS, synthetic_tables  # noqa: E402

IM_CASES = [("smpl-4096", "smpl_humanoid", 4096), ("smpl-8192", "smpl_humanoid", 8192), ("smplx-4096", "smplx_humanoid", 4096)]
OPTIONS = [(0, 1), (1, 1), (1, 3), (0, 3)]


def stats(ms):
    return dict(ms=float(np.mean(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/motion_state_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("motion_state_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu, dev, R = card(), torch.device("cuda:0"), args.reps
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    rows = []

    def emit(r):
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)

    for name, robot, N in IM_CASES:
        env = HumanoidImB200(make_cfg(env="im", robot=robot, overrides={"env.num_traj_samples": 3}),
                             lambda b: synthetic_tables(b, num_clips=64, frames=300), num_envs=N, device="cuda:0", seed=0)
        env.reset()
        env.step(torch.clamp(torch.randn(N, env.num_actions, generator=gen, device=dev) * 0.3, -1, 1))
        nb, J = env.model.nbody, len(env.tracked_bodies)
        r = dict(case="im_" + name, envs=N)
        for interp, T in OPTIONS:
            env._icfg.interpolate, env._icfg.num_future = interp, T
            events(lambda i: env._task(None, obs_only=False), 3, flush)
            ms = events(lambda i: env._task(None, obs_only=False), R, flush)
            # bytes per env: reference rows (13 floats a body; 2 per time blended, T + 1 times), simulated body state, self obs, obs row
            rows_read = (2 if interp else 1) * (T + 1)
            nbytes = N * ((rows_read + 1) * 13 * nb + env.batch.num_obs + env.batch.num_obs + 24 * J * T) * 4
            r[f"interp{interp}_T{T}"] = dict(stats(ms), GBps=nbytes / (np.mean(ms) * 1e-3) / 1e9)
        emit(r)
        if robot == "smpl_humanoid" and N == 4096:
            lib = env.lib
            for n in (4096, 65536):
                ids = lib.sample_motions(n)
                tm = lib.sample_time(ids)
                outs = [torch.empty(n, lib.tables[k].shape[1], device=dev) for k in TABLE_KEYS]
                width = sum(lib.tables[k].shape[1] for k in TABLE_KEYS)
                g = events(lambda i: lib.gather_into(TABLE_KEYS, ids, tm, outs), R, flush)
                b = events(lambda i: lib.blend_into(TABLE_KEYS, ids, tm, outs), R, flush)
                emit(dict(case=f"blend_{n}", rows=n, floats_per_row=width, gather=dict(stats(g), GBps=n * width * 8 / (np.mean(g) * 1e-3) / 1e9),
                          blend=dict(stats(b), GBps=n * width * 12 / (np.mean(b) * 1e-3) / 1e9)))
            lib.set_amp_cfg()
            n = 65536
            ids = lib.sample_motions(n)
            tm = lib.sample_time(ids, truncate_time=9 * env.dt) + 9 * env.dt
            out = lib.amp_obs_demo(motion_ids=ids, motion_times=tm)
            r = dict(case="amp_demo", rows=n, K=int(out.shape[1]), F=int(out.shape[2]))
            for interp in (0, 1):
                lib._amp_ccfg.interpolate = interp
                r[f"interp{interp}"] = stats(events(lambda i: lib.amp_obs_demo(motion_ids=ids, motion_times=tm, out=out), R, flush))
            emit(r)
        del env
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "motion_state_bench.jsonl"), "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
