"""Time of smplsim_render / smplsim_ray (HumanoidBatchB200.render / ray) on the H100.  Cases:

  depth64-side       SMPL, 4 096 envs, 64 x 64 depth from the "side" tracking camera (a vision observation)
  depth64-ego        the same from the egocentric head camera
  depth128-side      SMPL, 4 096 envs, 128 x 128 depth from "side" (the primary rays of the next case, without the shading)
  rgb128-side        SMPL, 4 096 envs, 128 x 128 RGB from "side"
  rgb320x240-1env    SMPL, 1 env, 320 x 240 RGB from "side" (the frame of the single-env render())
  ray256-4096        SMPL, 4 096 envs, 256 rays each: a 16 x 16 height scan, 4 cm grid around the root, straight down from 3 m
  smplx-depth64-side SMPL-X, 4 096 envs, 64 x 64 depth from "side"

Poses are those of a 4 096-env handle after a reset (Default init, speed task, stable PD) and 10 env steps with random actions.
Each case warms up 3 calls, then times 20 calls with CUDA events, each after a 256 MiB L2 flush (as bench.py) and a ~1 ms GPU spin that
keeps the host's enqueue out of the window, and reports the mean ms per call and primary rays per second.  For scale, the same run times cfg2's k_step5 (the env step of bench.py's workload) over 20
steps.  Prints one JSON line per case and a summary with the card's name and power limit, read in the same process.  Needs a CUDA
device.  --dump DIR also writes a few frames as PNG files; --profile DIR records the rgb128-side case with torch.profiler (CUDA
activities, a run of its own after the timed cases) and writes its kernel table to DIR/render_profile.txt.

    python tools/render_bench.py [--reps 20] [--out DIR] [--dump DIR] [--profile DIR]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

N = 4096
# GPU spin (cycles, ~1 ms) queued before each timed call: the host enqueues the call while the GPU is busy, so the events time the
# kernels and not the Python between them
HEADROOM = 2_000_000
# name, robot, envs, camera (None: rays), width, height, outputs
CASES = [("depth64-side", "smpl_humanoid", N, "side", 64, 64, "depth"), ("depth64-ego", "smpl_humanoid", N, "egocentric", 64, 64, "depth"),
         ("depth128-side", "smpl_humanoid", N, "side", 128, 128, "depth"), ("rgb128-side", "smpl_humanoid", N, "side", 128, 128, "rgb"), ("rgb320x240-1env", "smpl_humanoid", 1, "side", 320, 240, "rgb"),
         ("ray256-4096", "smpl_humanoid", N, None, 256, 1, "ray"), ("smplx-depth64-side", "smplx_humanoid", N, "side", 64, 64, "depth")]


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "nvidia-smi unavailable"


def write_png(path, img):
    """uint8 [H, W, 3] (or [H, W] grey) as an 8-bit PNG."""
    img = np.ascontiguousarray(img if img.ndim == 3 else np.repeat(img[..., None], 3, 2), dtype=np.uint8)
    h, w, _ = img.shape
    raw = b"".join(b"\x00" + img[r].tobytes() for r in range(h))

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6))
                + chunk(b"IEND", b""))


def settle(env, gen):
    env.reset()
    for _ in range(10):
        env.step(torch.clamp(torch.randn(env.num_envs, env.num_actions, generator=gen, device=env.device) * 0.3, -1, 1))
        env.reset_done()


def height_scan(env):
    """[N, 256, 3] origins 3 m above a 16 x 16 grid (4 cm) centred on each root, and their down vectors."""
    g = (torch.arange(16, device=env.device, dtype=torch.float32) - 7.5) * 0.04
    gx, gy = torch.meshgrid(g, g, indexing="ij")
    off = torch.stack([gx.reshape(-1), gy.reshape(-1), torch.full((256,), 3.0, device=env.device)], 1)
    root = env.xpos[:, 0].clone()
    root[:, 2] = 0.0
    pnt = (root[:, None, :] + off[None]).contiguous()
    vec = torch.zeros_like(pnt)
    vec[..., 2] = -1.0
    return pnt, vec


def timed(fn, reps, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        torch.cuda._sleep(HEADROOM)
        e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def cfg2_step_ms(reps, gen, flush):
    """k_step5 of bench.py's cfg2 workload (4 096 SMPL envs, speed task, stable PD, no side outputs): events around each step,
    a flush before it, the autoreset after it."""
    env = HumanoidBatchB200(make_cfg(env="speed"), num_envs=N, device="cuda:0", seed=0, with_aux=False)
    settle(env, gen)
    acts = torch.clamp(torch.randn(reps, N, env.num_actions, generator=gen, device=env.device) * 0.3, -1, 1)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for i, (e0, e1) in enumerate(ev):
        flush.zero_()
        torch.cuda._sleep(HEADROOM)
        e0.record(); env.step(acts[i]); e1.record()
        env.reset_done()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/render_bench.jsonl")
    ap.add_argument("--dump", default=None, help="write a few frames as PNG files to DIR")
    ap.add_argument("--profile", default=None, help="torch.profiler kernel table of the rgb128-side case to DIR/render_profile.txt")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("render_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    envs = {}
    for robot in ("smpl_humanoid", "smplx_humanoid"):
        envs[robot] = HumanoidBatchB200(make_cfg(env="speed", robot=robot), num_envs=N, device="cuda:0", seed=0)
        settle(envs[robot], gen)
    e2 = envs["smpl_humanoid"]
    step_ms = cfg2_step_ms(args.reps, gen, flush)
    rows = []
    for name, robot, n, camera, w, h, what in CASES:
        env = envs[robot]
        xp, xq = env.xpos[:n].contiguous(), env.xquat[:n].contiguous()
        if what == "ray":
            pnt, vec = height_scan(env)
            fn = lambda: env.ray(pnt, vec, xpos=xp, xquat=xq)          # noqa: E731
            nrays = n * pnt.shape[1]
        else:
            kw = dict(depth=what == "depth", rgb=what == "rgb")
            fn = lambda: env.render(camera, w, h, xpos=xp, xquat=xq, **kw)   # noqa: E731
            nrays = n * w * h
        ms = timed(fn, args.reps, flush)
        t = float(np.mean(ms)) / 1e3
        out = fn()
        finite = all(bool(torch.isfinite(v.float()).all().item()) for v in out.values())
        r = dict(case=name, robot=robot, envs=n, size=[w, h], ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)), ms_max=float(np.max(ms)),
                 rays_per_s=nrays / t, over_cfg2_step=float(np.mean(ms)) / float(np.mean(step_ms)), finite=finite, gpu=gpu)
        rows.append(r)
        print(json.dumps(r), flush=True)
        if args.dump and what != "ray":
            os.makedirs(args.dump, exist_ok=True)
            for i in range(min(n, 2)):
                if what == "rgb":
                    img = out["rgb"][i].cpu().numpy()
                else:
                    d = out["depth"][i].cpu().numpy()
                    img = np.uint8(255 * np.clip(1 - d / 8.0, 0, 1))        # near = bright, 8 m and beyond black
                write_png(os.path.join(args.dump, f"{name}_{i}.png"), img)
    if args.dump:
        for cam_name in ("back", "side", "front_side", "egocentric"):
            write_png(os.path.join(args.dump, f"rgb320x240_{cam_name}.png"), e2.render(cam_name, 320, 240, xpos=e2.xpos[:1].contiguous(),
                                                                                         xquat=e2.xquat[:1].contiguous())["rgb"][0].cpu().numpy())
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        xp, xq = e2.xpos.contiguous(), e2.xquat.contiguous()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                e2.render("side", 128, 128, xpos=xp, xquat=xq)
            torch.cuda.synchronize()
        os.makedirs(args.profile, exist_ok=True)
        with open(os.path.join(args.profile, "render_profile.txt"), "w") as f:
            f.write(gpu + "\n" + prof.key_averages().table(sort_by="cuda_time_total", row_limit=10) + "\n")
    summ = {"gpu": gpu, "cfg2_k_step5_ms": round(float(np.mean(step_ms)), 4),
            **{r["case"]: dict(ms=round(r["ms_mean"], 4), Grays_per_s=round(r["rays_per_s"] / 1e9, 3)) for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "render_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
