"""Time of smplsim_centroidal (HumanoidBatchB200.centroidal) on the H100, against the centroidal momentum matrix and bias composed in
torch from smplsim_dynamics.  Cases:

  smpl-4096-all     SMPL, 4 096 rows on a 4 096-env handle: subtree_com / linvel / angmom, cmm, cmm_bias and jac_com of 5 bodies
  smpl-4096-cmm     the same, cmm and cmm_bias only
  smpl-4096-com     the same, subtree_com only (no qvel)
  smpl-4096-jac5    the same, jac_com only: both hands, both feet (toes) and the head
  smpl-131072-all   SMPL, 131 072 rows on a 4 096-env handle, all outputs: 32 launches of 4 096 rows on the stream
  smplx-4096-all    SMPL-X, 4 096 rows, all outputs (wrists instead of hands)

Baseline (cases with cmm and cmm_bias): dynamics(mass_matrix=True, bias=True), then in torch the root rows of M (armature removed)
and of qfrc_bias, the whole-body first moment m (c - x_root) = -1/2 sum_k c_k x M[0:3, 3 + k], and the shift to the centre of mass
(DESIGN.md 2).  It is checked against the kernel in the same run (max error relative to each row's largest entry).

Inputs are states with floor contact: each handle resets (Default init, speed task, stable PD) and takes 10 env steps; its (qpos, qvel)
rows are then repeated, with seeded noise on the joint angles, up to the row count.  Each case warms up 3 calls, then times 20 calls
with CUDA events, each after a 256 MiB L2 flush (as bench.py), and reports the mean ms per call and rows/s.  Prints one JSON line per
case and a summary line with the card name, power limit and SM clock cap, read in the same process.  Needs a CUDA device.

    python tools/centroidal_bench.py [--reps 20] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

BODIES = {"smpl_humanoid": ["L_Hand", "R_Hand", "L_Toe", "R_Toe", "Head"],
          "smplx_humanoid": ["L_Wrist", "R_Wrist", "L_Toe", "R_Toe", "Head"]}
ALL = ("subtree_com", "subtree_linvel", "subtree_angmom", "cmm", "cmm_bias", "jac_com")
# name, robot, rows, outputs
CASES = [("smpl-4096-all", "smpl_humanoid", 4096, ALL), ("smpl-4096-cmm", "smpl_humanoid", 4096, ("cmm", "cmm_bias")),
         ("smpl-4096-com", "smpl_humanoid", 4096, ("subtree_com",)), ("smpl-4096-jac5", "smpl_humanoid", 4096, ("jac_com",)),
         ("smpl-131072-all", "smpl_humanoid", 131072, ALL), ("smplx-4096-all", "smplx_humanoid", 4096, ALL)]


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
    q[env.num_envs:, 7:] += torch.randn(rows - env.num_envs, env.num_actions, generator=gen, device=dev) * 0.05
    return q, v


def kernel_call(env, q, v, outs, jb):
    """One smplsim_centroidal call writing exactly `outs` (the C ABI: the Python method ties cmm_bias to the velocity outputs)."""
    m, n, f32 = env.model, q.shape[0], dict(dtype=torch.float32, device=q.device)
    shapes = {"subtree_com": (n, m.nbody, 3), "subtree_linvel": (n, m.nbody, 3), "subtree_angmom": (n, m.nbody, 3), "cmm": (n, 6, m.nv),
              "cmm_bias": (n, 6), "jac_com": (n, len(jb), 3, m.nv)}
    o = {k: torch.empty(shapes[k], **f32) for k in outs}
    p = lambda k: C.c_void_p(o[k].data_ptr()) if k in o else None  # noqa: E731
    need_v = any(k in o for k in ("subtree_linvel", "subtree_angmom", "cmm_bias"))
    ids = (C.c_int32 * len(jb))(*jb)
    nj = len(jb) if "jac_com" in o else 0
    env._check(env._L().smplsim_centroidal(env._h, C.c_void_p(q.data_ptr()), C.c_void_p(v.data_ptr()) if need_v else None, n, p("subtree_com"),
                                           p("subtree_linvel"), p("subtree_angmom"), p("cmm"), p("cmm_bias"), ids if nj else None, nj,
                                           p("jac_com"), env._stream()))
    return o


def baseline(env, q, v):
    """cmm [n, 6, nv] and cmm_bias [n, 6] composed in torch from dynamics(mass_matrix=True, bias=True)."""
    m = env.model
    d = env.dynamics(q, v, mass_matrix=True, bias=True)
    M6, b = d["qM"][:, :6].clone(), d["qfrc_bias"]
    arm = torch.as_tensor(np.asarray(m.dof_armature[:6], dtype=np.float32), device=q.device)
    M6[:, torch.arange(6), torch.arange(6)] -= arm
    w, x, y, z = (q[:, 3 + k] for k in range(4))
    s = 2.0 / (w * w + x * x + y * y + z * z)
    R = torch.stack([1 - s * (y * y + z * z), s * (x * y - w * z), s * (x * z + w * y),
                     s * (x * y + w * z), 1 - s * (x * x + z * z), s * (y * z - w * x),
                     s * (x * z - w * y), s * (y * z + w * x), 1 - s * (x * x + y * y)], 1).view(-1, 3, 3)
    mass = M6[:, 0, 0]
    md = -0.5 * sum(torch.linalg.cross(R[:, :, k], M6[:, 0:3, 3 + k]) for k in range(3))   # m (c - x_root)
    dlt = md / mass[:, None]
    p, LO = M6[:, 0:3], R @ M6[:, 3:6]
    A = torch.cat([p, LO - torch.linalg.cross(dlt[:, :, None].expand_as(p), p, dim=1)], 1)
    g = torch.as_tensor(np.asarray(m.gravity, dtype=np.float32), device=q.device).expand(q.shape[0], 3)
    F = b[:, 0:3] + mass[:, None] * g
    T = (R @ b[:, 3:6, None])[:, :, 0] + torch.linalg.cross(md, g)
    return A, torch.cat([F, T - torch.linalg.cross(dlt, F)], 1)


def timed(fn, reps, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for e0, e1 in ev:
        flush.zero_()
        e0.record(); out = fn(); e1.record()
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in ev], out


def run(name, robot, rows, outs, reps, gen, flush):
    env = HumanoidBatchB200(make_cfg(env="speed", robot=robot), num_envs=4096, device="cuda:0", seed=0)
    q, v = inputs(env, rows, gen)
    jb = [list(env.model.body_names).index(b) for b in BODIES[robot]]
    ms, out = timed(lambda: kernel_call(env, q, v, outs, jb), reps, flush)
    r = dict(case=name, rows=rows, launches=(rows + 4095) // 4096, outputs=list(outs), ms_mean=float(np.mean(ms)), ms_min=float(np.min(ms)),
             ms_max=float(np.max(ms)), rows_per_s=rows / (float(np.mean(ms)) / 1e3),
             finite=all(bool(torch.isfinite(x).all().item()) for x in out.values()))
    if "cmm" in outs and "cmm_bias" in outs:
        bms, (A, bias) = timed(lambda: baseline(env, q, v), reps, flush)
        rel = lambda a, b: float(((a - b).abs().flatten(1).amax(1) / b.abs().flatten(1).amax(1).clamp_min(1.0)).max())  # noqa: E731
        r.update(baseline_ms_mean=float(np.mean(bms)), speedup=float(np.mean(bms)) / r["ms_mean"],
                 baseline_err_cmm=rel(A, out["cmm"]), baseline_err_bias=rel(bias, out["cmm_bias"]))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/centroidal_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("centroidal_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)      # > 50 MB L2
    rows = []
    for name, robot, n, outs in CASES:
        r = run(name, robot, n, outs, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
    summ = {"gpu": gpu, **{r["case"]: dict(ms=round(r["ms_mean"], 4), **({"baseline_ms": round(r["baseline_ms_mean"], 4),
                                                                           "speedup": round(r["speedup"], 2)} if "speedup" in r else {}))
                           for r in rows}}
    print(json.dumps({"summary": summ}), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "centroidal_bench.jsonl"), "w") as f:
            for r in rows + [{"summary": summ}]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
