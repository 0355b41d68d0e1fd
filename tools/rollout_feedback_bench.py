"""Cost of closed-loop rollouts (HumanoidBatchB200.rollout(gains=...), smplsim_rollout_feedback) on the H100.  Cases:

  batch1k-smpl     1 024 rows x 30 action steps, SMPL
  batch4k-smpl     4 096 rows x 30 action steps, SMPL
  mjroll-smpl      256 rows x 450 ctrl steps with nsub = 1 (one mj_step per control row), SMPL
  batch1k-smplx    1 024 rows x 30 action steps, SMPL-X

Each case times, on the same rows, the open-loop rollout, the feedback rollout with shared gains (ref_rows = 1) and with per-row
gains (ref_rows = n), and the host loop a user could run instead: one step / mj_step launch per control row with the feedback
computed in torch in between (shared gains).  Gains are seeded noise; every row starts from one state and the reference is that
state's open-loop trajectory, so dx = 0 and the closed-loop rows run the open-loop trajectory bit for bit (checked): the times differ by
the feedback's own cost only.  It also reports how far the host loop's first controls are from the kernel's.  CUDA events, warm-up, each call after a 256 MiB L2 flush, as
tools/rollout_bench.py.

Then a stabilisation figure: TVLQR gains from transition_fd and a Riccati pass (fp64) around an open-loop nominal of 30 ctrl steps
(nsub = 1) from a reset SMPL state, and 256 starts perturbed from the nominal start; the tangent deviation from the nominal after 30
steps, open-loop (the nominal's controls) against closed-loop.

Prints one JSON line per case and a summary with the card name and power limit, read in the same process.  Needs a CUDA device.

    python tools/rollout_feedback_bench.py [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rollout_bench import card, inputs, timed  # noqa: E402

from smplsim_b200.batched import HumanoidBatchB200  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402

CASES = [("batch1k-smpl", "smpl_humanoid", "action", 1024, 30), ("batch4k-smpl", "smpl_humanoid", "action", 4096, 30),
         ("mjroll-smpl", "smpl_humanoid", "ctrl", 256, 450), ("batch1k-smplx", "smplx_humanoid", "action", 1024, 30)]


def host_loop(env, q, v, w, u, mode, K, qr, vr, clip):
    env.set_state(q, v)
    env.qacc_warm.copy_(w)
    first = None
    for t in range(u.shape[1]):
        dx = torch.cat([env.differentiate_pos(qr[0, t], env.qpos), env.qvel - vr[0, t]], -1)
        ut = u[:, t] + dx @ K[0, t].T
        if clip:
            ut = torch.clamp(ut, -1.0, 1.0)
        if first is None:
            first = ut.clone()
        if mode == "action":
            env.step(ut)
        else:
            env.mj_step(ut, 1)
    return first


def run(name, robot, mode, rows, T, reps, gen, flush):
    cfg, q, v, w, u = inputs(robot, mode, rows, rows, T, gen)
    env = HumanoidBatchB200(cfg, num_envs=rows, device="cuda:0", seed=0)
    m = env.model
    nx = 2 * m.nv
    kw = dict(mode=mode, nsub=1 if mode == "ctrl" else None, qacc_warmstart=w)
    # the reference is the open-loop run's own pre-step states of row 0, which every row starts from (the start states repeat one
    # state when rows == starts is not asked for): rows equal to row 0 run the open-loop trajectory exactly (dx = 0), so the
    # difference in time is the feedback's own cost whatever K is
    q, v, w = (x[:1].expand(rows, -1).contiguous() for x in (q, v, w))
    u = u[:1].expand(rows, -1, -1).contiguous()
    kw["qacc_warmstart"] = w
    nom = env.rollout(q[:1], v[:1], u[:1], **(kw | dict(qacc_warmstart=w[:1])))
    qr = torch.cat([q[:1, None], nom["qpos"][:, :-1]], 1).contiguous()
    vr = torch.cat([v[:1, None], nom["qvel"][:, :-1]], 1).contiguous()
    Ks = torch.randn(1, T, m.nu, nx, generator=gen, device=q.device)
    shared = dict(gains=Ks, qpos_ref=qr, qvel_ref=vr)
    ms_open = timed(lambda: env.rollout(q, v, u, **kw), reps, flush)
    same_as_open = bool(torch.equal(env.rollout(q, v, u, **kw)["qpos"], env.rollout(q, v, u, **kw, **shared)["qpos"]))
    ms_shared = timed(lambda: env.rollout(q, v, u, **kw, **shared), reps, flush)
    got = env.rollout(q, v, u, **kw, **shared)
    Kp = Ks.expand(rows, -1, -1, -1).contiguous()
    per = dict(gains=Kp, qpos_ref=qr.expand(rows, -1, -1).contiguous(), qvel_ref=vr.expand(rows, -1, -1).contiguous())
    ms_row = timed(lambda: env.rollout(q, v, u, **kw, **per), reps, flush)
    same_per_row = bool(torch.equal(env.rollout(q, v, u, **kw, **per)["qpos"], got["qpos"]))
    del Kp, per
    scratch = HumanoidBatchB200(cfg, num_envs=rows, device="cuda:0", seed=0)
    clip = mode == "action" and bool(cfg.env.clip_actions)
    first = host_loop(scratch, q, v, w, u, mode, Ks, qr, vr, clip)
    ctrl_err = float((first - got["control"][:, 0]).abs().max() / (got["control"][:, 0].abs().max() + 1e-12))
    ms_loop = timed(lambda: host_loop(scratch, q, v, w, u, mode, Ks, qr, vr, clip), reps, flush)
    o, s, r, lp = (float(np.mean(x)) for x in (ms_open, ms_shared, ms_row, ms_loop))
    return dict(case=name, robot=robot, mode=mode, rows=rows, steps=T, open_loop_ms=o, feedback_shared_ms=s, feedback_per_row_ms=r,
                host_loop_ms=lp, shared_over_open=s / o, per_row_over_open=r / o, speedup_vs_host_loop=lp / s,
                gain_bytes_per_row=T * m.nu * nx * 4, shared_equals_expanded=same_per_row, closed_equals_open_loop=same_as_open, host_first_control_relerr=ctrl_err,
                min_ms=dict(open=float(np.min(ms_open)), shared=float(np.min(ms_shared)), per_row=float(np.min(ms_row)),
                            host_loop=float(np.min(ms_loop))))


def stabilisation(gen, n=256, T=30):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "examples"))
    import ilqr_track as ex
    cfg = make_cfg(env="speed", robot="smpl_humanoid", overrides={"env.control_mode": "torque"})
    env = HumanoidBatchB200(cfg, num_envs=n, device="cuda:0", seed=0)
    m = env.model
    prob = ex.make_problem(env, T=T, seed=1)
    prob["u0"] = prob["u0"] / 0.3   # the nominal is the target itself: tracking a feasible trajectory
    nom = ex.nominal(env, prob)
    prob["qpos_tgt"], prob["qvel_tgt"] = nom["qpos"][0].double(), nom["qvel"][0].double()
    # perturbed starts: positions by integrate_pos of tangent noise, velocities by noise
    dq = torch.randn(n, m.nv, generator=gen, device=env.device) * 0.02
    q0 = env.integrate_pos(prob["q0"].expand(n, -1), dq).float().contiguous()
    v0 = (prob["v0"] + torch.randn(n, m.nv, generator=gen, device=env.device) * 0.2).contiguous()
    u = nom["control"].expand(n, -1, -1).contiguous()
    K, _, qs, vs = ex.backward(env, prob, nom)   # TVLQR around the nominal: its k is 0, the nominal being the target
    ol = env.rollout(q0, v0, u, mode="ctrl", nsub=1)
    cl = env.rollout(q0, v0, u, mode="ctrl", nsub=1, gains=K.float()[None].contiguous(), qpos_ref=qs[None].contiguous(),
                     qvel_ref=vs[None].contiguous())
    dev = lambda out: torch.cat([env.differentiate_pos(nom["qpos"][0, -1], out["qpos"][:, -1]),
                                 out["qvel"][:, -1] - nom["qvel"][0, -1]], -1).norm(dim=-1)  # noqa: E731
    d0 = torch.cat([dq, v0 - prob["v0"]], -1).norm(dim=-1)
    return dict(case="tvlqr-stabilisation-smpl", rows=n, steps=T, start_deviation_mean=float(d0.mean()),
                open_loop_final_deviation_mean=float(dev(ol).mean()), closed_loop_final_deviation_mean=float(dev(cl).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/rollout_feedback_bench.jsonl")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rollout_feedback_bench: no CUDA device (this measures the H100 kernels; there is no CPU mode)")
    gpu = card()
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    rows = []
    for case in CASES:
        r = run(*case, args.reps, gen, flush)
        r["gpu"] = gpu
        rows.append(r)
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()
    st = stabilisation(gen)
    st["gpu"] = gpu
    rows.append(st)
    print(json.dumps(st), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rollout_feedback_bench.jsonl"), "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
