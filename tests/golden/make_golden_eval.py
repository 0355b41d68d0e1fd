#!/usr/bin/env python
"""Generate tests/golden/eval_metrics.npz with the REFERENCE's tracking metrics: compute_metrics_lite, compute_metrics_obj, p_mpjpe,
compute_error_vel and compute_error_accel (smpl_sim/smpllib/smpl_eval.py), float64 on the CPU.  As in make_golden_motion_state.py the
functions are executed from the reference SOURCE TEXT (importing the module needs the SMPL stack).

Inputs, one group at 24 bodies (SMPL) and one at 52 (SMPL-X), float32: clips of 1, 2, 3 and several tens of frames.  Reference
positions: a fixed random body layout per clip (within ~0.8 m of the root) swaying frame to frame, the root walking up to ~2 m;
simulated = reference + N(0, 3 cm).  Planted frames in the long clip of each group:
  - scaled + rotated + shifted copy of the reference (Procrustes error ~0);
  - reflected copy (mirror through a plane, + 1 cm noise): the det(R) < 0 branch;
  - collinear frame: reference and simulated points all on lines (rank-1 cross-covariance, repeated zero singular values);
  - relative rotations near pi (pi - 1e-3) on every body.
Rotations are stored wxyz (this project's order) and handed to the reference as xyzw.

Stored per group g in (b24, b52): g_nframes [C], g_gt_pos / g_pred_pos [sum F, J, 3], g_gt_rot / g_pred_rot [sum F, J, 4] (wxyz);
the per-frame metrics (means over bodies) g_mpjpe_g, g_mpjpe_l, g_mpjpe_pa, g_rot_error [sum F], g_vel_dist [sum (F - 1)],
g_accel_dist [sum max(F - 2, 0)]; and the concatenated means g_mean_<metric> = compute_metrics_lite(..., concatenate=True)[k].mean()."""
import ast
import os
from collections import defaultdict

import numpy as np
from scipy.spatial.transform import Rotation as sRot

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SMPLSIM_REFERENCE", "/root/reference")
NAMES = ("compute_metrics_lite", "compute_metrics_obj", "p_mpjpe", "compute_error_vel", "compute_error_accel")
METRICS = ("mpjpe_g", "mpjpe_l", "mpjpe_pa", "vel_dist", "accel_dist", "rot_error")


def reference_functions():
    tree = ast.parse(open(os.path.join(REF, "smpl_sim/smpllib/smpl_eval.py")).read())
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert sorted(f.name for f in fns) == sorted(NAMES)
    ns = {"np": np, "sRot": sRot, "defaultdict": defaultdict, "tqdm": lambda x: x}
    exec(compile(ast.Module(body=fns, type_ignores=[]), "smpl_eval.py", "exec"), ns)
    return ns


def rot_about(axis, angle):
    axis = axis / np.linalg.norm(axis)
    return sRot.from_rotvec(axis * angle)


def make_group(rng, J, lengths):
    gt_pos, pred_pos, gt_rot, pred_rot = [], [], [], []
    for ci, F in enumerate(lengths):
        layout = rng.normal(size=(J, 3)) * 0.35
        layout[0] = 0.0                                        # body 0 is the root
        root = np.cumsum(rng.normal(size=(F, 3)) * [0.04, 0.04, 0.005], 0) + [0.0, 0.0, 0.9]
        sway = np.cumsum(rng.normal(size=(F, J, 3)) * 0.01, 0)
        sway[:, 0] = 0.0
        g = root[:, None, :] + layout[None] + sway
        p = g + rng.normal(size=g.shape) * 0.03
        qg = sRot.random(F * J, random_state=rng.integers(1 << 31)).as_quat().reshape(F, J, 4)           # xyzw
        dq = sRot.from_rotvec(rng.normal(size=(F * J, 3)) * 0.1)
        qp = (dq * sRot.from_quat(qg.reshape(-1, 4))).as_quat().reshape(F, J, 4)
        if F >= 20:
            # scaled, rotated and shifted copy: Procrustes error ~0
            R = rot_about(rng.normal(size=3), 1.1)
            p[5] = 1.3 * R.apply(g[5] - g[5, 0]) + g[5, 0] + [0.2, -0.1, 0.05]
            # reflected copy through the plane x = root_x, plus noise: the improper best fit is refused
            p[9] = g[9] * [-1.0, 1.0, 1.0] + [2 * g[9, 0, 0], 0.0, 0.0] + rng.normal(size=(J, 3)) * 0.01
            # collinear frame: every reference and simulated point on a line through its root
            u, v = rng.normal(size=3), rng.normal(size=3)
            u, v = u / np.linalg.norm(u), v / np.linalg.norm(v)
            s = rng.uniform(-0.8, 0.8, J)
            s[0] = 0.0
            g[13] = g[13, 0] + s[:, None] * u
            p[13] = p[13, 0] + (s + rng.normal(size=J) * 0.02)[:, None] * v
            # relative rotation pi - 1e-3 on every body
            ax = rng.normal(size=(J, 3))
            flip = sRot.from_rotvec(ax / np.linalg.norm(ax, axis=1, keepdims=True) * (np.pi - 1e-3))
            qp[17] = (flip.inv() * sRot.from_quat(qg[17])).as_quat()
        gt_pos.append(g.astype(np.float32)); pred_pos.append(p.astype(np.float32))
        gt_rot.append(qg.astype(np.float32)); pred_rot.append(qp.astype(np.float32))
    return gt_pos, pred_pos, gt_rot, pred_rot


def wxyz(q):
    return np.concatenate([q[..., 3:], q[..., :3]], -1)


def main():
    ref = reference_functions()
    rng = np.random.default_rng(23)
    out = {}
    for tag, J, lengths in (("b24", 24, [1, 2, 3, 41, 12]), ("b52", 52, [3, 1, 27, 2])):
        gt_pos, pred_pos, gt_rot, pred_rot = make_group(rng, J, lengths)
        f64 = lambda xs: [x.astype(np.float64) for x in xs]  # noqa: E731   the reference runs in float64 on the float32 inputs
        gp, pp, gr, pr = f64(gt_pos), f64(pred_pos), f64(gt_rot), f64(pred_rot)
        gr = [q / np.linalg.norm(q, axis=-1, keepdims=True) for q in gr]          # what sRot.from_quat does to its input
        pr = [q / np.linalg.norm(q, axis=-1, keepdims=True) for q in pr]
        lite = ref["compute_metrics_lite"](pp, gp, pr, gr, root_idx=0, use_tqdm=False, concatenate=False)
        obj = ref["compute_metrics_obj"](pp, gp, pr, gr, root_idx=0, use_tqdm=False, concatenate=False)
        per = defaultdict(list)
        for c, F in enumerate(lengths):
            per["mpjpe_g"].append(lite["mpjpe_g"][c].mean(1))
            per["mpjpe_l"].append(lite["mpjpe_l"][c].mean(1))
            per["mpjpe_pa"].append(lite["mpjpe_pa"][c].mean(1))
            per["rot_error"].append(lite["rot_error"][c].reshape(F, J).mean(1))
            per["vel_dist"].append(lite["vel_dist"][c])
            per["accel_dist"].append(lite["accel_dist"][c])
            for k in ("mpjpe_g", "rot_error", "vel_dist", "accel_dist"):        # the two reference functions agree
                assert np.allclose(lite[k][c], obj[k][c], rtol=0, atol=1e-9), k
            # p_mpjpe and the error functions called directly give the same arrays
            rel = lambda x: x - x[:, [0]]  # noqa: E731
            assert np.allclose(ref["p_mpjpe"](rel(pp[c]), rel(gp[c])) * 1000, lite["mpjpe_pa"][c], atol=1e-9)
            assert np.allclose(ref["compute_error_vel"](pp[c], gp[c]) * 1000, lite["vel_dist"][c], atol=1e-9)
            assert np.allclose(ref["compute_error_accel"](pp[c], gp[c]) * 1000, lite["accel_dist"][c], atol=1e-9)
        conc = ref["compute_metrics_lite"](pp, gp, pr, gr, root_idx=0, use_tqdm=False, concatenate=True)
        out[f"{tag}_nframes"] = np.asarray(lengths, np.int32)
        out[f"{tag}_gt_pos"], out[f"{tag}_pred_pos"] = np.concatenate(gt_pos), np.concatenate(pred_pos)
        out[f"{tag}_gt_rot"], out[f"{tag}_pred_rot"] = wxyz(np.concatenate(gt_rot)), wxyz(np.concatenate(pred_rot))
        for k in METRICS:
            out[f"{tag}_{k}"] = np.concatenate(per[k])
            out[f"{tag}_mean_{k}"] = np.float64(conc[k].mean())
        pa = out[f"{tag}_mpjpe_pa"]
        long_start = int(np.sum(lengths[:int(np.argmax(lengths))]))
        print(tag, "frames", sum(lengths), "PA at the planted frames (copy, reflected, collinear):",
              pa[long_start + 5], pa[long_start + 9], pa[long_start + 13], "rot near pi:", out[f"{tag}_rot_error"][long_start + 17])
    np.savez_compressed(os.path.join(HERE, "eval_metrics.npz"), **out)


if __name__ == "__main__":
    main()
