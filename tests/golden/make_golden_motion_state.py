#!/usr/bin/env python
"""Generate tests/golden/motion_state.npz with the REFERENCE's torch motion library: MotionLibBaseTorch.get_motion_state and
_calc_frame_blend (smpl_sim/smpllib/motion_lib_base_torch.py:434-499, 528-538) with torch_utils.slerp (smpl_sim/utils/torch_utils.py:
405-426), float32 on the CPU.  As in make_golden_motion.py the methods are executed from the reference SOURCE TEXT on a namespace that
carries the tables they read (importing the modules needs the SMPL / joblib / isaac stacks).

Inputs: four small clips of 2, 5, 9 and 14 frames at 30, 25, 60 and 30 fps, three bodies, random unit rotations with planted pairs of
consecutive frames: a negative dot product (clip 1, frames 1 -> 2), nearly equal rotations, the midpoint fallback (clip 2, frames
3 -> 4), and identical rotations (clip 3, frames 5 -> 6); query times negative, zero, on frames, between frames, at the clip's length
and past it; every query once without and once with a root offset."""
import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
REF = os.environ.get("SMPLSIM_REFERENCE", "/root/reference")


def _functions(path, names):
    tree = ast.parse(open(os.path.join(REF, path)).read())
    fns = [n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name in names]
    for f in fns:
        f.decorator_list = []   # torch.jit.script: the same arithmetic, run eagerly
    return fns


class _Dict(dict):
    __getattr__ = dict.__getitem__


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _rotate_small(q, angle, rng):
    """q times a rotation by `angle` about a random axis (wxyz)."""
    ax = _unit(rng.normal(size=3))
    d = np.array([np.cos(angle / 2), *(np.sin(angle / 2) * ax)])
    w1, x1, y1, z1 = q
    w2, x2, y2, z2 = d
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def main():
    ns = {"torch": torch}
    for f in _functions("smpl_sim/utils/torch_utils.py", ("slerp",)):
        exec(compile(ast.Module(body=[f], type_ignores=[]), "torch_utils.py", "exec"), ns)
    tu = types.SimpleNamespace(slerp=ns["slerp"])
    env = {"torch": torch, "torch_utils": tu, "EasyDict": _Dict}
    exec(compile(ast.Module(body=_functions("smpl_sim/smpllib/motion_lib_base_torch.py", ("get_motion_state", "_calc_frame_blend")),
                            type_ignores=[]), "motion_lib_base_torch.py", "exec"), env)

    rng = np.random.default_rng(11)
    nframes = np.array([2, 5, 9, 14])
    fps = np.array([30.0, 25.0, 60.0, 30.0])
    dt = (1.0 / fps).astype(np.float32)
    mlen = (dt * (nframes - 1)).astype(np.float32)
    starts = np.concatenate([[0], np.cumsum(nframes)[:-1]])
    Ftot, nb, nd = int(nframes.sum()), 3, 6
    gts = rng.normal(size=(Ftot, nb, 3)).astype(np.float32)
    grs = _unit(rng.normal(size=(Ftot, nb, 4)))
    # smooth-ish rotations inside each clip: frame k+1 = frame k turned by up to 0.5 rad, then planted pairs
    for c in range(4):
        for k in range(1, nframes[c]):
            for b in range(nb):
                grs[starts[c] + k, b] = _rotate_small(grs[starts[c] + k - 1, b], rng.uniform(0.05, 0.5), rng)
    r = starts[1] + 1
    grs[r + 1] = -np.stack([_rotate_small(grs[r, b], 0.3, rng) for b in range(nb)])          # negative dot product
    r = starts[2] + 3
    grs[r + 1] = np.stack([_rotate_small(grs[r, b], 1e-3, rng) for b in range(nb)])         # |sin(half angle)| = 5e-4 < 0.001
    r = starts[3] + 5
    grs[r + 1] = grs[r]                                                                        # identical
    grs = grs.astype(np.float32)
    gvs = rng.normal(size=(Ftot, nb, 3)).astype(np.float32)
    gavs = rng.normal(size=(Ftot, nb, 3)).astype(np.float32)
    dof_pos = rng.normal(size=(Ftot, nd)).astype(np.float32)
    dvs = rng.normal(size=(Ftot, nd // 3, 3)).astype(np.float32)   # [F, J, 3] as the library holds it: dof_vel's blend is [n, 1, 1]
    aa = rng.normal(size=(Ftot, 3 * nb)).astype(np.float32)
    bodies = rng.normal(size=(4, 17)).astype(np.float32)

    ids, times = [], []
    for c in range(4):
        L, d = float(mlen[c]), float(dt[c])
        ts = [-0.3, -1e-3, 0.0, L, L + 0.2, L + 10.0]
        ts += [np.float32(k) * np.float32(d) for k in range(nframes[c])]                      # on frames (float32 products)
        ts += list(rng.uniform(0.0, L, 6))                                                      # between frames
        ts += [(k + 0.5) * d for k in range(min(nframes[c] - 1, 7))]                           # mid-frame, every planted pair
        ids += [c] * len(ts)
        times += ts
    ids = np.array(ids, np.int64)
    times = np.array(times, np.float32)
    offset = rng.normal(size=(len(ids), 3)).astype(np.float32)

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    lib = types.SimpleNamespace(_motion_lengths=t(mlen), _motion_num_frames=t(nframes.astype(np.int64)), _motion_dt=t(dt),
                                length_starts=t(starts.astype(np.int64)), dof_pos=t(dof_pos), gvs=t(gvs), gavs=t(gavs), gts=t(gts),
                                dvs=t(dvs), grs=t(grs), _motion_aa=t(aa), _motion_bodies=t(bodies), num_bodies=nb)
    lib._get_num_bodies = types.MethodType(lambda self: self.num_bodies, lib)
    lib._calc_frame_blend = types.MethodType(env["_calc_frame_blend"], lib)
    gms = types.MethodType(env["get_motion_state"], lib)
    f0, f1, bl = lib._calc_frame_blend(t(times).clone(), lib._motion_lengths[t(ids)], lib._motion_num_frames[t(ids)], lib._motion_dt[t(ids)])
    out = dict(num_frames=nframes.astype(np.int32), motion_dt=dt, motion_len=mlen, length_starts=starts.astype(np.int32),
               gts=gts, grs=grs, gvs=gvs, gavs=gavs, dof_pos=dof_pos, dof_vel=dvs.reshape(Ftot, nd), motion_aa=aa, motion_bodies=bodies,
               ids=ids.astype(np.int32), times=times, offset=offset, frame_idx0=f0.numpy().astype(np.int32),
               frame_idx1=f1.numpy().astype(np.int32), blend=bl.numpy().astype(np.float32))
    keys = ("root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "motion_aa", "rg_pos", "rb_rot", "body_vel",
            "body_ang_vel", "motion_bodies")
    for tag, off in (("", None), ("off_", t(offset))):
        st = gms(t(ids), t(times), off)
        for k in keys:
            out["out_" + tag + k] = st[k].numpy()
    assert all(out["out_" + k].dtype == np.float32 for k in keys)
    np.savez_compressed(os.path.join(HERE, "motion_state.npz"), **out)
    print("motion_state.npz:", len(ids), "queries; blend in (0, 1):", int(((out["blend"] > 0) & (out["blend"] < 1)).sum()),
          "f0 == f1:", int((out["frame_idx0"] == out["frame_idx1"]).sum()))


if __name__ == "__main__":
    main()
