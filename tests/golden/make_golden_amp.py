#!/usr/bin/env python
"""Generate tests/golden/amp_obs.npz with the REFERENCE's own AMP observation code (build container only: needs the reference tree):

  compute_humanoid_observations_smpl   smpl_sim/envs/nv/humanoid.py:2530-2602
  dof_to_obs                           smpl_sim/envs/nv/humanoid.py:2276-2309
  remove_base_rot                      smpl_sim/envs/nv/humanoid.py:2523-2527

humanoid.py imports isaacgym, so the three functions are lifted out of its source (ast) without their @torch.jit.script decorators and
run with the reference's own quaternion helpers (smpl_sim/utils/torch_utils.py: quat_mul, quat_conjugate, quat_from_angle_axis,
calc_heading_quat_inv, quat_to_tan_norm, my_quat_rotate, exp_map_to_quat) in place of isaacgym.torch_utils.  Everything runs in float64.
Inputs are stored in this project's wxyz convention and converted to the reference's xyzw at the call.

    python tests/golden/make_golden_amp.py"""
import ast
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402  (installs the third-party stubs, puts the reference on sys.path)

import torch  # noqa: E402

torch.set_default_dtype(torch.float64)   # dof_to_obs allocates its output with the default dtype
tu = MG._import_with_stubs(lambda: importlib.import_module("smpl_sim.utils.torch_utils"))


def lift():
    src = open(os.path.join(MG.REF, "smpl_sim", "envs", "nv", "humanoid.py")).read()
    want = {"dof_to_obs", "remove_base_rot", "compute_humanoid_observations_smpl"}
    defs = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in want]
    assert {d.name for d in defs} == want
    for d in defs:
        d.decorator_list = []
    ns = dict(torch=torch, torch_utils=tu, quat_mul=tu.quat_mul, quat_conjugate=tu.quat_conjugate, quat_from_angle_axis=tu.quat_from_angle_axis)
    exec(compile(ast.Module(body=defs, type_ignores=[]), "humanoid.py", "exec"), ns)
    return ns["compute_humanoid_observations_smpl"]


def rand_quat(rng, m):
    q = rng.normal(size=(m, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def states(rng, nb, m, nkey):
    nj = nb - 1
    d = dict(root_pos=rng.normal(size=(m, 3)) + [0, 0, 0.9], root_rot=rand_quat(rng, m), root_vel=rng.normal(size=(m, 3)),
             root_ang_vel=rng.normal(size=(m, 3)) * 2, dof_pos=rng.uniform(-1.3, 1.3, (m, 3 * nj)), dof_vel=rng.normal(size=(m, 3 * nj)) * 3,
             key_pos=rng.normal(size=(m, nkey, 3)) * 0.6)
    dof = d["dof_pos"].reshape(m, nj, 3)
    dof[0] = 0.0                                                   # the zero pose
    d["root_rot"][0] = [1, 0, 0, 0]
    d["root_rot"][1] = [0.5, 0.5, 0.5, 0.5]                        # the SMPL base rotation (upright after remove_base_rot)
    u = rng.normal(size=(nj, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    for row, norm in ((2, 1e-5 * 1.01), (3, 1e-5 * 0.99), (4, 3.5), (5, 2 * np.pi - 1e-3), (6, 5.0), (7, 1e-6)):
        dof[row] = u * norm                                        # exp-map norms around the 1e-5 threshold and above pi
    dof[8, ::2] = u[::2] * 4.2
    d["dof_pos"] = dof.reshape(m, -1)
    return d


def main():
    ref = lift()
    rng = np.random.default_rng(20261016)
    out = {}
    cases = []
    for nb in (24, 52):
        combos = [(u, lo, rh) for u in (0, 1) for lo in (0, 1) for rh in (0, 1)] if nb == 24 else [(0, 1, 1), (1, 0, 0)]
        for upright, local, root_h in combos:
            m, nkey = 24, 4
            s = states(rng, nb, m, nkey)
            T = lambda a: torch.as_tensor(a, dtype=torch.float64)  # noqa: E731
            xyzw = s["root_rot"][:, [1, 2, 3, 0]]
            obs = ref(T(s["root_pos"]), T(xyzw), T(s["root_vel"]), T(s["root_ang_vel"]), T(s["dof_pos"]), T(s["dof_vel"]), T(s["key_pos"]),
                      6 * (nb - 1), list(range(0, 3 * nb - 2, 3)), torch.zeros(m, 1), bool(local), bool(root_h), bool(upright), False)
            i = len(cases)
            cases.append([nb, upright, local, root_h])
            for k, v in s.items():
                out[f"c{i}_{k}"] = v
            out[f"c{i}_obs"] = obs.numpy()
    out["cases"] = np.array(cases, dtype=np.int64)
    path = os.path.join(HERE, "amp_obs.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()
