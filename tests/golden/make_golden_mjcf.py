#!/usr/bin/env python
"""Generate tests/golden/mjcf_parse.npz: the in-repo MJCF parser's model tables for the original project's two humanoid XML
files, so that tests/test_model_assets_cpu.py can check the shipped assets against them without the original project's tree.

    python tests/golden/make_golden_mjcf.py <original project tree>

smpl  <- smpl_sim/data/assets/mjcf/smpl_humanoid.xml   (24 bodies)
smplx <- smpl_humanoid.xml at the tree's root          (52 bodies)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from smplsim_b200.model import load_model  # noqa: E402

XMLS = {"smpl": "smpl_sim/data/assets/mjcf/smpl_humanoid.xml", "smplx": "smpl_humanoid.xml"}
FIELDS = ("body_parent", "body_pos", "body_quat", "body_mass", "body_ipos", "body_inertia", "dof_armature", "dof_range", "dof_invweight0",
          "geom_type", "geom_body", "geom_pos", "geom_mat", "geom_size", "act_kp", "act_kd", "act_torque_lim", "act_scale", "act_offset")
NAMES = ("body_names", "joint_names", "geom_names")

if __name__ == "__main__":
    ref = sys.argv[1]
    out = {}
    for name, rel in XMLS.items():
        m = load_model(os.path.join(ref, rel))
        for f in FIELDS:
            out[f"{name}/{f}"] = np.asarray(getattr(m, f))
        for f in NAMES:
            out[f"{name}/{f}"] = np.asarray(getattr(m, f), dtype=str)
    np.savez_compressed(os.path.join(HERE, "mjcf_parse.npz"), **out)
    print("mjcf_parse.npz:", len(out), "arrays")
