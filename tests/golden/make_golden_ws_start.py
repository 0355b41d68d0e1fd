#!/usr/bin/env python
"""Generate tests/golden/ws_start_mj_step.npz: two `mj_step` substeps of 256 SMPL envs from seeded stepped states, run on the host
SIMT emulator build of the kernels (tests/emu).  The states come from fp64 oracle rollouts under stable PD with random actions:
standing, stumbling with foot strikes, falling and lying.  The first substep starts from an empty working-set memory (every
contact is new); the second starts from the working set the first leaves, which is where the solver's initial-working-set rule
acts.  The committed file was generated with the build before the rule took the union of the inherited and the predicted rows
(contacts held from the previous substep started from the inherited rows alone) and before slots were keyed by contact point
(they followed the contact's position in its geom's list), so tests/test_ws_start.py holds the current build to what that one
computed.

    SMPLSIM_EMU_SO=<emulator build> python tests/golden/make_golden_ws_start.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, os.path.join(HERE, "..", "emu"))
import emu_env  # noqa: E402
from util_states import make_models, rollout_states  # noqa: E402

N, NSUB = 256, 2


def inputs():
    """(q, v, qacc_warm, ctrl) of the fixture, all reproducible from the seeds."""
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], N, seed=23)
    ctrl = np.random.default_rng(7).uniform(-60, 60, (N, q.shape[1] - 7))
    return q, v, w, ctrl


def run(q, v, w, ctrl):
    import torch
    cfg, _ = make_models(control_mode="torque")
    env = emu_env.EmuBatch(cfg, N, seed=0)
    f = lambda x: torch.as_tensor(np.asarray(x, dtype=np.float32))  # noqa: E731
    env.set_state(f(q), f(v))
    env.qacc_warm.copy_(f(w))
    env.mj_step(f(ctrl), NSUB)
    return {"qpos": env.qpos.numpy().copy(), "qvel": env.qvel.numpy().copy(), "qacc": env.qacc.numpy().copy(),
            "solver_iter": env.solver_iter.numpy().copy(), "status": env.status.numpy().copy()}


if __name__ == "__main__":
    q, v, w, ctrl = inputs()
    out = run(q, v, w, ctrl)
    np.savez_compressed(os.path.join(HERE, "ws_start_mj_step.npz"), q=q, v=v, w=w, ctrl=ctrl, **out)
    print("wrote ws_start_mj_step.npz; solver_iter histogram", np.bincount(out["solver_iter"]), "status", np.unique(out["status"]))
