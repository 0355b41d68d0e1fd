"""Choose the default eps of smplsim_inverse_fd: dfrc on the host emulator against a centered fp64 oracle FD of the inverse at the same
eps, for x0.1, x1 and x10 of (eps_qpos, eps_qvel, eps_qacc) = (1e-2, 1e-1, 1.0) (CPU only; the emulator runs the kernel source).

States: 8 SMPL and 4 SMPL-X states of tests/test_forward_fd.py's _states (floor contacts, joint-limit rows, airborne), qacc the oracle's
forward qacc.  Per scale and block (dq / qvel / qacc): median and max over the states of ||K - O||_F / max(1, ||O||_F) on the columns
neither side flags, and the number of excluded columns (flagged by the kernel or switched in the oracle).

    python tools/inverse_fd_eps.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from conftest import Backend  # noqa: E402
from test_inverse_fd import _blocks, _inv_states, oracle_dfrc  # noqa: E402

BASE = (1e-2, 1e-1, 1.0)


def main() -> int:
    b = Backend("emu")
    for robot, n in (("smpl_humanoid", 8), ("smplx_humanoid", 4)):
        cfg, om, q, v, a, _ = _inv_states(robot, n, seed=11, nair=2)
        nv = om.model.nv
        env = b.batch(cfg, 64)
        for sc in (0.1, 1.0, 10.0):
            eps = tuple(e * sc for e in BASE)
            fd = env.inverse_fd(b.t(q), b.t(v), b.t(a), *eps)
            K, F = fd["dfrc"].numpy().astype(np.float64), fd["flags"].numpy()
            err = {k: [] for k in _blocks(nv)}
            exc = {k: 0 for k in _blocks(nv)}
            for i in range(n):
                O, sw = oracle_dfrc(om, q[i], v[i], a[i], eps)
                keep = (F[i] == 0) & ~sw
                for k, s in _blocks(nv).items():
                    kk = keep[s]
                    exc[k] += int((~kk).sum())
                    if kk.any():
                        d = K[i][:, s][:, kk] - O[:, s][:, kk]
                        err[k].append(np.linalg.norm(d) / max(1.0, np.linalg.norm(O[:, s][:, kk])))
            row = "  ".join(f"{k} {np.median(e):.1e} / {np.max(e):.1e} ({exc[k]}/{n * nv})" for k, e in err.items())
            print(f"{robot:<15} x{sc:<5} eps {eps}: {row}", flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
