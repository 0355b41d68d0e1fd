"""The active-set solve's initial working set changes where the search starts, not where it ends: two `mj_step` substeps of 256 SMPL
envs from stepped states (standing, stumbling with foot strikes, falling, lying) held to what the build before the current rule
computed (tests/golden/ws_start_mj_step.npz, emulator) and to the fp64 oracle.  The second substep starts from the working set the
first leaves, so both rules for held contacts run.

Bounds: the parity bound of tests/test_gpu_parity.py, 1e-4 norm-relative (max|d| / max(1, max|x|)) on qpos, qvel and qacc against
the earlier build (fp32 against fp32: the solves end on the same optimum, up to the line search's tolerance where one ends on a
line-search step); against the oracle qpos / qvel 1e-4 and qacc 5e-4 as there, outside the contact-margin guard band."""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from conftest import GOLDEN  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from util_states import make_models, relerr  # noqa: E402

TOL = 1e-4


def test_ws_start_matches_previous_rule_and_oracle(backend):
    g = np.load(os.path.join(GOLDEN, "ws_start_mj_step.npz"))
    q, v, w, ctrl = g["q"], g["v"], g["w"], g["ctrl"]
    n = q.shape[0]
    cfg, om = make_models(control_mode="torque")
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 2)
    gq, gv, ga = env.qpos.cpu().numpy(), env.qvel.cpu().numpy(), env.qacc.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    st = env.status.cpu().numpy()
    assert not (st & (8 | 16)).any(), ("rows dropped / iteration cap", st)
    assert not (g["status"] & (8 | 16)).any()
    worst = 0.0
    for i in range(n):
        for name, a, b in (("qpos", gq, g["qpos"]), ("qvel", gv, g["qvel"]), ("qacc", ga, g["qacc"])):
            worst = max(worst, relerr(a[i], b[i]))
            assert relerr(a[i], b[i]) < TOL, (name, i, relerr(a[i], b[i]))
    nskip = 0
    for i in range(n):
        e = orc.OracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]; e.ctrl[:] = ctrl[i]
        guard = False
        for _ in range(2):
            e.mj_step()
            con = e.contacts()
            guard |= bool((np.abs(con["dist"] - om.model.margin) < 1e-5).any()) if e.ncon else False
        if guard or int(gmask[i]) != e.contact_mask:
            nskip += 1
            continue
        assert relerr(gq[i], e.qpos) < TOL, ("qpos vs oracle", i, relerr(gq[i], e.qpos))
        assert relerr(gv[i], e.qvel) < TOL, ("qvel vs oracle", i, relerr(gv[i], e.qvel))
        assert relerr(ga[i], e.qacc) < 5e-4, ("qacc vs oracle", i, relerr(ga[i], e.qacc))
    assert nskip <= n // 10, f"{nskip} of {n} states skipped for a contact inside the guard band"
    same = int((ga.view(np.int32) == g["qacc"].view(np.int32)).all(axis=1).sum())
    print(f"{backend.name}: worst norm-relative vs the earlier rule {worst:.2e}; qacc bit-identical in {same} of {n} envs; "
          f"{nskip} states in the guard band")
