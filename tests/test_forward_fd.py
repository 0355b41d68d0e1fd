"""Forward dynamics on caller rows (smplsim_forward, HumanoidBatchB200.forward) and finite-difference transition derivatives
(smplsim_transition_fd, HumanoidBatchB200.transition_fd, envs.mjd_transitionFD) against the fp64 oracle.

States: rollouts of the speed task (floor contacts, joint-limit rows) and airborne states.  The kernel tests run on the H100 (-m gpu)
and on the host emulator build of the same kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from smplsim_b200.abi import SmplsimFdCfgC
from test_inverse import TOL as INV_TOL, _forward, _over_cap, _weight
from util_states import airborne_states, make_models, relerr, rollout_states

QACC_TOL = 5e-4     # forward qacc against the oracle, norm-relative (the mj_step qacc bound of test_xfrc)
EPS = (1e-2, 1e-1, 1.0)   # the defaults
# dqacc against a centered fp64 oracle FD at the same eps: per column max|k - o| / max(1, max|o|), and per block (dq / qvel / ctrl)
# ||K - O||_F / max(1, ||O||_F), on columns neither side flags; a column is held to the largest entry of its block.  Worst seen on the
# emulator: column 8.6e-4, block 3.2e-3 (SMPL), column 5.9e-4, block 2.8e-3 (SMPL-X).
COL_TOL, BLOCK_TOL = 1e-2, 2e-2
MAX_EXCLUDED = 0.05


def _rollout(robot, n, seed):
    """Speed-task rollout states under random stable-PD actions, those with constraint rows (floor contacts, joint limits) first."""
    om = make_models(robot=robot, control_mode="uhc_pd")[1]
    q, v, _ = rollout_states(om, 4 * n, seed=seed, every=3)
    rows = np.array([_forward(om, q[i], v[i]).nefc > 0 for i in range(len(q))])
    pick = np.concatenate([np.flatnonzero(rows), np.flatnonzero(~rows)])[:n]
    return q[pick], v[pick], None


def _states(robot, n, seed, nair=2):
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    qa, va = airborne_states(m, nair, seed=seed)
    qc, vc, _ = _rollout(robot, n - nair, seed + 1)
    q, v = np.concatenate([qc, qa]), np.concatenate([vc, va])
    u = np.random.default_rng(seed + 2).uniform(-30, 30, (n, m.nu))
    return cfg, om, np.float32(q), np.float32(v), np.float32(u)


def _qexp(q, k, a):
    """q (x) exp(a e_k), normalised (wxyz)."""
    d = np.zeros(4); d[0] = np.cos(0.5 * a); d[1 + k] = np.sin(0.5 * a)
    w1, x1, y1, z1 = q; w2, x2, y2, z2 = d
    r = np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                  w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])
    return r / np.linalg.norm(r)


def _perturb(m, q, v, u, col, s):
    """(qpos, qvel, ctrl) in fp64 with column col of [dq, qvel, ctrl] moved by s."""
    q, v, u = q.astype(np.float64).copy(), v.astype(np.float64).copy(), u.astype(np.float64).copy()
    nv = m.nv
    if col < 3:
        q[col] += s
    elif col < 6:
        q[3:7] = _qexp(q[3:7], col - 3, s)
    elif col < nv:
        q[col + 1] += s
    elif col < 2 * nv:
        v[col - nv] += s
    else:
        u[col - 2 * nv] += s
    return q, v, u


def _oracle_env(om, q, v, u):
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.ctrl[:] = u
    return e


def _active(e):
    efc = e.efc()
    con = e.contacts()
    return (e.ncon, e.nefc, tuple(con["geom"]), tuple(efc["force"] > 0))


def _eps_of(m, col, eps):
    return eps[0] if col < m.nv else eps[1] if col < 2 * m.nv else eps[2]


def oracle_dqacc(om, q, v, u, eps):
    """Centered fp64 FD of the oracle's forward qacc at the fp32 state; and per column whether the oracle's active set switched."""
    m = om.model
    ncol = 2 * m.nv + m.nu
    D = np.zeros((m.nv, ncol)); switched = np.zeros(ncol, bool)
    for j in range(ncol):
        e = _eps_of(m, j, eps)
        r = []
        for s in (e, -e):
            o = _oracle_env(om, *_perturb(m, q, v, u, j, s))
            o.forward()
            r.append((o.qacc.copy(), _active(o)))
        D[:, j] = (r[0][0] - r[1][0]) / (2 * e)
        switched[j] = r[0][1] != r[1][1]
    return D, switched


def _blocks(m):
    nv = m.nv
    return {"dq": slice(0, nv), "qvel": slice(nv, 2 * nv), "ctrl": slice(2 * nv, 2 * nv + m.nu)}


def dqacc_errors(m, K, O, keep):
    """(worst column max|K_j - O_j| / max(1, max|O|) over the column's block, worst block ||K - O||_F / max(1, ||O||_F)) on the kept
    columns."""
    col = blk = 0.0
    for s in _blocks(m).values():
        k = np.zeros_like(keep); k[s] = keep[s]
        if k.any():
            d = K[:, k] - O[:, k]
            col = max(col, np.abs(d).max() / max(1.0, np.abs(O[:, s]).max()))
            blk = max(blk, np.linalg.norm(d) / max(1.0, np.linalg.norm(O[:, k])))
    return col, blk


# ------------------------------------------------------------------ 1-3. forward
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_forward_matches_oracle(backend, robot):
    n = 24 if robot == "smpl_humanoid" else 10
    cfg, om, q, v, u = _states(robot, n, seed=3, nair=3)
    env = backend.batch(cfg, 8)
    out = env.forward(backend.t(q), backend.t(v), backend.t(u))
    qacc, mask, st = out["qacc"].cpu().numpy(), out["contact_mask"].cpu().numpy(), out["status"].cpu().numpy()
    worst, ncmp, rows = 0.0, 0, 0
    for i in range(n):
        e = _forward(om, q[i], v[i], u[i])
        if _over_cap(e) or st[i]:
            continue
        err = relerr(qacc[i], e.qacc)
        assert err <= QACC_TOL, (i, err)
        assert int(mask[i]) == e.contact_mask, i
        worst = max(worst, err); ncmp += 1; rows += e.nefc > 0
    print(f"{ncmp}/{n} rows, worst qacc error {worst:.2e}")
    assert ncmp >= n - n // 10 and rows >= n // 4


def test_forward_matches_mj_step(backend):
    """At an env's own state, ctrl and warm start, forward's qacc is mj_step(ctrl, 1)'s aux.qacc."""
    cfg, om, q, v, u = _states("smpl_humanoid", 16, seed=5)
    w = np.float32(np.random.default_rng(1).normal(size=v.shape))
    env = backend.batch(cfg, 16)
    out = env.forward(backend.t(q), backend.t(v), backend.t(u), qacc_warmstart=backend.t(w))
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(u), 1)
    a, b = out["qacc"].cpu().numpy(), env.qacc.cpu().numpy()
    for i in range(16):
        assert relerr(a[i], b[i]) <= 1e-5, (i, relerr(a[i], b[i]))
    assert np.array_equal(out["contact_mask"].cpu().numpy(), env.contact_mask.cpu().numpy())


def test_round_trip_with_inverse(backend):
    """mj_compareFwdInv: inverse(q, v, forward(q, v, u).qacc) = [0_6 ; u]; forward's contact wrench is the inverse's."""
    cfg, om, q, v, u = _states("smpl_humanoid", 24, seed=7)
    m = om.model
    env = backend.batch(cfg, 8)
    out = env.forward(backend.t(q), backend.t(v), backend.t(u), contact_wrench=True)
    qfrc, cw = env.inverse(backend.t(q), backend.t(v), out["qacc"], contact_wrench=True)
    qfrc, cw, fcw = qfrc.cpu().numpy(), cw.cpu().numpy(), out["contact_wrench"].cpu().numpy()
    st = out["status"].cpu().numpy()
    wt = _weight(m)
    ncmp = 0
    for i in range(len(q)):
        if st[i]:
            continue
        want = np.r_[np.zeros(6), u[i]]
        assert np.abs(qfrc[i] - want).max() / max(wt, float(np.abs(want).max())) <= INV_TOL, i
        assert np.abs(fcw[i] - cw[i]).max() / max(wt, float(np.abs(cw[i]).max())) <= INV_TOL, i
        ncmp += 1
    assert ncmp >= len(q) - len(q) // 10


# ------------------------------------------------------------------ 4-8. derivatives
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_dqacc_matches_oracle(backend, robot):
    n = 4 if robot == "smpl_humanoid" else 2
    cfg, om, q, v, u = _states(robot, n, seed=11, nair=1)
    m = om.model
    env = backend.batch(cfg, 64)
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), dqacc=True)
    K, F = fd["dqacc"].cpu().numpy().astype(np.float64), fd["flags"].cpu().numpy()
    excluded = total = 0
    worst = [0.0, 0.0]
    for i in range(n):
        O, sw = oracle_dqacc(om, q[i], v[i], u[i], EPS)
        keep = (F[i] == 0) & ~sw
        excluded += int((~keep).sum()); total += keep.size
        col, blk = dqacc_errors(m, K[i], O, keep)
        worst = [max(worst[0], col), max(worst[1], blk)]
    print(f"{robot}: {excluded}/{total} columns excluded, worst column {worst[0]:.2e}, worst block {worst[1]:.2e}")
    assert excluded <= MAX_EXCLUDED * total
    assert worst[0] <= COL_TOL and worst[1] <= BLOCK_TOL


def _tangent(m, q1, v1, q0, v0):
    """[mj_differentiatePos(q0 -> q1) ; v1 - v0] without the division by dt (root rotation in the body frame)."""
    nv = m.nv
    d = np.zeros(2 * nv)
    d[0:3] = q1[0:3] - q0[0:3]
    a, b = q0[3:7], q1[3:7]
    w = a[0] * b[0] + a[1:] @ b[1:]                          # q0^-1 q1
    vec = a[0] * b[1:] - b[0] * a[1:] - np.cross(a[1:], b[1:])
    s = np.linalg.norm(vec)
    d[3:6] = 0.0 if s == 0 else vec / s * 2 * np.arctan2(s, w)
    d[6:nv] = q1[7:] - q0[7:]
    d[nv:] = v1 - v0
    return d


def oracle_AB(om, q, v, u, qacc_warm, eps=1e-6):
    """A, B by a centered fp64 FD of one oracle mj_step at eps."""
    m = om.model
    nv, ncol = m.nv, 2 * m.nv + m.nu
    AB = np.zeros((2 * nv, ncol))
    for j in range(ncol):
        r = []
        for s in (eps, -eps):
            o = _oracle_env(om, *_perturb(m, q, v, u, j, s))
            o.qacc_warm[:] = qacc_warm
            o.mj_step()
            r.append((o.qpos.copy(), o.qvel.copy()))
        AB[:, j] = _tangent(m, r[0][0], r[0][1], r[1][0], r[1][1]) / (2 * eps)
    return AB[:, :2 * nv], AB[:, 2 * nv:]


def test_AB_matches_full_step_oracle(backend):
    """A - I and B against an fp64 FD of whole oracle steps; the root-rotation rows (R(th)^T, J_r(th)) on their own."""
    cfg, om, q, v, u = _states("smpl_humanoid", 3, seed=13, nair=1)
    m = om.model
    nv = m.nv
    v[:, 3:6] += np.float32([4.0, -6.0, 5.0])                 # a root rotation of ~0.02 rad per substep: R(th) and J_r(th) matter
    env = backend.batch(cfg, 64)
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u))
    A, B, F, qn = (fd[k].cpu().numpy().astype(np.float64) for k in ("A", "B", "flags", "qacc"))
    I = np.eye(2 * nv)
    worst = {}
    for i in range(len(q)):
        Ao, Bo = oracle_AB(om, q[i], v[i], u[i], qn[i])
        ka, kb = F[i, :2 * nv] == 0, F[i, 2 * nv:] == 0
        for name, K, O, keep in (("A - I", A[i] - I, Ao - I, ka), ("B", B[i], Bo, kb)):
            err = np.linalg.norm((K - O)[:, keep]) / max(1e-12, np.linalg.norm(O[:, keep]))
            worst[name] = max(worst.get(name, 0.0), err)
        rot = np.linalg.norm((A[i] - Ao)[3:6][:, ka]) / np.linalg.norm(Ao[3:6][:, ka])
        worst["rot rows"] = max(worst.get("rot rows", 0.0), rot)
    print({k: f"{x:.2e}" for k, x in worst.items()})
    # worst seen on the emulator: A - I 1.3e-3, B 5.4e-5, rotation rows 1.7e-6
    assert worst["A - I"] <= 1e-2 and worst["B"] <= 1e-3 and worst["rot rows"] <= 1e-4


def test_column_equals_forward_difference(backend):
    """Hinge-qvel and ctrl columns: the kernel's column is (forward(x+) - forward(x-)) / (x+ - x-) bit for bit, forward warm-started from
    the nominal qacc."""
    cfg, om, q, v, u = _states("smpl_humanoid", 4, seed=17, nair=1)
    m = om.model
    nv = m.nv
    env = backend.batch(cfg, 32)
    tq, tv, tu = backend.t(q), backend.t(v), backend.t(u)
    fd = env.transition_fd(tq, tv, tu, dqacc=True)
    cols = [nv + 6, nv + 20, 2 * nv - 1, 2 * nv, 2 * nv + 31, 2 * nv + m.nu - 1]
    for col in cols:
        tp, tm = [tv.clone(), tu.clone()], [tv.clone(), tu.clone()]
        k, e = (0, col - nv) if col < 2 * nv else (1, col - 2 * nv)
        eps = EPS[1] if k == 0 else EPS[2]
        tp[k][:, e] += eps; tm[k][:, e] -= eps
        ap = env.forward(tq, tp[0], tp[1], qacc_warmstart=fd["qacc"])["qacc"]
        am = env.forward(tq, tm[0], tm[1], qacc_warmstart=fd["qacc"])["qacc"]
        want = (ap - am) / (tp[k][:, e] - tm[k][:, e])[:, None]
        assert torch.equal(fd["dqacc"][:, :, col], want), col


def test_contact_free_structure(backend):
    """No constraint rows: d qacc / d ctrl = M^-1[:, 6:].  With contacts, eps_ctrl = 1 and 10 agree on unflagged columns (qacc is
    affine in ctrl for a fixed active set)."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    nv = m.nv
    q, v = airborne_states(m, 3, seed=19)
    q[:, 7:] *= 0.2
    q, v = np.float32(q), np.float32(v)
    u = np.float32(np.random.default_rng(3).uniform(-30, 30, (3, m.nu)))
    env = backend.batch(cfg, 64)
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), dqacc=True)
    M = env.dynamics(backend.t(q), backend.t(v))["qM"].cpu().numpy().astype(np.float64)
    K = fd["dqacc"].cpu().numpy()
    for i in range(3):
        assert _forward(om, q[i], v[i]).nefc == 0
        assert relerr(K[i][:, 2 * nv:], np.linalg.inv(M[i])[:, 6:]) <= 1e-3, i
    _, _, qc, vc, uc = _states("smpl_humanoid", 4, seed=23, nair=0)
    f1 = env.transition_fd(backend.t(qc), backend.t(vc), backend.t(uc), eps_ctrl=1.0, dqacc=True)
    f10 = env.transition_fd(backend.t(qc), backend.t(vc), backend.t(uc), eps_ctrl=10.0, dqacc=True)
    keep = ((f1["flags"] == 0) & (f10["flags"] == 0)).cpu().numpy()[:, 2 * nv:]
    a, b = f1["dqacc"].cpu().numpy()[:, :, 2 * nv:], f10["dqacc"].cpu().numpy()[:, :, 2 * nv:]
    assert keep.mean() >= 0.5          # eps_ctrl = 10 N m switches contact rows in some columns (0.85 kept on the emulator)
    for i in range(4):
        assert relerr(a[i][:, keep[i]], b[i][:, keep[i]]) <= 1e-3, i


def test_forward_differences(backend):
    """centered = 0 runs the + passes only and stays near the centered result on columns the centered run does not flag."""
    cfg, om, q, v, u = _states("smpl_humanoid", 3, seed=29, nair=1)
    m = om.model
    env = backend.batch(cfg, 64)
    c = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), dqacc=True)
    f = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), centered=False, dqacc=True)
    assert torch.equal(c["qacc"], f["qacc"])
    assert not bool((f["flags"] & 1).any())
    keep = (c["flags"] == 0).cpu().numpy()
    for i in range(len(q)):
        _, blk = dqacc_errors(m, f["dqacc"][i].cpu().numpy().astype(np.float64), c["dqacc"][i].cpu().numpy().astype(np.float64), keep[i])
        assert blk <= 0.5, (i, blk)   # O(eps) truncation: worst block 0.30 on the emulator (a state with floor contacts)


# ------------------------------------------------------------------ 9-10. launch shapes, no effect on the stepper
def _small_and_production(backend, cfg, monkeypatch):
    """A 32-env handle with 1-warp CTAs and a 4 096-env handle with the production 8-warp CTAs."""
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    small = backend.batch(cfg, 32)
    monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    big = backend.batch(cfg, 4096)
    wpb = lambda e: e._L().smplsim_warps_per_block(e._h)  # noqa: E731
    assert wpb(small) == 1 and wpb(big) == 8
    return small, big


def test_launch_shapes(backend, monkeypatch):
    """Forward on 37 rows (a ragged last CTA) and FD on 3 rows (chunked by 32 slots on the small handle, one launch on the large one):
    bit-identical; n = 0 returns empty outputs."""
    cfg, om, q, v, u = _states("smpl_humanoid", 37, seed=31, nair=4)
    small, big = _small_and_production(backend, cfg, monkeypatch)
    outs = [e.forward(backend.t(q), backend.t(v), backend.t(u), contact_wrench=True) for e in (small, big)]
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
    fds = [e.transition_fd(backend.t(q[:3]), backend.t(v[:3]), backend.t(u[:3]), dqacc=True) for e in (small, big)]
    for k in fds[0]:
        assert torch.equal(fds[0][k], fds[1][k]), k
    m = om.model
    z = [backend.t(np.zeros((0, w))) for w in (m.nq, m.nv, m.nu)]
    assert big.forward(*z)["qacc"].shape == (0, m.nv)
    f0 = big.transition_fd(*z, dqacc=True)
    assert f0["A"].shape == (0, 2 * m.nv, 2 * m.nv) and f0["dqacc"].shape == (0, m.nv, 2 * m.nv + m.nu)


def test_stepper_cannot_tell(backend):
    """step -> forward -> transition_fd -> step and step -> step from the same state: every output and state row bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_fd in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_fd and t == 0:        # every scratch row of the handle
                qq = env.qpos.repeat(3, 1)[: 2 * n + n // 2]
                vv = torch.as_tensor(rin.normal(size=(qq.shape[0], m.nv)), dtype=torch.float32, device=qq.device)
                uu = torch.as_tensor(rin.normal(size=(qq.shape[0], m.nu)) * 20, dtype=torch.float32, device=qq.device)
                env.forward(qq, vv, uu, contact_wrench=True)
                env.transition_fd(qq[:2], vv[:2], uu[:2], dqacc=True)
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------ 11. arguments
def test_arguments(backend, tmp_path):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    L, h, s = env._L(), env._h, env._stream()
    q, v = airborne_states(m, 4, seed=1)
    tq, tv, tu = backend.t(q), backend.t(v), backend.t(np.zeros((4, m.nu)))
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    qa = backend.t(np.zeros((4, m.nv)))
    A = backend.t(np.zeros((4, 2 * m.nv, 2 * m.nv)))
    good = SmplsimFdCfgC(1e-3, 1e-2, 1.0, 1, 0)

    def err(rc, code, text):
        assert rc == code, (rc, code)
        assert L.smplsim_last_error().decode() == text

    err(L.smplsim_forward(None, p(tq), p(tv), p(tu), None, 4, p(qa), None, None, None, None, s), -1, "smplsim_forward: null handle or n < 0")
    err(L.smplsim_forward(h, p(tq), p(tv), p(tu), None, -1, p(qa), None, None, None, None, s), -1, "smplsim_forward: null handle or n < 0")
    err(L.smplsim_forward(h, p(tq), p(tv), None, None, 4, p(qa), None, None, None, None, s), -1, "smplsim_forward: null argument")
    err(L.smplsim_forward(h, p(tq), p(tv), p(tu), None, 4, None, None, None, None, None, s), -1, "smplsim_forward: null argument")
    assert L.smplsim_forward(h, None, None, None, None, 0, None, None, None, None, None, s) == 0

    fd = lambda hh, cfg_, n, qacc, A_: L.smplsim_transition_fd(hh, cfg_, p(tq), p(tv), p(tu), n, qacc, None, A_, None, None, s)  # noqa: E731
    err(fd(None, C.byref(good), 4, p(qa), p(A)), -1, "smplsim_transition_fd: null handle / cfg or n < 0")
    err(fd(h, None, 4, p(qa), p(A)), -1, "smplsim_transition_fd: null handle / cfg or n < 0")
    err(fd(h, C.byref(good), -1, p(qa), p(A)), -1, "smplsim_transition_fd: null handle / cfg or n < 0")
    err(fd(h, C.byref(good), 4, None, p(A)), -1, "smplsim_transition_fd: null argument (qpos, qvel, ctrl and qacc are required)")
    err(fd(h, C.byref(good), 4, p(qa), None), -1, "smplsim_transition_fd: no derivative output requested (dqacc, A, B and flags all NULL)")
    for bad in ((0.0, 1e-2, 1.0), (1e-3, -1.0, 1.0), (1e-3, 1e-2, float("nan")), (float("inf"), 1e-2, 1.0)):
        err(fd(h, C.byref(SmplsimFdCfgC(*bad, 1, 0)), 4, p(qa), p(A)), -1,
            "smplsim_transition_fd: eps_qpos, eps_qvel and eps_ctrl must be finite and > 0")
    with pytest.raises(ValueError, match="eps_qvel"):
        env.transition_fd(tq, tv, tu, eps_qvel=0.0)
    with pytest.raises(ValueError, match="shape"):
        env.forward(tq, tv, tu[:, :-1])

    env.set_env_params(friction=backend.t(np.full(4, 0.8)))
    err(fd(h, C.byref(good), 4, p(qa), p(A)), -3,
        "smplsim_transition_fd: not available while the handle has per-env parameter records (smplsim_clear_env_params)")
    err(L.smplsim_forward(h, p(tq), p(tv), p(tu), None, 2, p(qa), None, None, None, None, s), -1,
        "smplsim_forward: with per-env parameters n must be the handle's num_envs (row i uses env i's parameters)")

    from smplsim_b200.abi import model_from_cfg
    shapes = backend.batch(cfg, 4, models=[model_from_cfg(cfg)] * 2, env_model=np.array([0, 1, 0, 1], dtype=np.int32))
    err(L.smplsim_transition_fd(shapes._h, C.byref(good), p(tq), p(tv), p(tu), 4, p(qa), None, p(A), None, None, s), -3,
        "smplsim_transition_fd: not available with per-env body shapes (the column slots of a row span CTAs of any shape)")

    scfg, _ = make_models(env="getup", control_mode="torque", self_collision=True)
    senv = backend.batch(scfg, 4)
    text = "the forward pass on caller rows does not build geom-geom contacts (handle created with self_collision = 1)"
    err(L.smplsim_forward(senv._h, p(tq), p(tv), p(tu), None, 4, p(qa), None, None, None, None, s), -3, "smplsim_forward: " + text)
    err(L.smplsim_transition_fd(senv._h, C.byref(good), p(tq), p(tv), p(tu), 4, p(qa), None, p(A), None, None, s), -3,
        "smplsim_transition_fd: " + text)


# ------------------------------------------------------------------ 12. single env
def test_single_env_mjd_transitionFD(backend):
    from smplsim_b200.envs import HumanoidSpeed, mjd_transitionFD
    cfg, om = make_models(env="speed", control_mode="torque")
    if backend.name == "gpu":
        env = HumanoidSpeed(cfg, device="cuda:0")
    else:
        backend.batch(cfg, 1)   # puts tests/emu on the path
        import emu_env

        class EmuSpeed(HumanoidSpeed):
            def _make_batch(self, cfg, device):
                return emu_env.EmuBatch(cfg, 1, seed=int(cfg.get("seed", 0)))
        env = EmuSpeed(cfg, device="cpu")
    env.reset()
    env.step(np.zeros(env.get_action_size(), dtype=np.float32))
    m = om.model
    d = env.mj_data
    A, B = np.zeros((2 * m.nv, 2 * m.nv)), np.zeros((2 * m.nv, m.nu))
    mjd_transitionFD(env.mj_model, d, 1e-3, True, A, B, None, None)
    b = env._b
    row = lambda x: torch.as_tensor(np.float32(x)[None], device=b.device)  # noqa: E731
    want = b.transition_fd(row(d.qpos), row(d.qvel), row(d.ctrl), 1e-3, 1e-3, 1e-3)
    assert np.array_equal(A, want["A"][0].cpu().numpy().astype(np.float64))
    assert np.array_equal(B, want["B"][0].cpu().numpy().astype(np.float64))
    with pytest.raises(NotImplementedError, match="C, D"):
        mjd_transitionFD(env.mj_model, d, 1e-3, True, A, B, np.zeros((1, 1)), None)
