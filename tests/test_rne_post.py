"""Body accelerations, joint reaction wrenches and IMU readings (smplsim_rne_post, k_rnep5, HumanoidBatchB200.rne_post, the single-env
mj_rnePostConstraint and MotionLibB200.rne_post) against fp64 references, on the host emulator and on the H100 (-m gpu).

References (no new oracle code), all in fp64 at the fp32 inputs the kernel reads:
- body_acc: a central difference in time of ref_jac(q(t)) v(t), q(t) = q (+) t qvel (the exponential map on the root rotation),
  v(t) = qvel + t qacc, t = +-1e-4, with the oracle's kinematics at q(t) -- independent of the kernel's recursion;
- joint_wrench: a numpy Newton-Euler inward sum over the oracle's poses: per body m (a_com - g) and I wd + w x I w from the model's
  masses and inertias, minus test_contact_wrench.ref_wrench of test_inverse.ref_inverse's row forces, minus xfrc_applied;
- IMU sites: from those two references, at random site offsets and orientations.

Tolerances: the worst case of test_rne_post_matches_references and of the fallen rows of test_airborne_planted_fallen (TOL,
TOL_JW), and of test_identities (TOL_ID), measured on the emulator / on an H100 80GB HBM3 (700 W), with a margin of at least 20x.
Each error is relative to its row's scale (body_acc and accelerometer to max(|g|, max|ref|), gyro to max(1, max|ref|),
joint_wrench / force / torque to max(m |g|, max|ref|)):
- TOL_JW 6e-4 on joint_wrench: 2.5e-5 / 3.0e-5;
- TOL 2e-4 on the other outputs: body_acc 2.7e-6 / 2.7e-6, accelerometer 2.3e-6 / 1.9e-6, gyro 5.8e-7 / 4.8e-7, force 3.9e-6 /
  2.9e-6, torque 1.2e-6 / 8.6e-7;
- TOL_ID 2e-5 on the identities against inverse() (relative to max(m |g|, max |qfrc_inverse|) or, for Newton-Euler, max(m |g|,
  max |joint_wrench|)): hinge and root projections 3.3e-7 / 3.6e-7, Newton-Euler 2.7e-7 / 6.0e-7.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from oracle import oracle as orc  # noqa: E402
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from test_contact_wrench import ref_wrench  # noqa: E402
from test_cta_shapes import N_DYN, N_SMPLX, _bit_equal, _one_warp_chunks, _production, _tiled  # noqa: E402
from test_dynamics import _ancestors, _qmat, _qmul, ref_jac  # noqa: E402
from test_env_params import draw, oracle_for  # noqa: E402
from test_gpu_parity import _shape_variant  # noqa: E402
from test_inverse import _near_switch, _over_cap, ref_inverse  # noqa: E402
from util_states import airborne_states, make_models, rollout_states  # noqa: E402

TOL = 2e-4
TOL_JW = 6e-4
TOL_ID = 2e-5
H_FD = 1e-4
BODY = ("body_acc", "joint_wrench")
SITE = ("accelerometer", "gyro", "force", "torque")
KEYS = BODY + SITE


def _np(d):
    return {k: x.cpu().numpy().copy() for k, x in d.items()}


def _oracle(om, q, v):
    """Oracle forward pass at fp64 (q, v) as given (the callers round to fp32 first where the kernel reads the same state)."""
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v
    e.forward()
    return e


def _f64(x):
    return np.float32(x).astype(np.float64)


def _shift(q, v, t):
    """q (+) t v: root position + t v[0:3], root quaternion (x) exp(t v[3:6]) (body frame), hinges + t v[6:]."""
    out = q.copy()
    out[0:3] += t * v[0:3]
    w = t * v[3:6]
    a = np.linalg.norm(w)
    dq = np.r_[1.0, 0.0, 0.0, 0.0] if a == 0 else np.r_[np.cos(a / 2), np.sin(a / 2) * w / a]
    out[3:7] = _qmul(q[3:7], dq)
    out[7:] += t * v[6:]
    return out


def random_sites(m, k, seed):
    """k sites on random bodies, offsets up to 0.2 m, random orientations (wxyz)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(k):
        qs = rng.normal(size=4)
        out.append((int(rng.integers(0, m.nbody)), rng.uniform(-0.2, 0.2, 3).astype(np.float32), (qs / np.linalg.norm(qs)).astype(np.float32)))
    return out


# ------------------------------------------------------------------ fp64 references
def ref_row(om, q, v, a, xf=None, sites=()):
    """References of one row (fp32 inputs, evaluated in fp64) plus the pieces the identities use."""
    m = om.model
    q, v, a = _f64(q), _f64(v), _f64(a)
    q[3:7] /= np.linalg.norm(q[3:7])
    nb = m.nbody
    g = np.asarray(m.gravity, dtype=np.float64)
    e = _oracle(om, q, v)
    xpos, xquat = e.xpos.copy(), e.xquat.copy()
    J = ref_jac(m, q, xpos, xquat)
    vel = J @ v
    js = []
    for t in (H_FD, -H_FD):
        qt = _shift(q, v, t)
        et = _oracle(om, qt, v)
        js.append(ref_jac(m, qt, et.xpos.copy(), et.xquat.copy()) @ (v + t * a))
    acc = (js[0] - js[1]) / (2 * H_FD)
    qfrc, f, _ = ref_inverse(e, a)
    con = e.contacts()
    nc = len(con["geom"])
    nlim = e.nefc - 4 * nc
    cw = ref_wrench(m, con, f[nlim:].reshape(nc, 4), xpos, xquat)
    lim = e.efc()["J"][:nlim].T @ f[:nlim] if nlim else np.zeros(m.nv)
    xf = np.zeros((nb, 6)) if xf is None else np.asarray(xf, dtype=np.float64)
    mass = np.asarray(m.body_mass, dtype=np.float64)
    Rs = [_qmat(xquat[b]) for b in range(nb)]
    r = np.array([Rs[b] @ np.asarray(m.body_ipos[b], dtype=np.float64) for b in range(nb)])
    xipos = xpos + r
    w, wd = vel[:, 3:], acc[:, 3:]
    fo, to = np.zeros((nb, 3)), np.zeros((nb, 3))   # own wrench: force, torque about the world origin
    for b in range(nb):
        xx, yy, zz, xy, xz, yz = np.asarray(m.body_inertia[b], dtype=np.float64)
        Ic = Rs[b] @ np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]]) @ Rs[b].T
        acom = acc[b, :3] + np.cross(wd[b], r[b]) + np.cross(w[b], np.cross(w[b], r[b]))
        fb = mass[b] * (acom - g) - cw[b, :3] - xf[b, :3]
        tb = Ic @ wd[b] + np.cross(w[b], Ic @ w[b]) - cw[b, 3:] - xf[b, 3:]
        fo[b], to[b] = fb, tb + np.cross(xipos[b], fb)
    jw = np.zeros((nb, 6))
    for b in range(nb):
        sub = [c for c in range(nb) if b in _ancestors(m, c)]
        F, T = fo[sub].sum(0), to[sub].sum(0)
        jw[b] = np.r_[F, T - np.cross(xpos[b], F)]
    out = {"body_acc": acc, "joint_wrench": jw}
    if len(sites):
        s_out = {k: [] for k in SITE}
        for b, p, qs in sites:
            Rsite = Rs[b] @ _qmat(np.asarray(qs, dtype=np.float64))
            d = Rs[b] @ np.asarray(p, dtype=np.float64)
            asite = acc[b, :3] + np.cross(wd[b], d) + np.cross(w[b], np.cross(w[b], d))
            Fb, Tb = jw[b, :3], jw[b, 3:]
            s_out["accelerometer"].append(Rsite.T @ (asite - g))
            s_out["gyro"].append(Rsite.T @ w[b])
            s_out["force"].append(Rsite.T @ Fb)
            s_out["torque"].append(Rsite.T @ (Tb - np.cross(d, Fb)))
        out.update({k: np.array(x) for k, x in s_out.items()})
    extra = dict(e=e, J=J, vel=vel, qfrc=qfrc, lim=lim, cw=cw, xpos=xpos, xquat=xquat, skip=_over_cap(e) or _near_switch(e, a))
    return out, extra


def _scales(m, ref):
    gn = float(np.linalg.norm(m.gravity))
    wt = float(np.sum(m.body_mass)) * gn
    return {"body_acc": max(gn, np.abs(ref["body_acc"]).max()), "accelerometer": max(gn, np.abs(ref.get("accelerometer", 0)).max()),
            "gyro": max(1.0, np.abs(ref.get("gyro", 0)).max()),
            **{k: max(wt, np.abs(ref["joint_wrench"]).max(), np.abs(ref.get(k, 0)).max()) for k in ("joint_wrench", "force", "torque")}}


def _errors(om, q, v, a, out, sites=(), xf=None, worst=None):
    """Worst relative errors of kernel rows `out` (numpy) against ref_row, per output; rows near a row-set switch or past the
    joint-limit row cap are skipped.  Returns (worst, rows checked)."""
    worst = dict.fromkeys([k for k in KEYS if k in out], 0.0) if worst is None else worst
    checked = 0
    for i in range(len(q)):
        ref, ex = ref_row(om, q[i], v[i], a[i], None if xf is None else xf[i], sites)
        if ex["skip"]:
            continue
        checked += 1
        sc = _scales(om.model, ref)
        for k in worst:
            worst[k] = max(worst[k], float(np.abs(out[k][i] - ref[k]).max() / sc[k]))
    return worst, checked


def _assert_within(worst, tag):
    for k, x in worst.items():
        assert x <= (TOL_JW if k == "joint_wrench" else TOL), (tag, k, x)


def _states(robot, n, seed, qacc_scale=5.0):
    """Airborne and stable-PD rollout states (standing, stumbling, lying) with random qacc."""
    _, om = make_models(robot=robot, control_mode="uhc_pd")
    na = max(2, n // 3)
    qa, va = airborne_states(om.model, na, seed=seed)
    qc, vc, _ = rollout_states(om, n - na, seed=seed + 1)
    q, v = np.concatenate([qa, qc]), np.concatenate([va, vc])
    a = np.random.default_rng(seed + 2).normal(size=v.shape) * qacc_scale
    return q, v, a


# ------------------------------------------------------------------ 1. the references hold the definitions (CPU, oracle only)
def test_references_match_oracle():
    """The FD body accelerations at qacc = 0, qvel = 0 vanish and match J qacc in the qvel = 0 case; the Newton-Euler joint wrench
    of the root equals the oracle inverse's root rows plus armature, and each hinge's projection its qfrc_inverse entry, to 2e-5 (the
    O(t^2) truncation of the central difference: 6.6e-6 at most)."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v, a = _states("smpl_humanoid", 5, seed=3)
    arm = np.asarray(m.dof_armature, dtype=np.float64)
    for i in range(len(q)):
        ref, ex = ref_row(om, q[i], np.zeros(m.nv), a[i])
        assert np.abs(ref["body_acc"] - ex["J"] @ _f64(a[i])).max() < 1e-6 * max(1.0, np.abs(ref["body_acc"]).max()), i
        ref, ex = ref_row(om, q[i], v[i], a[i])
        _check_identities(m, ref["joint_wrench"], ex, ex["qfrc"], _f64(a[i]), arm, 2e-5, i)


def _check_identities(m, jw, ex, qfrc, a, arm, tol, tag):
    """Root: force = qfrc[0:3] - arm a, torque about the root origin on c_k = qfrc[3 + k] - arm a; hinge d of body b: axis_d . torque_b
    = qfrc_d - arm_d a_d + the limit force on d.  Returns the worst error relative to max(m |g|, max|qfrc|)."""
    sc = max(float(np.sum(m.body_mass)) * float(np.linalg.norm(m.gravity)), float(np.abs(qfrc).max()))
    R0 = _qmat(ex["xquat"][0])
    err = np.abs(jw[0, :3] - (qfrc[0:3] - arm[0:3] * a[0:3])).max()
    err = max(err, np.abs(R0.T @ jw[0, 3:] - (qfrc[3:6] - arm[3:6] * a[3:6])).max())
    for d in range(6, m.nv):
        b = (d - 6) // 3 + 1
        err = max(err, abs(ex["J"][b, 3:, d] @ jw[b, 3:] - (qfrc[d] - arm[d] * a[d] + ex["lim"][d])))
    assert err <= tol * sc, (tag, err / sc)
    return err / sc


# ------------------------------------------------------------------ 2. kernel against the references, identities
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_rne_post_matches_references(backend, robot):
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    n = 12 if robot == "smpl_humanoid" else 6
    q, v, a = _states(robot, n, seed=11)
    sites = random_sites(m, 7, seed=12)
    xf = np.random.default_rng(13).normal(size=(n, m.nbody, 6)) * 20.0
    xf[: n // 2] = 0.0
    env = backend.batch(cfg, 8)
    t = backend.t
    out = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites, xfrc_applied=t(xf)))
    worst, checked = _errors(om, q, v, a, out, sites, _f64(xf))
    print(robot, checked, {k: f"{x:.1e}" for k, x in worst.items()})
    assert checked >= n - 2
    _assert_within(worst, robot)


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_identities(backend, robot):
    """Against inverse() on the same rows: the root and hinge projections of joint_wrench (with the oracle's limit forces), and
    Newton-Euler per body with inverse(contact_wrench=True): F_b - sum_children F_c + contact_b = I_b a_b + v x* I_b v - m_b g."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    n = 10 if robot == "smpl_humanoid" else 5
    q, v, a = _states(robot, n, seed=21)
    env = backend.batch(cfg, 8)
    t = backend.t
    out = _np(env.rne_post(t(q), t(v), t(a)))
    qfrc, cw = (x.cpu().numpy().astype(np.float64) for x in env.inverse(t(q), t(v), t(a), contact_wrench=True))
    arm = np.asarray(m.dof_armature, dtype=np.float64)
    worst, ne = 0.0, 0.0
    for i in range(n):
        ref, ex = ref_row(om, q[i], v[i], a[i])
        if ex["skip"]:
            continue
        jw = out["joint_wrench"][i].astype(np.float64)
        worst = max(worst, _check_identities(m, jw, ex, qfrc[i], _f64(a[i]), arm, TOL_ID, (robot, i)))
        # Newton-Euler per body with the kernel's accelerations and contact wrenches
        xpos, xquat = ex["xpos"], ex["xquat"]
        acc = out["body_acc"][i].astype(np.float64)
        g = np.asarray(m.gravity, dtype=np.float64)
        sc = max(float(np.sum(m.body_mass)) * float(np.linalg.norm(g)), float(np.abs(jw).max()))
        for b in range(m.nbody):
            R = _qmat(xquat[b])
            r = R @ np.asarray(m.body_ipos[b], dtype=np.float64)
            xx, yy, zz, xy, xz, yz = np.asarray(m.body_inertia[b], dtype=np.float64)
            Ic = R @ np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]]) @ R.T
            w, wd = ex["vel"][b, 3:], acc[b, 3:]
            acom = acc[b, :3] + np.cross(wd, r) + np.cross(w, np.cross(w, r))
            F, T = jw[b, :3].copy(), jw[b, 3:] - np.cross(r, jw[b, :3])   # torque about xipos
            for c in range(b + 1, m.nbody):
                if int(m.body_parent[c]) == b:
                    F -= jw[c, :3]
                    T -= jw[c, 3:] + np.cross(xpos[c] - xpos[b] - r, jw[c, :3])
            F += cw[i, b, :3]; T += cw[i, b, 3:]
            e_f = np.abs(F - float(m.body_mass[b]) * (acom - g)).max()
            e_t = np.abs(T - (Ic @ wd + np.cross(w, Ic @ w))).max()
            ne = max(ne, max(e_f, e_t) / sc)
    print(robot, f"identities {worst:.1e}, Newton-Euler {ne:.1e}")
    assert ne <= TOL_ID, ne


# ------------------------------------------------------------------ 3. physical cases
def test_airborne_planted_fallen(backend):
    """Airborne at forward()'s qacc: joint_wrench[0] ~ 0 on every row, every accelerometer ~ 0 from rest with ctrl = 0 and no rows.
    Planted static poses (qvel = qacc = 0): every accelerometer reads R_s^T (-g), and joint_wrench[0] plus the contact forces carry the
    weight.  Fallen (lying) rows against the references."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    t = backend.t
    env = backend.batch(cfg, 8)
    g = np.asarray(m.gravity, dtype=np.float64)
    wt = float(np.sum(m.body_mass)) * float(np.linalg.norm(g))
    qa, va = airborne_states(m, 6, seed=31)
    ctrl = np.random.default_rng(32).uniform(-30, 30, (6, m.nu))
    va[3:], ctrl[3:] = 0.0, 0.0
    fw = env.forward(t(qa), t(va), t(ctrl))
    out = _np(env.rne_post(t(qa), t(va), fw["qacc"], imu_sites="bodies"))
    assert np.abs(out["joint_wrench"][:, 0]).max() <= TOL * wt, np.abs(out["joint_wrench"][:, 0]).max() / wt
    free = [i for i in range(3, 6) if _oracle(om, _f64(qa[i]), np.zeros(m.nv)).nefc == 0]
    assert free, "no airborne row without joint-limit rows"
    assert np.abs(out["accelerometer"][free]).max() <= TOL * np.linalg.norm(g), np.abs(out["accelerometer"][free]).max()
    # planted: rollout states at rest
    qc, _, _ = rollout_states(make_models(control_mode="uhc_pd")[1], 6, seed=33)
    z = np.zeros((len(qc), m.nv))
    out = _np(env.rne_post(t(qc), t(z), t(z), imu_sites="bodies"))
    _, cw = env.inverse(t(qc), t(z), t(z), contact_wrench=True)
    cw = cw.cpu().numpy().astype(np.float64)
    xq = env.kinematics(t(qc))[1].cpu().numpy().astype(np.float64)
    for i in range(len(qc)):
        want = np.array([_qmat(xq[i, b]).T @ (-g) for b in range(m.nbody)])
        assert np.abs(out["accelerometer"][i] - want).max() <= TOL * np.linalg.norm(g), i
        carried = out["joint_wrench"][i, 0, :3] + cw[i, :, :3].sum(0)
        assert np.abs(carried - (-wt / np.linalg.norm(g)) * g).max() <= TOL * wt, (i, carried)
    # fallen: lying rows of the rollout pool at random qvel / qacc
    qf, vf, _ = rollout_states(make_models(control_mode="uhc_pd")[1], 8, seed=34, init_mode=1)
    af = np.random.default_rng(35).normal(size=vf.shape) * 3.0
    sites = random_sites(m, 5, seed=36)
    out = _np(env.rne_post(t(qf), t(vf), t(af), imu_sites=sites))
    worst, checked = _errors(om, qf, vf, af, out, sites)
    print(f"fallen {checked}", {k: f"{x:.1e}" for k, x in worst.items()})
    assert checked >= len(qf) - 2
    _assert_within(worst, "fallen")


# ------------------------------------------------------------------ 4. launch paths and edges
def _run_all(env, t, q, v, a, sites):
    return _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites))


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_production_shapes_and_chunks(backend, monkeypatch, robot):
    """8-warp SMPL with num_envs rows plus a ragged second launch, 4-warp SMPL-X with a ragged last CTA: bit-identical with 1-warp
    CTAs; each output requested alone (through the C ABI for the sites) is bit-identical with the all-outputs call; n == 0 reads
    nothing."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    t = backend.t
    if robot == "smpl_humanoid":
        nenv, extra = N_DYN[backend.name]
        n, wpb, ragged = nenv + extra, 8, False
    else:
        nenv = n = N_SMPLX[backend.name]
        wpb, ragged = 4, True
    q, v, _, kinds, _, idx = _tiled(robot, n)
    keep = np.array([k != "bad" for k in kinds])
    idx = np.array([j if keep[j] else int(np.flatnonzero(keep)[0]) for j in idx])
    q, v = q[idx], v[idx]
    a = np.random.default_rng(41).normal(size=v.shape) * 5.0
    sites = random_sites(m, 9, seed=42)
    env = _production(backend, monkeypatch, cfg, nenv, wpb, ragged=ragged)
    if robot == "smpl_humanoid":
        assert n > env.num_envs
    got = _run_all(env, t, q, v, a, sites)
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), lambda e, s: _run_all(e, t, q[s], v[s], a[s], sites))
    _bit_equal(got, ref, "production vs 1-warp CTAs")
    for k, kw in (("body_acc", dict(acc=True, joint_wrench=False)), ("joint_wrench", dict(acc=False, joint_wrench=True))):
        o = _np(env.rne_post(t(q), t(v), t(a), **kw))
        assert list(o) == [k]
        _bit_equal(o, {k: got[k]}, k + " alone")
    L = env._L()
    tq, tv, ta = t(q), t(v), t(a)
    sb, sp, sq = env._imu_sites(sites)
    hp = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    for j, k in enumerate(SITE):
        o = torch.empty(n, len(sites), 3, dtype=torch.float32, device=tq.device)
        outs = [None] * 4
        outs[j] = C.c_void_p(o.data_ptr())
        assert L.smplsim_rne_post(env._h, C.c_void_p(tq.data_ptr()), C.c_void_p(tv.data_ptr()), C.c_void_p(ta.data_ptr()), None, n, None,
                                  None, hp(sb), hp(sp), hp(sq), len(sites), *outs, env._stream()) == 0
        _bit_equal({k: o.cpu().numpy()}, {k: got[k]}, k + " alone")
    e0 = env.rne_post(t(q[:0]), t(v[:0]), t(a[:0]), imu_sites=sites)
    assert set(e0) == set(KEYS) and all(x.shape[0] == 0 for x in e0.values())
    assert L.smplsim_rne_post(env._h, None, None, None, None, 0, None, None, None, None, None, 0, None, None, None, None, env._stream()) == 0


# ------------------------------------------------------------------ 5. handle kinds and options
def test_per_env_shapes(backend, tmp_path):
    """Three body shapes interleaved: row i against the references of env i's shape; n must be num_envs."""
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]
    cfgs, oms = [], []
    for p in paths:
        cfg, om = make_models(control_mode="torque", **({} if p is None else {"robot.xml_path": str(p)}))
        cfgs.append(cfg); oms.append(om)
    models = [model_from_cfg(c) for c in cfgs]
    n = 9
    env_model = np.array([i % 3 for i in range(n)], dtype=np.int32)
    q, v, a = _states("smpl_humanoid", n, seed=51)
    sites = random_sites(oms[0].model, 4, seed=52)
    env = backend.batch(cfgs[0], n, models=models, env_model=env_model)
    t = backend.t
    out = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites))
    for i in range(n):
        row = {k: x[i:i + 1] for k, x in out.items()}
        w, _ = _errors(oms[env_model[i]], q[i:i + 1], v[i:i + 1], a[i:i + 1], row, sites)
        _assert_within(w, ("shape", i))
    with pytest.raises(Exception, match="num_envs"):
        env.rne_post(t(q[:3]), t(v[:3]), t(a[:3]))


def test_parameter_records(backend):
    """Gravity and body mass scales per env: rows against each env's variant model; a gravity change moves the accelerometer and
    mass scales move joint_wrench; n must be num_envs."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    n = 6
    P = draw(m, n, seed=61)
    t = backend.t
    q, v, a = _states("smpl_humanoid", n, seed=62)
    sites = random_sites(m, 4, seed=63)
    plain = _np(backend.batch(cfg, n).rne_post(t(q), t(v), t(a), imu_sites=sites))
    env = backend.batch(cfg, n)
    env.set_env_params(None, **{k: t(x) for k, x in P.items()})
    out = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites))
    for i in range(n):
        ov = oracle_for(cfg, m, P, i)
        row = {k: x[i:i + 1] for k, x in out.items()}
        w, _ = _errors(ov, q[i:i + 1], v[i:i + 1], a[i:i + 1], row, sites)
        _assert_within(w, ("records", i))
        assert np.abs(out["accelerometer"][i] - plain["accelerometer"][i]).max() > 1e-3, i
        assert np.abs(out["joint_wrench"][i] - plain["joint_wrench"][i]).max() > 1e-2, i
    assert np.array_equal(out["body_acc"], plain["body_acc"])
    with pytest.raises(Exception, match="num_envs"):
        env.rne_post(t(q[:2]), t(v[:2]), t(a[:2]))


def test_xfrc_applied(backend):
    """xfrc_applied set moves joint_wrench and the site forces by exactly its subtree sums (within rounding); all-zero xfrc_applied is
    bit-identical with none; body_acc and the kinematic site outputs never see it."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    t = backend.t
    q, v, a = _states("smpl_humanoid", 6, seed=71)
    sites = random_sites(m, 5, seed=72)
    env = backend.batch(cfg, 8)
    none = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites))
    zero = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites, xfrc_applied=t(np.zeros((6, m.nbody, 6)))))
    _bit_equal(zero, none, "zero xfrc vs none")
    xf = np.random.default_rng(73).normal(size=(6, m.nbody, 6)) * 30.0
    got = _np(env.rne_post(t(q), t(v), t(a), imu_sites=sites, xfrc_applied=t(xf)))
    for k in ("body_acc", "accelerometer", "gyro"):
        assert np.array_equal(got[k], none[k]), k
    wt = float(np.sum(m.body_mass)) * 9.81
    d = got["joint_wrench"][:, 0, :3].astype(np.float64) - none["joint_wrench"][:, 0, :3]
    assert np.abs(d + _f64(xf)[:, :, :3].sum(1)).max() <= TOL * max(wt, np.abs(xf).sum(1).max()), np.abs(d + xf[:, :, :3].sum(1)).max()


# ------------------------------------------------------------------ 6. argument errors
def test_errors(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    t = backend.t
    q, v, a = (x[:2] for x in _states("smpl_humanoid", 3, seed=81))
    tq, tv, ta = t(q), t(v), t(a)
    L, h, s = env._L(), env._h, env._stream()
    p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    hp = lambda x: C.c_void_p(x.ctypes.data)  # noqa: E731
    o6 = torch.empty(2, m.nbody, 6, dtype=torch.float32, device=tq.device)
    o3 = torch.empty(2, 64, 3, dtype=torch.float32, device=tq.device)
    EINVAL, EUNSUP = -1, -3

    def sites(k, body=0, quat=(1.0, 0.0, 0.0, 0.0)):
        sb = np.full(k, body, dtype=np.int32)
        sp = np.zeros((k, 3), dtype=np.float32)
        sq = np.tile(np.asarray(quat, dtype=np.float32), (k, 1))
        return hp(sb), hp(sp), hp(sq), (sb, sp, sq)

    def call(qp, qv, qa, n, acc, jw, site, ns, accel, gyro=None, force=None, torque=None):
        return L.smplsim_rne_post(h, qp, qv, qa, None, n, acc, jw, *site[:3], ns, accel, gyro, force, torque, s)

    ok = sites(2)
    none = (None, None, None)
    assert call(p(tq), p(tv), p(ta), 2, p(o6), None, none, 0, None) == 0
    assert call(p(tq), p(tv), p(ta), 2, None, None, ok, 2, p(o3)) == 0
    for args in ((None, p(tv), p(ta)), (p(tq), None, p(ta)), (p(tq), p(tv), None)):
        assert call(*args, 2, p(o6), None, none, 0, None) == EINVAL
        assert "null qpos, qvel or qacc" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), -1, p(o6), None, none, 0, None) == EINVAL
    assert call(p(tq), p(tv), p(ta), 2, None, None, none, 0, None) == EINVAL
    assert "no output" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(1, body=m.nbody), 1, p(o3)) == EINVAL
    assert "out of range" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(1, body=-1), 1, p(o3)) == EINVAL
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(65), 65, p(o3)) == EINVAL
    assert "nsite > 64" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, p(o6), None, ok, 2, None) == EINVAL
    assert "needs a site output" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, p(o6), None, none, 0, p(o3)) == EINVAL
    assert "needs nsite > 0" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(1, quat=(1.002, 0.0, 0.0, 0.0)), 1, p(o3)) == EINVAL
    assert "unit quaternion" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(1, quat=(1.0005, 0.0, 0.0, 0.0)), 1, p(o3)) == 0
    assert call(p(tq), p(tv), p(ta), 2, None, None, sites(1, quat=(float("nan"), 0.0, 0.0, 0.0)), 1, p(o3)) == EINVAL
    assert call(p(tq), p(tv), p(ta), 2, None, None, none, 1, p(o3)) == EINVAL
    assert L.smplsim_rne_post(None, p(tq), p(tv), p(ta), None, 2, p(o6), None, None, None, None, 0, None, None, None, None, s) == EINVAL
    cfg_s, _ = make_models(control_mode="torque", self_collision=True)
    es = backend.batch(cfg_s, 4)
    assert es._L().smplsim_rne_post(es._h, p(tq), p(tv), p(ta), None, 2, p(o6), None, None, None, None, 0, None, None, None, None,
                                    es._stream()) == EUNSUP
    with pytest.raises(Exception, match="self_collision"):
        es.rne_post(tq, tv, ta)
    # Python checks
    with pytest.raises(ValueError, match="qacc must have shape"):
        env.rne_post(tq, tv, ta[:, :5])
    with pytest.raises(ValueError, match="float32"):
        env.rne_post(tq, tv, ta.double())
    with pytest.raises(ValueError, match="xfrc_applied must have shape"):
        env.rne_post(tq, tv, ta, xfrc_applied=t(np.zeros((3, m.nbody, 6))))
    with pytest.raises(ValueError, match="contiguous"):
        env.rne_post(tq, tv, ta, xfrc_applied=t(np.zeros((2, 6, m.nbody))).transpose(1, 2))
    with pytest.raises(ValueError, match="unknown body name"):
        env.rne_post(tq, tv, ta, imu_sites=[("nope", (0, 0, 0), (1, 0, 0, 0))])
    with pytest.raises(ValueError, match="imu_sites bodies"):
        env.rne_post(tq, tv, ta, imu_sites=[(m.nbody, (0, 0, 0), (1, 0, 0, 0))])
    with pytest.raises(ValueError, match="unit quaternion"):
        env.rne_post(tq, tv, ta, imu_sites=[(0, (0, 0, 0), (2, 0, 0, 0))])
    with pytest.raises(ValueError, match="pos"):
        env.rne_post(tq, tv, ta, imu_sites=[(0, (0, 0), (1, 0, 0, 0))])
    with pytest.raises(ValueError, match="at most 64"):
        env.rne_post(tq, tv, ta, imu_sites=[(0, (0, 0, 0), (1, 0, 0, 0))] * 65)
    with pytest.raises(ValueError, match="'bodies'"):
        env.rne_post(tq, tv, ta, imu_sites="all")
    assert env.rne_post(tq, tv, ta, acc=False, joint_wrench=False) == {}
    by_name = env.rne_post(tq, tv, ta, imu_sites=[(m.body_names[4], (0.1, 0, 0), (1, 0, 0, 0))])
    by_index = env.rne_post(tq, tv, ta, imu_sites=[(4, (0.1, 0, 0), (1, 0, 0, 0))])
    for k in KEYS:
        assert torch.equal(by_name[k], by_index[k]), k


# ------------------------------------------------------------------ 7. the stepper is untouched
def test_stepper_untouched(backend):
    """rne_post between steps leaves the next steps' obs / reward / flags / state bit-identical with a batch that never called it."""
    cfg, om = make_models(control_mode="uhc_pd")
    n = 6
    a, b = backend.batch(cfg, n, seed=3), backend.batch(cfg, n, seed=3)
    a.reset(); b.reset()
    rng = np.random.default_rng(91)
    for step in range(3):
        act = backend.t(rng.normal(size=(n, a.num_actions)) * 0.3)
        a.rne_post(a.qpos.clone(), a.qvel.clone(), a.qacc.clone(), imu_sites="bodies")
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra, rb):
            assert torch.equal(x.cpu(), y.cpu()), step
        for k in ("qpos", "qvel", "qacc_warm", "qpos_fwd", "qvel_fwd"):
            assert torch.equal(getattr(a, k).cpu(), getattr(b, k).cpu()), (step, k)


# ------------------------------------------------------------------ 8. single env and motion library
def test_single_env(backend):
    """mj_rnePostConstraint fills cacc / cfrc_int / cfrc_ext [nbody + 1, 6] from the batch outputs at the last forward pass: each
    row against the batch's body_acc / joint_wrench and inverse()'s contact wrench plus xfrc_applied, converted to MuJoCo's layout."""
    from smplsim_b200 import envs as E
    from smplsim_b200.cfg import make_cfg
    cfg = make_cfg(env="speed", seed=4)

    class Env(E.HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    env = Env(cfg, device=backend.device)
    env.reset()
    rng = np.random.default_rng(101)
    for _ in range(2):
        env.step(rng.normal(size=env.get_action_size()) * 0.3)
    env.mj_data.xfrc_applied[3] = (5.0, -2.0, 7.0, 0.5, 0.1, -0.3)
    d = env.mj_data
    assert E.mj_rnePostConstraint(env.mj_model, d) is None
    b = env._b
    m = b.model
    nb = m.nbody
    for k in ("cacc", "cfrc_int", "cfrc_ext"):
        assert getattr(d, k).shape == (nb + 1, 6) and getattr(d, k).dtype == np.float64, k
    g = _f64(m.gravity)   # the env's gravity as the kernels hold it
    assert np.array_equal(d.cacc[0], np.r_[0.0, 0.0, 0.0, -g]) and not d.cfrc_int[0].any() and not d.cfrc_ext[0].any()
    xf = torch.as_tensor(env._xfrc_applied[1:], dtype=torch.float32, device=b.device)[None].contiguous()
    out = _np(b.rne_post(b.qpos_fwd, b.qvel_fwd, b.qacc, xfrc_applied=xf))
    c = d.subtree_com[0]
    xpos = b.kinematics(b.qpos_fwd)[0][0].cpu().numpy().astype(np.float64)
    jw = out["joint_wrench"][0].astype(np.float64)
    assert np.allclose(d.cfrc_int[1:, 3:], jw[:, :3], rtol=0, atol=0)
    assert np.allclose(d.cfrc_int[1:, :3], jw[:, 3:] + np.cross(xpos - c, jw[:, :3]), rtol=1e-12, atol=1e-9)
    assert np.array_equal(d.cacc[1:, :3], out["body_acc"][0, :, 3:].astype(np.float64))
    # the com-based acceleration is the spatial acceleration at c: the classical acceleration of the body point at c less w x v_c,
    # i.e. cacc = [wd ; a_x + wd x (c - x) - w x v_x - g] with the body origin's acceleration a_x and velocity v_x
    jac = b.dynamics(b.qpos_fwd, None, mass_matrix=False, bias=False, jac_bodies=list(range(nb)))
    vel = torch.cat([jac["jacp"], jac["jacr"]], 2)[0].cpu().numpy().astype(np.float64) @ b.qvel_fwd[0].cpu().numpy().astype(np.float64)
    acc = out["body_acc"][0].astype(np.float64)
    lin = acc[:, :3] + np.cross(acc[:, 3:], c - xpos) - np.cross(vel[:, 3:], vel[:, :3]) - g
    assert np.allclose(d.cacc[1:, 3:], lin, rtol=1e-12, atol=1e-9)
    _, cw = b.inverse(b.qpos_fwd, b.qvel_fwd, b.qacc, contact_wrench=True)
    cw = cw[0].cpu().numpy().astype(np.float64)
    f_ext = cw[:, :3] + env._xfrc_applied[1:, :3]
    assert np.array_equal(d.cfrc_ext[1:, 3:], f_ext)
    assert np.abs(d.cfrc_ext[3, 3:] - cw[2, :3] - (5.0, -2.0, 7.0)).max() < 1e-12   # MuJoCo body 3 is robot body 2
    # Newton for the whole robot: the root joint's force plus the external forces equal sum_b m_b (a_com,b - g)
    mt = float(np.sum(m.body_mass))
    xq = b.kinematics(b.qpos_fwd)[1][0].cpu().numpy().astype(np.float64)
    mom = np.zeros(3)
    for k in range(nb):
        r = _qmat(xq[k]) @ np.asarray(m.body_ipos[k], dtype=np.float64)
        w, wd = vel[k, 3:], acc[k, 3:]
        mom += float(m.body_mass[k]) * (acc[k, :3] + np.cross(wd, r) + np.cross(w, np.cross(w, r)) - g)
    assert np.abs(d.cfrc_int[1, 3:] + d.cfrc_ext[1:, 3:].sum(0) - mom).max() <= TOL * mt * np.linalg.norm(g)


def test_motion_lib(backend):
    """MotionLibB200.rne_post() equals a direct call on the library's tables at inverse_dynamics()'s qacc, bit for bit, and
    inverse_dynamics() is the direct inverse at that qacc."""
    from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables
    cfg, om = make_models(control_mode="torque")
    env = backend.batch(cfg, 8)
    tab = synthetic_tables(env, num_clips=3, frames=7, fps=30.0, seed=2)
    ml = MotionLibB200(env, tab)
    qacc = ml._frame_qacc()
    got = ml.rne_post(imu_sites="bodies")
    want = env.rne_post(backend.t(tab["qpos"]), backend.t(tab["qvel"]), qacc, imu_sites="bodies")
    assert list(got) == list(want) and got["body_acc"].shape == (len(tab["qpos"]), om.model.nbody, 6)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(ml.inverse_dynamics(), env.inverse(backend.t(tab["qpos"]), backend.t(tab["qvel"]), qacc))
    # qacc: forward differences within each clip, none across clips
    qv = np.asarray(tab["qvel"])
    dt = 1.0 / 30.0
    qa = qacc.cpu().numpy()
    assert np.allclose(qa[0], (qv[1] - qv[0]) / dt, rtol=1e-5, atol=1e-4) and np.allclose(qa[6], qa[5])
