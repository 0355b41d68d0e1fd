"""Centre of mass and centroidal momentum (smplsim_centroidal, k_cent5, HumanoidBatchB200.centroidal, the single-env
mj_data.subtree_com / mj_subtreeVel / mj_jacSubtreeCom and MotionLibB200.centroidal) against fp64 references, on the host emulator
and on the H100 (-m gpu).

References (no new oracle code):
- cmm and cmm_bias from the oracle's M and qfrc_bias: every body descends from the root, so the root rows of M are the momentum
  matrix about the root origin (linear rows M[0:3], angular rows R_root M[3:6] without the root armature), and qfrc_bias[0:6] is the
  RNE's root wrench with gravity; both are shifted to the centre of mass (DESIGN.md 2);
- subtree quantities and jac_com from numpy over the oracle's xpos / xquat and the model's masses and inertias, its body velocities
  pinned to the oracle's body-origin velocity sensors and its whole-body centre of mass to the oracle's;
- Newton-Euler against forward(contact_wrench=True): cmm qacc + cmm_bias = [m g + sum F_b ; sum t_b + (xipos_b - c) x F_b].

Tolerances: the worst case of test_centroidal_matches_references and test_newton_euler, measured on the emulator / on an H100
80GB HBM3, with a margin of at least 20x (test_dynamics' rule):
- TOL_COM 1e-5 m on subtree_com: 3.1e-7 / 3.0e-7;
- TOL 3e-5 on the other outputs, each relative to its scale (subtree_linvel and jac_com to max(1, max|ref|); subtree_angmom and cmm to
  max(m, max|ref|); cmm_bias to max(m g, max|ref|)): subtree_linvel 1.1e-6 / 1.1e-6, subtree_angmom 3.0e-7 / 2.1e-7, cmm 5.5e-8 /
  5.2e-8, cmm_bias 6.0e-7 / 4.0e-7, jac_com 5.1e-7 / 4.9e-7;
- TOL_NE 3e-5 on Newton-Euler (relative to m |g| or the size of the summed terms, _newton_euler): 1.1e-6 / 1.5e-6.
"""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from test_cta_shapes import EPW, N_DYN, N_SMPLX, _bit_equal, _one_warp_chunks, _production, _tiled  # noqa: E402
from test_dynamics import _ancestors, _forward, _qmat, ref_jac  # noqa: E402
from test_env_params import draw, oracle_for, variant  # noqa: E402
from test_gpu_parity import _shape_variant  # noqa: E402
from util_states import airborne_states, make_models, rollout_states  # noqa: E402

TOL_COM = 1e-5
TOL = 3e-5
TOL_NE = 3e-5
KEYS = ("subtree_com", "subtree_linvel", "subtree_angmom", "cmm", "cmm_bias", "jac_com")


def _np(d):
    return {k: x.cpu().numpy().copy() for k, x in d.items()}


def _skew(c):
    return np.array([[0, -c[2], c[1]], [c[2], 0, -c[0]], [-c[1], c[0], 0]])


# ------------------------------------------------------------------ fp64 references
def ref_subtree(m, q, e):
    """(com, linvel, angmom [nb, 3], jac_com [nb, 3, nv], Jc [nb, 3, nv]) from the oracle env e after its forward pass at q."""
    nb = m.nbody
    xpos, xquat = e.xpos.copy(), e.xquat.copy()
    J = ref_jac(m, np.float32(q).astype(np.float64), xpos, xquat)
    mass = np.asarray(m.body_mass, dtype=np.float64)
    Rs = [_qmat(xquat[b]) for b in range(nb)]
    r = np.array([Rs[b] @ np.asarray(m.body_ipos[b], dtype=np.float64) for b in range(nb)])
    xipos = xpos + r
    Jc = np.array([J[b, :3] - _skew(r[b]) @ J[b, 3:] for b in range(nb)])   # velocity of xipos: v + w x r
    lin0, w = e.sensor[0].copy(), e.sensor[1].copy()
    vcom = lin0 + np.cross(w, r)
    Iw = []
    for b in range(nb):
        xx, yy, zz, xy, xz, yz = np.asarray(m.body_inertia[b], dtype=np.float64)
        Iw.append(Rs[b] @ np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]]) @ Rs[b].T)
    com, lv, am, jc = np.zeros((nb, 3)), np.zeros((nb, 3)), np.zeros((nb, 3)), np.zeros((nb, 3, m.nv))
    for b in range(nb):
        sub = [c for c in range(nb) if b in _ancestors(m, c)]
        M = mass[sub].sum()
        com[b] = (mass[sub, None] * xipos[sub]).sum(0) / M
        lv[b] = (mass[sub, None] * vcom[sub]).sum(0) / M
        am[b] = sum(Iw[c] @ w[c] + mass[c] * np.cross(xipos[c] - com[b], vcom[c] - lv[b]) for c in sub)
        jc[b] = sum(mass[c] * Jc[c] for c in sub) / M
    return com, lv, am, jc, Jc


def ref_cmm(m, e, gravity=None):
    """(cmm [6, nv], cmm_bias [6]) from the oracle's M and qfrc_bias (rows i < 6), shifted from the root origin to the centre of mass."""
    g = np.asarray(m.gravity if gravity is None else gravity, dtype=np.float64)
    mt = float(np.sum(m.body_mass))
    M = e.M.copy()
    M[np.arange(6), np.arange(6)] -= np.asarray(m.dof_armature[:6], dtype=np.float64)
    R0 = _qmat(e.xquat[0])
    d = e.sub_com.copy() - e.xpos[0]                  # c - x_root
    p, LO = M[0:3], R0 @ M[3:6]
    A = np.concatenate([p, LO - np.cross(d, p.T).T])
    F = e.qfrc_bias[0:3].copy() + mt * g
    T = R0 @ e.qfrc_bias[3:6] + mt * np.cross(d, g)
    return A, np.concatenate([F, T - np.cross(d, F)])


def _states(robot, n, seed):
    _, om = make_models(robot=robot, control_mode="uhc_pd")
    na = max(2, n // 3)
    qa, va = airborne_states(om.model, na, seed=seed)
    qc, vc, _ = rollout_states(om, n - na, seed=seed + 1)
    return np.concatenate([qa, qc]), np.concatenate([va, vc])


def _errors(m, q, v, out, om):
    """Worst errors of kernel rows `out` (numpy) against the references, per output."""
    mt = float(np.sum(m.body_mass))
    worst = dict.fromkeys(KEYS, 0.0)
    for i in range(len(q)):
        e = _forward(om, q[i], v[i])
        com, lv, am, jc, _ = ref_subtree(om.model, q[i], e)
        A, bias = ref_cmm(om.model, e)
        sc = max(1.0, mt)
        errs = {"subtree_com": np.abs(out["subtree_com"][i] - com).max(),
                "subtree_linvel": np.abs(out["subtree_linvel"][i] - lv).max() / max(1.0, np.abs(lv).max()),
                "subtree_angmom": np.abs(out["subtree_angmom"][i] - am).max() / max(sc, np.abs(am).max()),
                "cmm": np.abs(out["cmm"][i] - A).max() / max(sc, np.abs(A).max()),
                "cmm_bias": np.abs(out["cmm_bias"][i] - bias).max() / max(sc * 9.81, np.abs(bias).max()),
                "jac_com": np.abs(out["jac_com"][i] - jc[out["_jb"]]).max() / max(1.0, np.abs(jc).max())}
        for k, x in errs.items():
            worst[k] = max(worst[k], float(x))
    return worst


def _assert_within(worst, tag):
    for k, x in worst.items():
        assert x <= (TOL_COM if k == "subtree_com" else TOL), (tag, k, x)


# ------------------------------------------------------------------ 1. the references hold the definitions (CPU, oracle only)
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_references_match_oracle(robot):
    """The numpy COM velocities reproduce the body-origin sensors through Jc (so the body velocities are the oracle's), the whole-body
    COM is the oracle's, and the cmm / bias built from M and qfrc_bias equal the numpy momentum and its identities, to 1e-9."""
    _, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    q, v = _states(robot, 6, seed=3)
    for i in range(len(q)):
        e = _forward(om, q[i], v[i])
        com, lv, am, jc, Jc = ref_subtree(m, q[i], e)
        vv = e.qvel.copy()
        lin0 = e.sensor[0].copy()
        Rs = [_qmat(e.xquat[b]) for b in range(m.nbody)]
        vcom = lin0 + np.cross(e.sensor[1], np.array([Rs[b] @ m.body_ipos[b] for b in range(m.nbody)]))
        assert np.abs(Jc @ vv - vcom).max() < 1e-9 * max(1.0, np.abs(vcom).max()), i
        assert np.abs(com[0] - e.sub_com).max() < 1e-9, i
        assert np.abs(jc @ vv - lv).max() < 1e-9 * max(1.0, np.abs(lv).max()), i
        A, _ = ref_cmm(m, e)
        mt = float(np.sum(m.body_mass))
        h = A @ vv
        assert np.abs(h - np.concatenate([mt * lv[0], am[0]])).max() < 1e-9 * max(1.0, np.abs(h).max()), i
        assert np.abs(A[0:3] - mt * jc[0]).max() < 1e-9 * mt, i


# ------------------------------------------------------------------ 2. kernel against the references, identities
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_centroidal_matches_references(backend, robot):
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    n = 12 if robot == "smpl_humanoid" else 6
    q, v = _states(robot, n, seed=11)
    env = backend.batch(cfg, 8)
    jb = list(range(m.nbody))
    out = _np(env.centroidal(backend.t(q), backend.t(v), jac_com_bodies=jb))
    out["_jb"] = np.array(jb)
    worst = _errors(m, q, v, out, om)
    print(robot, {k: f"{x:.1e}" for k, x in worst.items()})
    _assert_within(worst, robot)
    mt = float(np.sum(m.body_mass))
    for i in range(n):   # identities on the kernel's own outputs
        vv = np.float32(v[i]).astype(np.float64)
        lv0, am0 = out["subtree_linvel"][i, 0].astype(np.float64), out["subtree_angmom"][i, 0].astype(np.float64)
        assert np.abs(out["jac_com"][i, 0] @ vv - lv0).max() <= TOL * max(1.0, np.abs(lv0).max()), i
        assert np.abs(out["cmm"][i, 0:3] - mt * out["jac_com"][i, 0]).max() <= TOL * mt, i
        h = out["cmm"][i].astype(np.float64) @ vv
        ref = np.concatenate([mt * lv0, am0])
        assert np.abs(h - ref).max() <= TOL * max(mt, np.abs(ref).max()), i


def _newton_euler(env, backend, m, q, v, ctrl, gravity, masses):
    """Worst |cmm qacc + cmm_bias - [m g + sum F ; sum t + (xipos - c) x F]| over the rows, relative to m |g| or, where larger, to the
    size of the terms summed (sum |cmm| |qacc| + |cmm_bias|: rows past their joint limits reach |qacc| ~ 1e7, and fp32 holds the sum
    to its terms' rounding, not to m g).  Rows whose forward pass flags a bad state (status bits 1 / 2 / 4: unspecified qacc) are
    skipped; returns (worst, rows checked)."""
    t = backend.t
    fw = env.forward(t(q), t(v), t(ctrl), contact_wrench=True)
    c = _np(env.centroidal(t(q), t(v), com=True, velocity=True, cmm=True))
    xpos, xquat = (x.cpu().numpy().astype(np.float64) for x in env.kinematics(t(q)))
    qacc, cw = fw["qacc"].cpu().numpy().astype(np.float64), fw["contact_wrench"].cpu().numpy().astype(np.float64)
    worst, checked = 0.0, 0
    st = fw["status"].cpu().numpy()
    for i in range(len(q)):
        if st[i] & 7:
            continue
        checked += 1
        g = np.asarray(gravity[i], dtype=np.float64)
        mt = float(np.sum(masses[i]))
        hd = c["cmm"][i].astype(np.float64) @ qacc[i] + c["cmm_bias"][i]
        xipos = np.array([xpos[i, b] + _qmat(xquat[i, b]) @ m.body_ipos[b] for b in range(m.nbody)])
        com = c["subtree_com"][i, 0].astype(np.float64)
        F, T = cw[i, :, :3], cw[i, :, 3:]
        ref = np.concatenate([mt * g + F.sum(0), (T + np.cross(xipos - com, F)).sum(0)])
        scale = max(mt * np.linalg.norm(g), float((np.abs(c["cmm"][i]) @ np.abs(qacc[i]) + np.abs(c["cmm_bias"][i])).max()))
        worst = max(worst, float(np.abs(hd - ref).max() / scale))
    return worst, checked


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_newton_euler(backend, robot):
    """The momentum rate the kernel gives at forward()'s qacc is the net external wrench: gravity alone on airborne rows, gravity
    plus the floor's contact wrenches on planted and fallen rows."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    qa, va = airborne_states(m, 4, seed=5)
    qc, vc, _ = rollout_states(om, 12 if robot == "smpl_humanoid" else 6, seed=6)
    q, v = np.concatenate([qa, qc]), np.concatenate([va, vc])
    ctrl = np.random.default_rng(7).uniform(-30, 30, (len(q), m.nu))
    env = backend.batch(cfg, 8)
    grav = np.broadcast_to(np.asarray(m.gravity, dtype=np.float64), (len(q), 3))
    masses = np.broadcast_to(np.asarray(m.body_mass, dtype=np.float64), (len(q), m.nbody))
    air, na = _newton_euler(env, backend, m, qa, va, ctrl[:4], grav[:4], masses[:4])
    worst, nall = _newton_euler(env, backend, m, q, v, ctrl, grav, masses)
    assert na == 4 and nall >= len(q) - 2, (na, nall)
    print(robot, f"airborne {air:.1e}, all {worst:.1e}")
    assert max(air, worst) <= TOL_NE, (air, worst)


# ------------------------------------------------------------------ 3. launch paths and edges
def _run_all(env, t, q, v, jb):
    return _np(env.centroidal(t(q), t(v), jac_com_bodies=jb))


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_production_shapes_and_chunks(backend, monkeypatch, robot):
    """8-warp SMPL with num_envs rows plus a ragged second launch, 4-warp SMPL-X with a ragged last CTA: bit-identical with 1-warp CTAs;
    each output requested alone is bit-identical with the all-outputs call; n == 0 reads nothing."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    t = backend.t
    jb = [0, 3, m.nbody - 1, 3]
    if robot == "smpl_humanoid":
        nenv, extra = N_DYN[backend.name]
        n, wpb, ragged = nenv + extra, 8, False
    else:
        nenv = n = N_SMPLX[backend.name]
        wpb, ragged = 4, True
    q, v, _, kinds, _, idx = _tiled(robot, n)
    keep = np.array([k != "bad" for k in kinds])
    v = np.where(keep[:, None], v, 0.0)
    q, v = q[idx], v[idx]
    env = _production(backend, monkeypatch, cfg, nenv, wpb, ragged=ragged)
    if robot == "smpl_humanoid":
        assert n > env.num_envs and extra % (8 * EPW) != 0
    got = _run_all(env, t, q, v, jb)
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), lambda e, s: _run_all(e, t, q[s], v[s], jb))
    _bit_equal(got, ref, "production vs 1-warp CTAs")
    alone = {"subtree_com": dict(com=True, velocity=False, cmm=False), "cmm": dict(com=False, velocity=False, cmm=True)}
    for k, kw in alone.items():
        o = _np(env.centroidal(t(q), None, **kw))
        assert list(o) == [k]
        _bit_equal(o, {k: got[k]}, k + " alone")
    o = _np(env.centroidal(t(q), t(v), com=False, velocity=True, cmm=False))
    _bit_equal(o, {k: got[k] for k in ("subtree_linvel", "subtree_angmom")}, "velocity alone")
    o = _np(env.centroidal(t(q), None, com=False, velocity=False, cmm=False, jac_com_bodies=jb))
    _bit_equal(o, {"jac_com": got["jac_com"]}, "jac_com alone")
    # cmm_bias alone through the C ABI
    L = env._L()
    tq, tv = t(q), t(v)
    cb = torch.empty(n, 6, dtype=torch.float32, device=tq.device)
    assert L.smplsim_centroidal(env._h, C.c_void_p(tq.data_ptr()), C.c_void_p(tv.data_ptr()), n, None, None, None, None,
                                C.c_void_p(cb.data_ptr()), None, 0, None, env._stream()) == 0
    _bit_equal({"cmm_bias": cb.cpu().numpy()}, {"cmm_bias": got["cmm_bias"]}, "cmm_bias alone")
    e0 = env.centroidal(t(q[:0]), t(v[:0]), jac_com_bodies=jb)
    assert all(x.shape[0] == 0 for x in e0.values())
    assert L.smplsim_centroidal(env._h, None, None, 0, None, None, None, None, None, None, 0, None, env._stream()) == 0


# ------------------------------------------------------------------ 4. handle kinds
def test_per_env_shapes(backend, tmp_path):
    """Three body shapes interleaved: row i against the references of env i's shape."""
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]
    cfgs, oms = [], []
    for p in paths:
        cfg, om = make_models(control_mode="torque", **({} if p is None else {"robot.xml_path": str(p)}))
        cfgs.append(cfg); oms.append(om)
    models = [model_from_cfg(c) for c in cfgs]
    n = 9
    env_model = np.array([i % 3 for i in range(n)], dtype=np.int32)
    q, v = _states("smpl_humanoid", n, seed=21)
    env = backend.batch(cfgs[0], n, models=models, env_model=env_model)
    jb = [0, 5]
    out = _np(env.centroidal(backend.t(q), backend.t(v), jac_com_bodies=jb))
    out["_jb"] = np.array(jb)
    for i in range(n):
        row = {k: x[i:i + 1] for k, x in out.items() if k != "_jb"}
        row["_jb"] = out["_jb"]
        w = _errors(oms[env_model[i]].model, q[i:i + 1], v[i:i + 1], row, oms[env_model[i]])
        _assert_within(w, ("shape", i))
    with pytest.raises(Exception, match="num_envs"):
        env.centroidal(backend.t(q[:3]), backend.t(v[:3]))


def test_parameter_records(backend):
    """body_mass_scale moves the centre of mass: rows against the references of each env's variant model; Newton-Euler with the
    env's gravity and masses; n must be num_envs."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    n = 6
    P = draw(m, n, seed=31)
    env = backend.batch(cfg, n)
    env.set_env_params(None, **{k: backend.t(x) for k, x in P.items()})
    q, v = _states("smpl_humanoid", n, seed=32)
    jb = [0, 2]
    out = _np(env.centroidal(backend.t(q), backend.t(v), jac_com_bodies=jb))
    for i in range(n):
        vm = variant(m, P, i)
        ov = oracle_for(cfg, m, P, i)
        row = {k: x[i:i + 1] for k, x in out.items()}
        row["_jb"] = np.array(jb)
        w = _errors(vm, q[i:i + 1], v[i:i + 1], row, ov)
        _assert_within(w, ("records", i))
    masses = np.array([np.asarray(variant(m, P, i).body_mass, dtype=np.float64) for i in range(n)])
    ctrl = np.random.default_rng(33).uniform(-30, 30, (n, m.nu))
    ne, checked = _newton_euler(env, backend, m, q, v, ctrl, P["gravity"].astype(np.float64), masses)
    print(f"records: Newton-Euler {ne:.1e}")
    assert ne <= TOL_NE and checked >= n - 1, (ne, checked)
    with pytest.raises(Exception, match="num_envs"):
        env.centroidal(backend.t(q[:2]), backend.t(v[:2]))


def test_self_collision_handle(backend):
    """A self-collision handle runs the same outputs (nothing here depends on contacts): bit-identical with a plain handle."""
    cfg, om = make_models(control_mode="torque")
    cfg_s, _ = make_models(control_mode="torque", self_collision=True)
    q, v = _states("smpl_humanoid", 5, seed=41)
    t = backend.t
    a = _np(backend.batch(cfg, 8).centroidal(t(q), t(v), jac_com_bodies=[0, 7]))
    b = _np(backend.batch(cfg_s, 8).centroidal(t(q), t(v), jac_com_bodies=[0, 7]))
    _bit_equal(b, a, "self-collision vs plain handle")


# ------------------------------------------------------------------ 5. argument errors
def test_errors(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    t = backend.t
    q, v = (x[:2] for x in _states("smpl_humanoid", 3, seed=51))
    tq, tv = t(q), t(v)
    L, h, s = env._L(), env._h, env._stream()
    p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731
    out3 = torch.empty(2, m.nbody, 3, dtype=torch.float32, device=tq.device)
    cm = torch.empty(2, 6, m.nv, dtype=torch.float32, device=tq.device)
    jac = torch.empty(2, m.nbody + 1, 3, m.nv, dtype=torch.float32, device=tq.device)
    EINVAL = -1

    def call(*a):
        return L.smplsim_centroidal(h, *a, s)

    jb = (C.c_int32 * (m.nbody + 1))(*([0] * (m.nbody + 1)))
    bad = (C.c_int32 * 1)(m.nbody)
    neg = (C.c_int32 * 1)(-1)
    assert call(p(tq), p(tv), 2, None, None, None, None, None, bad, 1, p(jac)) == EINVAL
    assert "out of range" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), 2, None, None, None, None, None, neg, 1, p(jac)) == EINVAL
    assert call(p(tq), p(tv), 2, None, None, None, None, None, jb, m.nbody + 1, p(jac)) == EINVAL
    assert "njac > nbody" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), 2, None, None, None, None, None, jb, 1, None) == EINVAL
    assert "jac_com_dev" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), 2, None, None, None, None, None, None, 1, p(jac)) == EINVAL
    for k in range(3):   # velocity outputs without qvel
        a = [None] * 5
        a[1 + k if k < 2 else 4] = p(cm) if k == 2 else p(out3)
        assert call(p(tq), None, 2, *a, None, 0, None) == EINVAL
        assert "need qvel" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), 2, None, None, None, None, None, None, 0, None) == EINVAL
    assert "no output" in L.smplsim_last_error().decode()
    assert call(None, p(tv), 2, p(out3), None, None, None, None, None, 0, None) == EINVAL
    assert "null qpos" in L.smplsim_last_error().decode()
    assert call(p(tq), p(tv), -1, p(out3), None, None, None, None, None, 0, None) == EINVAL
    assert L.smplsim_centroidal(None, p(tq), p(tv), 2, p(out3), None, None, None, None, None, 0, None, s) == EINVAL
    assert call(p(tq), p(tv), 2, p(out3), None, None, None, None, None, 0, None) == 0
    # Python checks
    with pytest.raises(ValueError, match="needs qvel"):
        env.centroidal(tq)
    with pytest.raises(ValueError, match="jac_com_bodies"):
        env.centroidal(tq, tv, jac_com_bodies=[m.nbody])
    with pytest.raises(ValueError, match="unknown body name"):
        env.centroidal(tq, tv, jac_com_bodies=["nope"])
    with pytest.raises(ValueError, match="qvel must have shape"):
        env.centroidal(tq, tv[:, :5])
    with pytest.raises(ValueError, match="float32"):
        env.centroidal(tq.double(), tv)
    assert env.centroidal(tq, None, velocity=False)["subtree_com"].shape == (2, m.nbody, 3)
    by_name = env.centroidal(tq, tv, jac_com_bodies=[m.body_names[4]])["jac_com"]
    assert torch.equal(by_name, env.centroidal(tq, tv, jac_com_bodies=[4])["jac_com"])


# ------------------------------------------------------------------ 6. the stepper is untouched
def test_stepper_untouched(backend):
    """centroidal between steps leaves the next steps' obs / reward / flags / state bit-identical with a batch that never called it."""
    cfg, om = make_models(control_mode="uhc_pd")
    n = 6
    a, b = backend.batch(cfg, n, seed=3), backend.batch(cfg, n, seed=3)
    a.reset(); b.reset()
    rng = np.random.default_rng(61)
    for step in range(3):
        act = backend.t(rng.normal(size=(n, a.num_actions)) * 0.3)
        a.centroidal(a.qpos.clone(), a.qvel.clone(), jac_com_bodies=[0, 1])
        ra, rb = a.step(act), b.step(act)
        for x, y in zip(ra, rb):
            assert torch.equal(x.cpu(), y.cpu()), step
        for k in ("qpos", "qvel", "qacc_warm", "qpos_fwd", "qvel_fwd"):
            assert torch.equal(getattr(a, k).cpu(), getattr(b, k).cpu()), (step, k)


# ------------------------------------------------------------------ 7. single env and motion library
def test_single_env(backend):
    from smplsim_b200 import envs as E
    from smplsim_b200.cfg import make_cfg
    cfg = make_cfg(env="speed", seed=4)

    class Env(E.HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    env = Env(cfg, device=backend.device)
    env.reset()
    rng = np.random.default_rng(71)
    for _ in range(2):
        env.step(rng.normal(size=env.get_action_size()) * 0.3)
    b = env._b
    ref = _np(b.centroidal(b.qpos_fwd, b.qvel_fwd, jac_com_bodies=[0, 4]))
    d = env.mj_data
    sc = d.subtree_com
    nb = b.model.nbody
    assert sc.shape == (nb + 1, 3) and sc.dtype == np.float64
    assert np.array_equal(sc[1:], ref["subtree_com"][0]) and np.array_equal(sc[0], ref["subtree_com"][0, 0])
    model = env.mj_model
    assert E.mj_subtreeVel(model, d) is None
    assert np.array_equal(d.subtree_linvel[1:], ref["subtree_linvel"][0]) and np.array_equal(d.subtree_linvel[0], ref["subtree_linvel"][0, 0])
    assert np.array_equal(d.subtree_angmom[1:], ref["subtree_angmom"][0]) and np.array_equal(d.subtree_angmom[0], ref["subtree_angmom"][0, 0])
    nv = b.model.nv
    jacp = np.full((3, nv), 7.0)
    assert E.mj_jacSubtreeCom(model, d, jacp, 5) is None
    assert np.array_equal(jacp, ref["jac_com"][0, 1])
    flat = np.zeros(3 * nv)
    E.mj_jacSubtreeCom(model, d, flat, 0)
    assert np.array_equal(flat.reshape(3, nv), ref["jac_com"][0, 0])
    with pytest.raises(ValueError):
        E.mj_jacSubtreeCom(model, d, jacp, nb + 1)


def test_motion_lib(backend):
    """MotionLibB200.centroidal() equals a direct call on the library's qpos / qvel tables, bit for bit."""
    from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables
    cfg, om = make_models(control_mode="torque")
    env = backend.batch(cfg, 8)
    tab = synthetic_tables(env, num_clips=3, frames=7, fps=30.0, seed=2)
    ml = MotionLibB200(env, tab)
    got = ml.centroidal(jac_com_bodies=[0, 3])
    want = env.centroidal(backend.t(tab["qpos"]), backend.t(tab["qvel"]), jac_com_bodies=[0, 3])
    assert list(got) == list(want) and got["subtree_com"].shape == (len(tab["qpos"]), om.model.nbody, 3)
    for k in want:
        assert torch.equal(got[k], want[k]), k
    only = ml.centroidal(velocity=False, cmm=False)
    assert list(only) == ["subtree_com"] and torch.equal(only["subtree_com"], want["subtree_com"])
