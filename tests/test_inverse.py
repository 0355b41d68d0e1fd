"""Inverse dynamics (smplsim_inverse, HumanoidBatchB200.inverse, MotionLibB200.inverse_dynamics) against a reference built from the
fp64 oracle.

The reference is test-side numpy on an oracle forward pass at the same fp32 (qpos, qvel): M qacc + qfrc_bias - J^T f with
f = -D min(0, J qacc - aref) over the pass's rows (joint-limit rows first, then four pyramid rows per floor contact).  The kernel
tests run on the H100 (-m gpu) and on the host emulator build of the same kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from smplsim_b200 import _lib
from test_contact_wrench import ref_wrench
from util_states import airborne_states, make_models, rollout_states
from xfrc_oracle import XfrcOracleEnv

# per-env max |kernel - reference| over the nv row, in units of the humanoid's weight m_total g, or of the row's largest reference
# component where that is larger (the contact-wrench test's bound).  Worst case seen in test_inverse_matches_reference: 3.7e-5 on the
# emulator and 4.1e-5 on an H100 (SMPL); TOL keeps a margin above 10x.
TOL = 2e-3
G = 9.81


def _weight(m):
    return float(np.sum(m.body_mass)) * G


def _forward(om, q, v, ctrl=None, w=None, xf=None):
    """Oracle forward pass at the fp32-rounded state (what the kernel reads)."""
    e = XfrcOracleEnv(om) if xf is not None else orc.OracleEnv(om)
    e.qpos[:] = np.float32(q); e.qvel[:] = np.float32(v)
    if w is not None:
        e.qacc_warm[:] = w
    if ctrl is not None:
        e.ctrl[:] = ctrl
    if xf is not None:
        e.xfrc_applied[:] = xf
    e.forward()
    return e


def ref_inverse(e, qacc):
    """(qfrc_inverse, row forces, row residuals) of the oracle env's last forward pass at acceleration qacc."""
    efc = e.efc()
    r = efc["J"] @ qacc - efc["aref"]
    f = -efc["D"] * np.minimum(0.0, r)
    return e.M @ qacc + e.qfrc_bias - efc["J"].T @ f, f, r


def _near_switch(e, qacc):
    """A contact in the |dist - margin| < 1e-5 band, or a row whose residual is within 1e-4 |aref| of zero: fp32 may set it either way."""
    con = e.contacts()
    if e.ncon and bool((np.abs(con["dist"] - e.m.margin) < 1e-5).any()):
        return True
    _, _, r = ref_inverse(e, qacc)
    return bool((np.abs(r) < 1e-4 * np.abs(e.efc()["aref"])).any())


def _states(robot, mode, n, seed):
    """A handle config with control mode `mode`; airborne states followed by stable-PD rollout states (standing, stumbling, lying)."""
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    na = max(2, n // 8)
    qa, va = airborne_states(m, na, seed=seed)
    qc, vc, wc = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], n - na, seed=seed + 1)
    return cfg, om, np.concatenate([qa, qc]), np.concatenate([va, vc]), np.concatenate([np.zeros((na, m.nv)), wc])


NLS = 16   # joint-limit rows the kernels hold per env (LCfg NLS); past it rows are dropped, as smplsim_step does (status bit 8)


def _over_cap(e):
    return e.nefc - 4 * e.ncon > NLS


# ------------------------------------------------------------------ 1. the reference holds the definition (CPU, oracle only)
@pytest.mark.parametrize("kind", ["rollout", "airborne", "xfrc"])
def test_reference_reproduces_ctrl(kind):
    """ref(e, e.qacc) at an oracle forward state is [0_6 ; ctrl] (+ qfrc_applied with a wrench) to the oracle's solver tolerance."""
    _, om = make_models(control_mode="torque")
    m = om.model
    if kind == "airborne":
        q, v = airborne_states(m, 8, seed=2)
        w = np.zeros_like(v)
    else:
        q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], 32, seed=5)
    rng = np.random.default_rng(1)
    nrows = 0
    for i in range(len(q)):
        ctrl = rng.uniform(-50, 50, m.nu)
        xf = None
        if kind == "xfrc":
            xf = np.concatenate([rng.uniform(-1, 1, (m.nbody, 3)) * G * np.asarray(m.body_mass)[:, None],
                                 rng.uniform(-1, 1, (m.nbody, 3)) * 5.0], axis=1)
        e = _forward(om, q[i], v[i], ctrl, w[i], xf)
        want = np.r_[np.zeros(6), ctrl] + (e.qfrc_applied if xf is not None else 0.0)
        scale = max(1.0, float(np.linalg.norm(want - e.qfrc_bias)))     # |qfrc_smooth|
        got, _, _ = ref_inverse(e, e.qacc.copy())
        assert np.abs(got - want).max() / scale < 1e-9, (i, np.abs(got - want).max(), scale)
        nrows += e.nefc > 0
    if kind != "airborne":
        assert nrows >= len(q) // 4


# ------------------------------------------------------------------ 2. kernel against the reference
@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_inverse_matches_reference(backend, robot, mode):
    """qacc = the oracle's forward qacc, that qacc plus noise (rows switch, non-zero root residual) and zero; contact wrench too."""
    n = 48 if robot == "smpl_humanoid" else 20
    cfg, om, q, v, w = _states(robot, mode, n, seed=11)
    m = om.model
    rng = np.random.default_rng(7)
    ctrl = rng.uniform(-50, 50, (n, m.nu))
    envs = [_forward(om, q[i], v[i], ctrl[i], w[i]) for i in range(n)]
    qf = np.array([e.qacc.copy() for e in envs])
    env = backend.batch(cfg, 16)
    wt = _weight(m)
    worst, flipped, root = 0.0, 0, 0.0
    for name, qacc in (("forward", qf), ("noise", qf + rng.normal(size=qf.shape) * 5.0), ("zero", np.zeros_like(qf))):
        out, cw = env.inverse(backend.t(q), backend.t(v), backend.t(qacc), contact_wrench=True)
        out = out.cpu().numpy().astype(np.float64); cw = cw.cpu().numpy().astype(np.float64)
        skipped = over = 0
        for i, e in enumerate(envs):
            a = np.float32(qacc[i]).astype(np.float64)
            if _over_cap(e):
                over += 1
                continue
            if _near_switch(e, a):
                skipped += 1
                continue
            ref, f, r = ref_inverse(e, a)
            err = np.abs(out[i] - ref).max() / max(wt, float(np.abs(ref).max()))
            assert err <= TOL, (name, i, err, e.ncon, e.nefc)
            worst = max(worst, err)
            nc = e.ncon
            W = ref_wrench(m, e.contacts(), f[e.nefc - 4 * nc:].reshape(nc, 4), e.xpos.copy(), e.xquat.copy())
            werr = np.abs(cw[i] - W).max() / max(wt, float(np.abs(W).max()))
            assert werr <= TOL, (name, i, werr)
            if nc == 0:
                assert np.all(cw[i] == 0.0)
            if name == "noise":
                _, f0, _ = ref_inverse(e, qf[i])
                flipped += int(((f > 0) != (f0 > 0)).sum())
                root = max(root, float(np.abs(ref[:6]).max()) / wt)
        assert skipped <= n // 10 and over <= n // 5, (name, skipped, over)
    print(f"{n} states ({over} past the limit-row cap), worst {worst:.2e}, {flipped} rows switched by the noise, largest root residual {root:.2f} m g")
    assert flipped > 0 and root > 0.1


# ------------------------------------------------------------------ 3. analytic checks
def test_static_and_free_fall(backend):
    """Airborne at rest with qacc = 0: qfrc_inverse = qfrc_bias (gravity only), root force (0, 0, m g).  Free fall (ctrl = 0, the
    oracle's contact-free qacc): qfrc_inverse = 0."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    wt = _weight(m)
    q, v = airborne_states(m, 8, seed=3)
    q[:, 7:] *= 0.2                                                    # inside the joint ranges: no rows at all
    env = backend.batch(cfg, 8)
    z = np.zeros_like(v)
    out = env.inverse(backend.t(q), backend.t(z), backend.t(z)).cpu().numpy().astype(np.float64)
    for i in range(len(q)):
        e = _forward(om, q[i], z[i])
        assert e.nefc == 0
        assert np.abs(out[i] - e.qfrc_bias).max() / wt < 1e-4, i
        assert np.abs(out[i, :3] - [0.0, 0.0, wt]).max() / wt < 1e-5, out[i, :3]
    envs = [_forward(om, q[i], v[i], np.zeros(m.nu)) for i in range(len(q))]
    qacc = np.array([e.qacc.copy() for e in envs])
    out = env.inverse(backend.t(q), backend.t(v), backend.t(qacc)).cpu().numpy().astype(np.float64)
    scale = [max(wt, float(np.abs(e.qfrc_bias).max())) for e in envs]
    assert max(np.abs(out[i]).max() / scale[i] for i in range(len(q))) < TOL


# ------------------------------------------------------------------ 4. forward / inverse round trip on the kernel
@pytest.mark.parametrize("with_xfrc", [False, True])
def test_round_trip_with_mj_step(backend, with_xfrc):
    """mj_step(ctrl, 1), then inverse at the pre-step state with aux.qacc: [0_6 ; ctrl] (+ the wrench's qfrc_applied)."""
    cfg, om, q, v, w = _states("smpl_humanoid", "uhc_pd", 32, seed=21)
    m = om.model
    n = len(q)
    rng = np.random.default_rng(5)
    ctrl = rng.uniform(-50, 50, (n, m.nu))
    xf = None
    if with_xfrc:
        xf = np.concatenate([rng.uniform(-1, 1, (n, m.nbody, 3)) * G * np.asarray(m.body_mass)[None, :, None],
                             rng.uniform(-1, 1, (n, m.nbody, 3)) * 5.0], axis=2)
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    if xf is not None:
        env.xfrc_applied = backend.t(xf)
    env.mj_step(backend.t(ctrl), 1)
    st = env.status.cpu().numpy()
    out = env.inverse(backend.t(q), backend.t(v), env.qacc.clone()).cpu().numpy().astype(np.float64)
    wt = _weight(m)
    ncmp = 0
    for i in range(n):
        if st[i] & (1 | 2 | 4 | 8 | 16):
            continue
        want = np.r_[np.zeros(6), ctrl[i]]
        if xf is not None:
            want = want + _forward(om, q[i], v[i], ctrl[i], w[i], xf[i]).qfrc_applied
        err = np.abs(out[i] - want).max() / max(wt, float(np.abs(want).max()))
        assert err <= TOL, (i, err)
        ncmp += 1
    assert ncmp >= n - n // 10


# ------------------------------------------------------------------ 5. batching, shapes, arguments
def test_chunking_and_empty_batch(backend):
    """n = 2.5 num_envs equals three separate calls bit for bit; n = 0 is a no-op."""
    cfg, om, q, v, w = _states("smpl_humanoid", "uhc_pd", 20, seed=31)
    qacc = np.random.default_rng(2).normal(size=v.shape) * 3.0
    env = backend.batch(cfg, 8)
    out, cw = env.inverse(backend.t(q), backend.t(v), backend.t(qacc), contact_wrench=True)
    for s in (slice(0, 8), slice(8, 16), slice(16, 20)):
        o, c = env.inverse(backend.t(q[s]), backend.t(v[s]), backend.t(qacc[s]), contact_wrench=True)
        assert torch.equal(o, out[s]) and torch.equal(c, cw[s])
    e0 = backend.t(np.zeros((0, om.model.nq)))
    o, c = env.inverse(e0, backend.t(np.zeros((0, om.model.nv))), backend.t(np.zeros((0, om.model.nv))), contact_wrench=True)
    assert o.shape == (0, om.model.nv) and c.shape == (0, om.model.nbody, 6)


def test_per_env_shapes(backend, tmp_path):
    """Three body shapes interleaved: row i against its own shape's oracle; n != num_envs is refused."""
    from smplsim_b200.abi import model_from_cfg
    from test_gpu_parity import _shape_variant
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a", leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2),
             _shape_variant(tmp_path / "b", leg=0.9, arm=1.1, trunk=0.95, girth=0.9, density=0.9)]
    mk = [make_models(control_mode="torque", **({"robot.xml_path": p} if p else {})) for p in paths]
    n = 24
    env_model = np.array([i % 3 for i in range(n)], dtype=np.int32)
    states = [rollout_states(make_models(control_mode="uhc_pd", **({"robot.xml_path": p} if p else {}))[1], n, seed=17, every=7) for p in paths]
    q = np.stack([states[k][0][i] for i, k in enumerate(env_model)])
    v = np.stack([states[k][1][i] for i, k in enumerate(env_model)])
    qacc = np.random.default_rng(4).normal(size=v.shape) * 3.0
    env = backend.batch(mk[0][0], n, models=[model_from_cfg(c) for c, _ in mk], env_model=env_model)
    out = env.inverse(backend.t(q), backend.t(v), backend.t(qacc)).cpu().numpy().astype(np.float64)
    ncmp = 0
    for i, k in enumerate(env_model):
        om = mk[k][1]
        e = _forward(om, q[i], v[i])
        a = np.float32(qacc[i]).astype(np.float64)
        if _over_cap(e) or _near_switch(e, a):
            continue
        ref, _, _ = ref_inverse(e, a)
        assert np.abs(out[i] - ref).max() / max(_weight(om.model), float(np.abs(ref).max())) <= TOL, (i, k)
        ncmp += 1
    assert ncmp >= n - n // 10
    with pytest.raises(_lib.SmplsimError, match="num_envs"):
        env.inverse(backend.t(q[:8]), backend.t(v[:8]), backend.t(qacc[:8]))


def test_arguments_and_self_collision_refused(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    q, v = airborne_states(m, 4, seed=1)
    tq, tv = backend.t(q), backend.t(v)
    with pytest.raises(ValueError, match="shape"):
        env.inverse(tq[:, :-1], tv, tv)
    with pytest.raises(ValueError, match="shape"):
        env.inverse(tq, tv[:3], tv)
    with pytest.raises(ValueError, match="float32"):
        env.inverse(tq, tv.double(), tv)
    with pytest.raises(ValueError, match="live on"):
        env.inverse(tq, tv, tv.to("meta"))
    L, p = env._L(), lambda t: C.c_void_p(t.data_ptr())
    out = backend.t(np.zeros((4, m.nv)))
    assert L.smplsim_inverse(env._h, None, p(tv), p(tv), p(out), None, 4, env._stream()) == -1
    assert L.smplsim_inverse(env._h, p(tq), p(tv), p(tv), None, None, 4, env._stream()) == -1
    assert L.smplsim_inverse(env._h, p(tq), p(tv), p(tv), p(out), None, -1, env._stream()) == -1
    assert L.smplsim_inverse(None, p(tq), p(tv), p(tv), p(out), None, 4, env._stream()) == -1
    scfg, _ = make_models(env="getup", control_mode="torque", self_collision=True)
    senv = backend.batch(scfg, 4)
    assert L.smplsim_inverse(senv._h, p(tq), p(tv), p(tv), p(out), None, 4, senv._stream()) == -3
    with pytest.raises(_lib.SmplsimError, match="geom-geom"):
        senv.inverse(tq, tv, tv)


def test_nan_row_leaves_other_rows_alone(backend):
    cfg, om, q, v, w = _states("smpl_humanoid", "uhc_pd", 16, seed=41)
    qacc = np.random.default_rng(3).normal(size=v.shape)
    env = backend.batch(cfg, 8)
    ref, rcw = env.inverse(backend.t(q), backend.t(v), backend.t(qacc), contact_wrench=True)
    q2, v2, a2 = q.copy(), v.copy(), qacc.copy()
    a2[3, 10] = np.nan; q2[9, 4] = np.nan; v2[12, 0] = np.inf
    out, cw = env.inverse(backend.t(q2), backend.t(v2), backend.t(a2), contact_wrench=True)
    keep = [i for i in range(len(q)) if i not in (3, 9, 12)]
    assert torch.equal(out[keep], ref[keep]) and torch.equal(cw[keep], rcw[keep])


# ------------------------------------------------------------------ 6. no effect on the stepper
def test_inverse_leaves_the_stepper_alone(backend):
    """step -> inverse -> step and step -> step from the same state: every output and every state row bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_inverse in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_inverse and t == 0:     # every scratch row of the handle, rows that touch the floor and switch limits
                qq = env.qpos.repeat(3, 1)[: 2 * n + n // 2]
                qq[:, 7:] += torch.as_tensor(rin.normal(size=(qq.shape[0], m.nu)) * 0.5, dtype=torch.float32, device=qq.device)
                vv = torch.as_tensor(rin.normal(size=(qq.shape[0], m.nv)), dtype=torch.float32, device=qq.device)
                env.inverse(qq, vv, vv * 10.0, contact_wrench=True)
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------ 7. motion-library helper
def test_motion_lib_inverse_dynamics(backend):
    """inverse_dynamics() equals env.inverse on numpy-differenced qacc bit for bit, clip-boundary frames included."""
    from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables
    cfg, om = make_models(control_mode="torque")
    env = backend.batch(cfg, 8)
    tab = synthetic_tables(env, num_clips=3, frames=7, fps=30.0, seed=2)
    ml = MotionLibB200(env, tab)
    qfrc, cw = ml.inverse_dynamics(contact_wrench=True)
    qv, dt = tab["qvel"], tab["motion_dt"]
    qacc = np.zeros_like(qv)
    for k, (s, nf) in enumerate(zip(tab["length_starts"], tab["motion_num_frames"])):
        d = (qv[s + 1:s + nf] - qv[s:s + nf - 1]) / dt[k]
        qacc[s:s + nf - 1] = d
        qacc[s + nf - 1] = d[-1]
    want, wcw = env.inverse(backend.t(tab["qpos"]), backend.t(qv), backend.t(qacc), contact_wrench=True)
    assert qfrc.shape == (len(qv), om.model.nv) and cw.shape == (len(qv), om.model.nbody, 6)
    assert torch.equal(qfrc, want) and torch.equal(cw, wcw)
    assert bool(torch.isfinite(qfrc).all()) and float(qfrc[:, :6].abs().max()) > 0.0
