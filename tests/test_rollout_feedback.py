"""Closed-loop rollouts (smplsim_rollout_feedback, HumanoidBatchB200.rollout(gains=...)): time-varying linear state feedback inside the
rollout kernel, u_t = ubar_t + K_t (x_t (-) xbar_t), and the position tangent it is written in (differentiate_pos / integrate_pos,
envs.mj_differentiatePos / mj_integratePos).

The kernel tests run on the H100 (-m gpu) and on the host emulator build of the same kernels; sizes marked gpu_only are H100 only."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_forward_fd import _tangent
from test_rollout import CASES, _bit_equal, _controls, _over_cap_row, _states
from util_states import airborne_states, make_models

from smplsim_b200 import envs

KEYS = ("qpos", "qvel", "status")
POSE_KEYS = KEYS + ("xpos", "xquat")


def _np_diff(qr, q):
    """fp64 [dq] of qr -> q: the law of smplsim.h, written independently of the library."""
    nv = len(q) - 1
    b, c = qr[3:7] / np.linalg.norm(qr[3:7]), q[3:7] / np.linalg.norm(q[3:7])
    rw = b[0] * c[0] + b[1:] @ c[1:]
    rv = b[0] * c[1:] - c[0] * b[1:] - np.cross(b[1:], c[1:])
    if rw < 0:
        rw, rv = -rw, -rv
    s = np.linalg.norm(rv)
    d = np.zeros(nv)
    d[0:3] = q[0:3] - qr[0:3]
    d[3:6] = 0.0 if s == 0 else rv / s * 2 * np.arctan2(s, rw)
    d[6:] = q[7:] - qr[7:]
    return d


def _pre_states(q0, v0, out):
    """x_t of every step: the start state, then the output rows 0 .. T-2."""
    qs = torch.cat([q0[:, None], out["qpos"][:, :-1]], 1)
    vs = torch.cat([v0[:, None], out["qvel"][:, :-1]], 1)
    return qs, vs


def _problem(backend, om, m, n, T, mode, seed, scale=0.05):
    """Start rows, feedforward, random gains and references perturbed from an open-loop run of the rows."""
    q, v, w = _states(om, n, seed=seed)
    u = _controls(m, n, T, mode, seed=seed + 1)
    rng = np.random.default_rng(seed + 2)
    K = np.float32(rng.normal(size=(n, T, m.nu, 2 * m.nv)) * scale * (1.0 if mode == "action" else 20.0))
    return q, v, w, u, K, rng


# ------------------------------------------------------------------ 1. zero gains are the open-loop rollout
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
@pytest.mark.parametrize("control_mode,mode,nsub", CASES)
def test_zero_gains_match_rollout(backend, robot, control_mode, mode, nsub):
    cfg, om = make_models(robot=robot, control_mode=control_mode)
    m = om.model
    q, v, w = _states(make_models(robot=robot, control_mode="uhc_pd")[1], 4, seed=3)
    T = 3
    u = _controls(m, 4, T, mode, seed=4) * 3
    u[3, 1] = np.nan
    env = backend.batch(cfg, 4)
    t = backend.t
    rng = np.random.default_rng(5)
    qr, vr = t(np.tile(q[:, None], (1, T, 1))), t(rng.normal(size=(4, T, m.nv)))
    for poses in (True, False):
        ref = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=poses)
        got = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=poses,
                          gains=t(np.zeros((1, T, m.nu, 2 * m.nv))), qpos_ref=qr[:1], qvel_ref=vr[:1])
        _bit_equal(got, ref, POSE_KEYS if poses else KEYS, f"zero gains, poses {poses}")
        uc = t(u)
        if mode == "action" and cfg.env.clip_actions:
            uc = torch.clamp(uc, -1.0, 1.0)
        assert torch.equal(torch.nan_to_num(got["control"], 7.0), torch.nan_to_num(uc, 7.0))


# ------------------------------------------------------------------ 2. replay of the applied controls
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
@pytest.mark.parametrize("control_mode,mode,nsub", CASES)
def test_replay_applied_controls(backend, robot, control_mode, mode, nsub):
    """Random gains and perturbed references, one row driven into an auto-reset: the open-loop rollout of the feedback run's own
    controls gives every output bit for bit."""
    cfg, om = make_models(robot=robot, control_mode=control_mode)
    m = om.model
    T = 3
    q, v, w, u, K, rng = _problem(backend, make_models(robot=robot, control_mode="uhc_pd")[1], m, 4, T, mode, seed=11)
    env = backend.batch(cfg, 4)
    t = backend.t
    nom = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w))
    qs, vs = _pre_states(t(q), t(v), nom)
    qr = qs + t(rng.normal(size=qs.shape) * 0.01)
    vr = vs + t(rng.normal(size=vs.shape) * 0.1)
    Kt = t(K)
    Kt[2, 1] = float("nan") if mode == "ctrl" or control_mode == "uhc_pd" else 1e30   # row 2 resets at step 1
    got = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=True, gains=Kt, qpos_ref=qr, qvel_ref=vr)
    assert got["status"][2, 1].item() & 7 or mode == "action" and control_mode != "uhc_pd"
    rep = env.rollout(t(q), t(v), got["control"], mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=True)
    _bit_equal(got, rep, POSE_KEYS, "feedback run vs replay of its controls")


# ------------------------------------------------------------------ 3. the law, in fp64
@pytest.mark.parametrize("control_mode,mode,nsub", [("uhc_pd", "action", None), ("torque", "ctrl", 1)])
def test_law_in_fp64(backend, control_mode, mode, nsub):
    """Every control[i, t] recomputed in fp64 from the recorded x_t.  References with the opposite quaternion sign, non-unit
    quaternions and a relative root rotation near pi; the action-mode clamp and its NaN rule."""
    cfg, om = make_models(control_mode=control_mode)
    m = om.model
    n, T = 4, 3
    q, v, w, u, K, rng = _problem(backend, om, m, n, T, mode, seed=21, scale=0.02)
    env = backend.batch(cfg, n)
    t = backend.t
    nom = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w))
    qs, vs = (x.cpu().numpy().astype(np.float64) for x in _pre_states(t(q), t(v), nom))
    qr = qs + rng.normal(size=qs.shape) * 0.01
    vr = vs + rng.normal(size=vs.shape) * 0.1
    qr[1, :, 3:7] *= -1.0                                   # -qbar: the same rotation
    qr[2, :, 3:7] *= 1.7                                    # not unit
    for s in range(T):                                      # row 3: relative root rotation of pi - 0.05 about a random axis
        a = rng.normal(size=3); a /= np.linalg.norm(a)
        th = np.pi - 0.05
        e = np.concatenate([[np.cos(th / 2)], np.sin(th / 2) * a])
        b = qs[3, s, 3:7]
        qr[3, s, 3:7] = [b[0] * e[0] - b[1:] @ e[1:], *(b[0] * e[1:] + e[0] * b[1:] + np.cross(b[1:], e[1:]))]
    uu = u.copy()
    if mode == "action":
        uu[0, 0, :5] = 30.0                                 # clamped
        uu[0, 2, 7] = np.nan                                # passes
    got = env.rollout(t(q), t(v), t(uu), mode=mode, nsub=nsub, qacc_warmstart=t(w), gains=t(K), qpos_ref=t(qr), qvel_ref=t(vr))
    xq, xv = (x.cpu().numpy().astype(np.float64) for x in _pre_states(t(q), t(v), got))
    ug = got["control"].cpu().numpy().astype(np.float64)
    qr32, vr32, K64 = np.float32(qr).astype(np.float64), np.float32(vr).astype(np.float64), K.astype(np.float64)
    worst = 0.0
    for i in range(n):
        for s in range(T):
            if mode == "action" and i == 0 and s == 2:
                continue                                    # the NaN row: checked below
            dx = np.concatenate([_np_diff(qr32[i, s], xq[i, s]), xv[i, s] - vr32[i, s]])
            Kdx = K64[i, s] * dx[None]
            ref = uu[i, s].astype(np.float64) + Kdx.sum(1)
            scale = np.abs(Kdx).sum(1) + np.abs(uu[i, s])
            if mode == "action" and cfg.env.clip_actions:
                ref = np.clip(ref, -1, 1)
            worst = max(worst, float(np.max(np.abs(ug[i, s] - ref) / scale)))
    assert worst < 1e-5, worst
    if mode == "action":
        assert np.all(ug[0, 0, :5] == 1.0)
        assert np.isnan(ug[0, 2, 7]) and got["status"][0, 2].item() & 7


# ------------------------------------------------------------------ 4. zero deviation is exact
@pytest.mark.parametrize("control_mode,mode,nsub", [("uhc_pd", "action", None), ("torque", "ctrl", 1)])
def test_zero_deviation_is_exact(backend, control_mode, mode, nsub):
    """The reference is an open-loop run's own pre-step states, K large and random: bit-identical with that run (dx is exactly 0)."""
    cfg, om = make_models(control_mode=control_mode)
    m = om.model
    T = 3
    q, v, w, u, K, _ = _problem(backend, om, m, 4, T, mode, seed=31, scale=50.0)
    env = backend.batch(cfg, 4)
    t = backend.t
    nom = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=True)
    qs, vs = _pre_states(t(q), t(v), nom)
    got = env.rollout(t(q), t(v), t(u), mode=mode, nsub=nsub, qacc_warmstart=t(w), body_poses=True, gains=t(K), qpos_ref=qs, qvel_ref=vs)
    _bit_equal(got, nom, POSE_KEYS, "zero deviation")


# ------------------------------------------------------------------ 5. shared against per-row
def test_shared_matches_expanded(backend):
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    T = 3
    q, v, w, u, K, rng = _problem(backend, om, m, 5, T, "action", seed=41)
    env = backend.batch(cfg, 8)
    t = backend.t
    qr = t(np.tile(q[:1, None], (1, T, 1)) + rng.normal(size=(1, T, m.nq)) * 0.01)
    vr = t(rng.normal(size=(1, T, m.nv)))
    Ks = t(K[:1])
    one = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), gains=Ks, qpos_ref=qr, qvel_ref=vr)
    allr = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), gains=Ks.expand(5, -1, -1, -1).contiguous(),
                       qpos_ref=qr.expand(5, -1, -1).contiguous(), qvel_ref=vr.expand(5, -1, -1).contiguous())
    _bit_equal(one, allr, KEYS + ("control",), "ref_rows 1 vs n")


# ------------------------------------------------------------------ 6. launch shapes
def _fb_rows(om, m, n, T, mode, seed):
    q, v, w = _states(om, n, seed=seed, nair=5 if n > 10 else 1)
    rng = np.random.default_rng(seed + 1)
    u = _controls(m, n, T, mode, seed=seed + 2)
    K = np.float32(rng.normal(size=(n, T, m.nu, 2 * m.nv)) * (0.05 if mode == "action" else 1.0))
    qr = np.float32(q[:, None] + rng.normal(size=(n, T, m.nq)) * 0.01)
    vr = np.float32(v[:, None] + rng.normal(size=(n, T, m.nv)) * 0.1)
    return q, v, w, u, K, qr, vr


def test_launch_shapes(backend, monkeypatch):
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    n, T = 37, 2
    q, v, w, u, K, qr, vr = _fb_rows(om, m, n, T, "action", seed=51)
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    small = backend.batch(cfg, 32)
    monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    big = backend.batch(cfg, 4096)
    wpb = lambda e: e._L().smplsim_warps_per_block(e._h)  # noqa: E731
    assert wpb(small) == 1 and wpb(big) == 8
    t = backend.t
    for kw in (dict(mode="action"), dict(mode="ctrl", nsub=2)):
        uu = u if kw["mode"] == "action" else u * 40
        outs = [e.rollout(t(q), t(v), t(uu), qacc_warmstart=t(w), body_poses=True, gains=t(K), qpos_ref=t(qr), qvel_ref=t(vr), **kw)
                for e in (small, big)]
        _bit_equal(outs[0], outs[1], POSE_KEYS + ("control",), f"{kw}: 1-warp chunks vs 8-warp CTAs")
    z = big.rollout(t(np.zeros((0, m.nq))), t(np.zeros((0, m.nv))), t(np.zeros((0, 4, m.nu))), gains=t(np.zeros((1, 4, m.nu, 2 * m.nv))),
                    qpos_ref=t(np.zeros((1, 4, m.nq))), qvel_ref=t(np.zeros((1, 4, m.nv))))
    assert z["qpos"].shape == (0, 4, m.nq) and z["control"].shape == (0, 4, m.nu)


@pytest.mark.gpu_only
def test_production_launch_shapes(backend, monkeypatch):
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q, v, w, u, K, qr, vr = _fb_rows(om, m, 64, 4, "action", seed=53)
    idx = np.random.default_rng(54).integers(0, 64, 5000)
    t = backend.t
    args = (t(q[idx]), t(v[idx]), t(u[idx]))
    kw = dict(qacc_warmstart=t(w[idx]), body_poses=True, gains=t(K[idx]), qpos_ref=t(qr[idx]), qvel_ref=t(vr[idx]))
    got = backend.batch(cfg, 4096).rollout(*args, **kw)
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    small = backend.batch(cfg, 1024)
    monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    _bit_equal(got, small.rollout(*args, **kw), POSE_KEYS + ("control",), "4 096-env handle vs 1-warp chunks")


# ------------------------------------------------------------------ 7. per-env shapes and parameter records
def test_per_env_shapes_and_parameters(backend, tmp_path):
    """Row i follows env i: replaying its applied controls on the open-loop path of the same handle gives the same bits; n !=
    num_envs is refused."""
    from smplsim_b200.abi import model_from_cfg
    from test_cta_shapes import _shape_variant
    path = _shape_variant(tmp_path, leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)
    cfg, om = make_models(control_mode="uhc_pd")
    cfg_b = make_models(control_mode="uhc_pd", **{"robot.xml_path": path})[0]
    m = om.model
    q, v, w, u, K, qr, vr = _fb_rows(om, m, 4, 2, "action", seed=61)
    t = backend.t
    kw = dict(gains=t(K), qpos_ref=t(qr), qvel_ref=t(vr))
    shaped = backend.batch(cfg, 4, models=[model_from_cfg(cfg), model_from_cfg(cfg_b)], env_model=np.array([0, 1, 1, 0], dtype=np.int32))
    penv = backend.batch(cfg, 4)
    penv.set_env_params(friction=t(np.array([1.0, 0.6, 1.0, 1.2])),
                        kp=t(np.tile(m.act_kp, (4, 1)) * np.array([[1.0], [1.3], [0.7], [1.0]])))
    plain = backend.batch(cfg, 4).rollout(t(q), t(v), t(u), qacc_warmstart=t(w), **kw)
    for env in (shaped, penv):
        got = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), body_poses=True, **kw)
        rep = env.rollout(t(q), t(v), got["control"], qacc_warmstart=t(w), body_poses=True)
        _bit_equal(got, rep, POSE_KEYS, "per-env handle: replay")
        assert not torch.equal(got["qvel"][1], plain["qvel"][1])   # row 1 is env 1's: another shape, other parameters
        if env is shaped:
            assert torch.equal(got["qvel"][0], plain["qvel"][0])      # env 0 has the handle's first shape
        with pytest.raises(Exception, match="n must be the handle's num_envs"):
            env.rollout(t(q[:3]), t(v[:3]), t(u[:3]), gains=t(K[:1]), qpos_ref=t(qr[:1]), qvel_ref=t(vr[:1]))


# ------------------------------------------------------------------ 8. bad rows stay local
def test_bad_rows_stay_local(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v, w, u, K, qr, vr = _fb_rows(make_models(control_mode="uhc_pd")[1], m, 5, 2, "ctrl", seed=71)
    t = backend.t
    env = backend.batch(cfg, 5)
    good = env.rollout(t(q), t(v), t(u * 30), mode="ctrl", qacc_warmstart=t(w), gains=t(K), qpos_ref=t(qr), qvel_ref=t(vr))
    Kb, qrb, vrb = K.copy(), qr.copy(), vr.copy()
    Kb[1, 0, 3, 7] = np.nan
    qrb[2, 0, 12] = np.nan
    vrb[3, 1, 4] = np.nan
    bad = env.rollout(t(q), t(v), t(u * 30), mode="ctrl", qacc_warmstart=t(w), gains=t(Kb), qpos_ref=t(qrb), qvel_ref=t(vrb))
    st = bad["status"].cpu().numpy()
    assert st[1, 0] & 7 and st[2, 0] & 7 and st[3, 1] & 7, st
    for k in KEYS + ("control",):
        for i in (0, 4):
            assert torch.equal(bad[k][i], good[k][i]), (k, i)


# ------------------------------------------------------------------ 9. no side effects
def test_stepper_cannot_tell(backend):
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_roll in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for s in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_roll and s == 0:   # more rows than envs: every scratch row of the handle, twice
                nn = n + n // 2
                qq = env.qpos.repeat(2, 1)[:nn]
                f = lambda *s_: torch.as_tensor(rin.normal(size=s_), dtype=torch.float32, device=qq.device)  # noqa: E731
                env.rollout(qq, f(nn, m.nv), f(nn, 2, m.nu), body_poses=True, gains=f(1, 2, m.nu, 2 * m.nv) * 0.05,
                            qpos_ref=qq[:1, None].repeat(1, 2, 1), qvel_ref=f(1, 2, m.nv))
                env.rollout(qq, f(nn, m.nv), f(nn, 2, m.nu) * 30, mode="ctrl", nsub=2, gains=f(nn, 2, m.nu, 2 * m.nv),
                            qpos_ref=qq[:, None].repeat(1, 2, 1), qvel_ref=f(nn, 2, m.nv))
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel,
                                                  env.body_angvel, env.xpos, env.xquat, env.obs_buf, env.task_target, env.progress_buf)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------ 10. arguments
def test_arguments(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    L, h, s = env._L(), env._h, env._stream()
    q, v = airborne_states(m, 4, seed=1)
    t = backend.t
    tq, tv, tu = t(q), t(v), t(np.zeros((4, 2, m.nu)))
    tK, tqr, tvr = t(np.zeros((1, 2, m.nu, 2 * m.nv))), t(np.tile(q[:1, None], (1, 2, 1))), t(np.zeros((1, 2, m.nv)))
    oq, ov, oc = t(np.zeros((4, 2, m.nq))), t(np.zeros((4, 2, m.nv))), t(np.zeros((4, 2, m.nu)))
    p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731

    def call(hh=h, mode=0, nsub=0, n=4, K=p(tK), qr=p(tqr), vr=p(tvr), rows=1, uo=p(oc)):
        return L.smplsim_rollout_feedback(hh, mode, nsub, p(tq), p(tv), None, None, None, p(tu), n, 2, p(oq), p(ov), None, None, None,
                                          K, qr, vr, rows, 1, uo, s)

    def err(rc, code, text):
        assert rc == code, (rc, code)
        assert L.smplsim_last_error().decode() == text

    err(call(hh=None), -1, "smplsim_rollout_feedback: null handle, n < 0 or nstep < 1")
    err(call(mode=1, nsub=0), -1, "smplsim_rollout_feedback: SMPLSIM_ROLLOUT_CTRL needs nsub >= 1")
    null = "smplsim_rollout_feedback: null argument (gain, qpos_ref and qvel_ref are required)"
    err(call(K=None), -1, null)
    err(call(qr=None), -1, null)
    err(call(vr=None), -1, null)
    rows = "smplsim_rollout_feedback: ref_rows must be 1 (one schedule for every row) or n (one per row)"
    err(call(rows=2), -1, rows)
    err(call(rows=0), -1, rows)
    assert call() == 0 and call(uo=None) == 0
    penv = backend.batch(make_models(control_mode="simple_pid")[0], 4)
    err(call(hh=penv._h), -3,
        "smplsim_rollout_feedback: control_mode simple_pid keeps its integral / last error in env state, which rollout rows do not have")
    senv = backend.batch(make_models(env="getup", control_mode="torque", self_collision=True)[0], 4)
    err(call(hh=senv._h), -3,
        "smplsim_rollout_feedback: the rollout on caller rows does not build geom-geom contacts (handle created with self_collision = 1)")

    K4 = t(np.zeros((4, 2, m.nu, 2 * m.nv)))
    with pytest.raises(ValueError, match="give gains"):
        env.rollout(tq, tv, tu, qpos_ref=tqr)
    with pytest.raises(ValueError, match="give gains"):
        env.rollout(tq, tv, tu, qvel_ref=tvr)
    with pytest.raises(ValueError, match="need qpos_ref and qvel_ref"):
        env.rollout(tq, tv, tu, gains=tK, qpos_ref=tqr)
    with pytest.raises(ValueError, match="leading dimension 1"):
        env.rollout(tq, tv, tu, gains=K4[:2], qpos_ref=tqr, qvel_ref=tvr)
    with pytest.raises(ValueError, match="gains must have shape"):
        env.rollout(tq, tv, tu, gains=K4[:, :, :, :-1], qpos_ref=tqr, qvel_ref=tvr)
    with pytest.raises(ValueError, match="qpos_ref must have shape"):
        env.rollout(tq, tv, tu, gains=K4, qpos_ref=tqr, qvel_ref=tvr)
    with pytest.raises(ValueError, match="qvel_ref must have shape"):
        env.rollout(tq, tv, tu, gains=tK, qpos_ref=tqr, qvel_ref=tvr[:, :1])


# ------------------------------------------------------------------ 11. differentiate_pos / integrate_pos
def test_tangent_helpers(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    rng = np.random.default_rng(81)
    q0, _ = airborne_states(m, 6, seed=82)
    q0 = q0.astype(np.float64)
    dq = rng.normal(size=(6, m.nv)) * 0.3
    dq[5, 3:6] = [2.9, 0.4, -0.3]                       # a large root rotation
    dv = torch.device(env.device)
    T = lambda x: torch.as_tensor(x, dtype=torch.float64, device=dv)  # noqa: E731
    q1 = env.integrate_pos(T(q0), T(dq))
    back = env.differentiate_pos(T(q0), q1).cpu().numpy()
    assert np.abs(back - dq).max() < 1e-9
    for i in range(6):                                   # the numpy shims, in place
        qq = q0[i].copy()
        envs.mj_integratePos(None, qq, dq[i] / 0.5, 0.5)
        assert np.abs(qq - q1[i].cpu().numpy()).max() < 1e-12
        d = np.zeros(m.nv)
        envs.mj_differentiatePos(None, d, 0.5, q0[i], qq)
        assert np.abs(d * 0.5 - dq[i]).max() < 1e-9
        ref = _tangent(m, qq, np.zeros(m.nv), q0[i], np.zeros(m.nv))[:m.nv]
        assert np.abs(ref - back[i]).max() < 1e-9
    neg = T(q0.copy()); neg[:, 3:7] *= -2.0               # sign and scale of the reference quaternion do not matter
    assert torch.allclose(env.differentiate_pos(neg, q1), env.differentiate_pos(T(q0), q1), atol=1e-12, rtol=0)
    f32 = env.differentiate_pos(T(q0).float(), q1.float()).double().cpu().numpy()
    assert np.abs(f32 - dq).max() < 1e-5

    # the position update of a ctrl-mode rollout step: q' = integrate_pos(q, h v')
    q, v, w = _states(make_models(control_mode="uhc_pd")[1], 4, seed=83)
    u = _controls(m, 4, 1, "ctrl", seed=84)
    out = env.rollout(backend.t(q), backend.t(v), backend.t(u), mode="ctrl", qacc_warmstart=backend.t(w))
    h = float(env.model.timestep)
    pred = env.integrate_pos(T(q), h * out["qvel"][:, 0].double())
    assert torch.abs(pred - out["qpos"][:, 0].double()).max().item() < 1e-5


# ------------------------------------------------------------------ 12. one iLQR iteration
@pytest.mark.gpu_only
def test_one_ilqr_iteration(backend):
    """The example's iteration inlined (SMPL, ctrl mode, nsub = 1, T = 10): the alpha = 0 row reproduces the nominal bit for bit and
    the best row's tracking cost is strictly below the nominal's."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("ilqr_track", os.path.join(os.path.dirname(__file__), "..", "examples", "ilqr_track.py"))
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    cfg, om = make_models(control_mode="torque")
    env = backend.batch(cfg, 8)
    prob = ex.make_problem(env, T=10, seed=91)
    nom = ex.nominal(env, prob)
    it = ex.iteration(env, prob, nom)
    _bit_equal(it["rows"][0], nom, KEYS, "alpha = 0 row vs nominal")
    assert it["best_cost"] < nom["cost"], (it["best_cost"], nom["cost"])
