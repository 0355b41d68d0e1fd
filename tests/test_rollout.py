"""Rollouts from caller states (smplsim_rollout, HumanoidBatchB200.rollout, envs.rollout): bit-identical with the env path they
stand for (set_state + T x step / mj_step on a fresh batch), against the fp64 oracle, and without effect on the envs.

The kernel tests run on the H100 (-m gpu) and on the host emulator build of the same kernels; sizes marked gpu_only are H100 only."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from test_inverse import _forward, _over_cap
from util_states import airborne_states, make_models, relerr, rollout_states

SELF_CONTACT = 32   # SMPLSIM_STATUS_SELF_CONTACT: raised by step, not evaluated by the rollout
CASES = [("uhc_pd", "action", None), ("pd", "action", None), ("torque", "action", None), ("torque", "ctrl", 1), ("torque", "ctrl", 15)]


def _states(om, n, seed, nair=1):
    """n start rows: contact-rich states of stable-PD rollouts (with their warm starts), then nair airborne states."""
    m = om.model
    q, v, w = rollout_states(om, n - nair, seed=seed, every=7)
    qa, va = airborne_states(m, nair, seed=seed + 1)
    return (np.float32(np.concatenate([q, qa])), np.float32(np.concatenate([v, va])),
            np.float32(np.concatenate([w, np.zeros((nair, m.nv))])))


def _controls(m, n, T, mode, seed):
    rng = np.random.default_rng(seed)
    return np.float32(rng.normal(size=(n, T, m.nu)) * (0.4 if mode == "action" else 25.0))


def _env_path(backend, cfg, q, v, w, u, mode, nsub, qf=None, vf=None, **kw):
    """What the rollout stands for: a fresh batch, set_state + qacc_warm (+ the last forward state), then one call per control row."""
    env = backend.batch(cfg, len(q), **kw)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    if qf is not None:
        env.qpos_fwd.copy_(backend.t(qf)); env.qvel_fwd.copy_(backend.t(vf))
    out = {k: [] for k in ("qpos", "qvel", "status", "xpos", "xquat")}
    for t in range(u.shape[1]):
        if mode == "action":
            env.step(backend.t(u[:, t]))
        else:
            env.mj_step(backend.t(u[:, t]), nsub)
        for k, x in (("qpos", env.qpos), ("qvel", env.qvel), ("status", env.status & ~SELF_CONTACT), ("xpos", env.xpos), ("xquat", env.xquat)):
            out[k].append(x.clone())
    return {k: torch.stack(x, 1) for k, x in out.items()}


def _bit_equal(got, ref, keys, what):
    for k in keys:
        a, b = got[k].cpu().numpy(), ref[k].cpu().numpy()
        assert a.shape == b.shape, (what, k, a.shape, b.shape)
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (what, k, np.argwhere(a.view(np.uint8) != b.view(np.uint8))[:4])


# ------------------------------------------------------------------ 1. the env path, bit for bit
@pytest.mark.parametrize("poses", [True, False])
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
@pytest.mark.parametrize("control_mode,mode,nsub", CASES)
def test_matches_env_path(backend, robot, control_mode, mode, nsub, poses):
    """Contact-rich and airborne rows, and one row driven into an auto-reset at step 1 (a NaN control row): every recorded qpos,
    qvel, status and (with poses) pose bit-identical with set_state + T calls on a fresh batch.  Without poses the rollout normalises
    the root quaternion on one lane instead of in the pose sweep; both branches are held to the env path."""
    cfg, om = make_models(robot=robot, control_mode=control_mode)
    m = om.model
    q, v, w = _states(make_models(robot=robot, control_mode="uhc_pd")[1], 4, seed=3)
    T = 3
    u = _controls(m, 4, T, mode, seed=4)
    u[3, 1] = np.nan
    got = backend.batch(cfg, 4).rollout(backend.t(q), backend.t(v), backend.t(u), mode=mode, nsub=nsub, qacc_warmstart=backend.t(w),
                                        body_poses=poses)
    ref = _env_path(backend, cfg, q, v, w, u, mode, nsub)
    _bit_equal(got, ref, ("qpos", "qvel", "status") + (("xpos", "xquat") if poses else ()), "rollout vs env path")
    assert ("xpos" in got) == poses
    st = got["status"].cpu().numpy()
    if control_mode == "uhc_pd" or mode == "ctrl":   # the pd / torque controllers clamp a NaN action to a finite torque
        assert st[3, 1] & 7, st[3]
    assert np.isfinite(got["qpos"].cpu().numpy()).all()


def test_forward_state_rows(backend):
    """Stable PD with stale inertia reads the state of the last forward pass: qpos_fwd / qvel_fwd given to the rollout equal an env
    whose qpos_fwd / qvel_fwd hold the same rows (and differ from the default, the start state)."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q, v, w = _states(om, 4, seed=8)
    qf, vf, _ = _states(om, 4, seed=9)
    u = _controls(m, 4, 2, "action", seed=10)
    env = backend.batch(cfg, 4)
    t = backend.t
    got = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), qpos_fwd=t(qf), qvel_fwd=t(vf))
    _bit_equal(got, _env_path(backend, cfg, q, v, w, u, "action", None, qf, vf), ("qpos", "qvel", "status"), "qpos_fwd / qvel_fwd rows")
    plain = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w))
    assert not torch.equal(plain["qvel"], got["qvel"])


def test_continues_an_env(backend):
    """An env's own rows (qpos, qvel, qacc_warm, qpos_fwd, qvel_fwd) continue its physics to the solver's tolerance: only the
    working-set memory, which the rollout starts empty, differs."""
    cfg, om = make_models(env="speed", control_mode="uhc_pd")
    m = om.model
    n, T = 4, 3
    env = backend.batch(cfg, n, seed=2)
    env.reset()
    rng = np.random.default_rng(3)
    for _ in range(3):
        env.step(backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.3, -1, 1)))
    u = _controls(m, n, T, "action", seed=4)
    got = env.rollout(env.qpos.clone(), env.qvel.clone(), backend.t(u), qacc_warmstart=env.qacc_warm.clone(), qpos_fwd=env.qpos_fwd.clone(),
                      qvel_fwd=env.qvel_fwd.clone())
    for t in range(T):
        env.step(backend.t(u[:, t]))
        assert relerr(got["qpos"][:, t].cpu().numpy(), env.qpos.cpu().numpy()) < 1e-3 * (t + 1), t
        assert relerr(got["qvel"][:, t].cpu().numpy(), env.qvel.cpu().numpy()) < 2e-2 * (t + 1), t


# ------------------------------------------------------------------ 2. against the fp64 oracle
def _oracle_from(om, q, v, w):
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w
    e.warn = 0
    return e


def test_steps_match_oracle(backend):
    """Every recorded step t of a ctrl-mode rollout (nsub = 1) from contact-rich states against one oracle mj_step from the kernel's
    recorded state t - 1: norm-relative 1e-4, the bound test_gpu_parity holds one mj_step to."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    n, T = 4, 3
    q, v, w = _states(make_models(control_mode="uhc_pd")[1], n, seed=12)
    u = _controls(m, n, T, "ctrl", seed=13)
    got = backend.batch(cfg, n).rollout(backend.t(q), backend.t(v), backend.t(u), mode="ctrl", qacc_warmstart=backend.t(w))
    gq, gv = got["qpos"].cpu().numpy().astype(np.float64), got["qvel"].cpu().numpy().astype(np.float64)
    assert not got["status"].cpu().numpy().any()
    for i in range(n):
        for t in range(T):
            q0, v0 = (q[i], v[i]) if t == 0 else (gq[i, t - 1], gv[i, t - 1])
            e = _oracle_from(om, q0, v0, w[i] if t == 0 else np.zeros(m.nv))
            e.ctrl[:] = u[i, t]
            e.mj_step()
            assert relerr(gq[i, t], e.qpos) < 1e-4, (i, t, relerr(gq[i, t], e.qpos))
            assert relerr(gv[i, t], e.qvel) < 1e-4, (i, t, relerr(gv[i, t], e.qvel))


@pytest.mark.parametrize("control_mode,tol", [("torque", 1e-4), ("pd", 5e-4)])
def test_action_steps_match_oracle(backend, control_mode, tol):
    """Action mode against the oracle's env step, which applies the controller (torque: scale and clamp; pd: PD torque on the state,
    clamp) before each substep: every recorded step t from the kernel's state t - 1, on a model with one substep per action step, so
    that each step is one controller evaluation and one mj_step.  (With the default 15 substeps the pd and torque controllers drive
    contact-rich states into joint-limit and contact switches within a step, where fp32 and fp64 part ways.)  Norm-relative: torque
    1e-4, the one-mj_step bound; pd 5e-4, as kp times the fp32 rounding of the joint angle enters the torque (worst seen on the
    emulator 1.8e-4)."""
    cfg, om = make_models(control_mode=control_mode, control_frequency_inv=1)
    m = om.model
    n, T = 6, 3
    q, v, w = _states(make_models(control_mode="uhc_pd")[1], n, seed=12, nair=0)
    u = np.clip(_controls(m, n, T, "action", seed=13), -1, 1)
    got = backend.batch(cfg, n).rollout(backend.t(q), backend.t(v), backend.t(u), qacc_warmstart=backend.t(w))
    gq, gv = got["qpos"].cpu().numpy().astype(np.float64), got["qvel"].cpu().numpy().astype(np.float64)
    assert not got["status"].cpu().numpy().any()
    for i in range(n):
        for t in range(T):
            q0, v0 = (q[i], v[i]) if t == 0 else (gq[i, t - 1], gv[i, t - 1])
            e = _oracle_from(om, q0, v0, w[i] if t == 0 else np.zeros(m.nv))
            e.step(u[i, t])
            assert relerr(gq[i, t], e.qpos) < tol, (i, t, relerr(gq[i, t], e.qpos))
            assert relerr(gv[i, t], e.qvel) < tol, (i, t, relerr(gv[i, t], e.qvel))


def test_free_run_matches_oracle(backend):
    """Five mj_step substeps free-running from airborne states (no contacts: the trajectories stay close), ctrl mode nsub = 1."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v = airborne_states(m, 4, seed=21)
    q, v = np.float32(q), np.float32(v)
    u = _controls(m, 4, 5, "ctrl", seed=22)
    got = backend.batch(cfg, 4).rollout(backend.t(q), backend.t(v), backend.t(u), mode="ctrl")
    gq, gv = got["qpos"].cpu().numpy(), got["qvel"].cpu().numpy()
    for i in range(4):
        e = _oracle_from(om, q[i], v[i], np.zeros(m.nv))
        for t in range(5):
            e.ctrl[:] = u[i, t]
            e.mj_step()
            assert relerr(gq[i, t], e.qpos) < 1e-4 * (t + 1), (i, t)
            assert relerr(gv[i, t], e.qvel) < 1e-4 * (t + 1), (i, t)


# ------------------------------------------------------------------ 3. poses
def test_poses(backend):
    """Poses on or off: qpos / qvel bit-identical; xpos / xquat those of kinematics at the recorded qpos."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q, v, w = _states(om, 3, seed=31)
    u = _controls(m, 3, 3, "action", seed=32)
    env = backend.batch(cfg, 3)
    t = backend.t
    on = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), body_poses=True)
    off = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w))
    _bit_equal(on, off, ("qpos", "qvel", "status"), "poses on vs off")
    assert "xpos" not in off
    xp, xq = env.kinematics(on["qpos"].reshape(-1, m.nq))
    assert torch.allclose(on["xpos"].reshape(-1, m.nbody, 3), xp, atol=1e-6, rtol=0)
    assert torch.allclose(on["xquat"].reshape(-1, m.nbody, 4), xq, atol=1e-6, rtol=0)


# ------------------------------------------------------------------ 4. no side effects
def test_stepper_cannot_tell(backend):
    """step -> rollout -> step and step -> step from the same state: every env tensor, aux output and contact wrench bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_roll in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_roll and t == 0:   # more rows than envs: every scratch row of the handle, twice
                qq = env.qpos.repeat(2, 1)[: n + n // 2]
                vv = torch.as_tensor(rin.normal(size=(qq.shape[0], m.nv)), dtype=torch.float32, device=qq.device)
                uu = torch.as_tensor(rin.normal(size=(qq.shape[0], 2, m.nu)), dtype=torch.float32, device=qq.device)
                env.rollout(qq, vv, uu, body_poses=True)
                env.rollout(qq, vv, uu * 30, mode="ctrl", nsub=2)
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel,
                                                  env.body_angvel, env.xpos, env.xquat, env.obs_buf, env.task_target, env.progress_buf)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------ 5. launch shapes
def test_launch_shapes(backend, monkeypatch):
    """37 rows on a 32-env handle with 1-warp CTAs (two launches) and on a 4 096-env handle with 8-warp CTAs (a ragged second CTA):
    bit-identical in action and ctrl mode; n = 0 returns empty outputs."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    n = 37
    q, v, w = _states(om, n, seed=41, nair=5)
    u = _controls(m, n, 2, "action", seed=42)
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    small = backend.batch(cfg, 32)
    monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    big = backend.batch(cfg, 4096)
    wpb = lambda e: e._L().smplsim_warps_per_block(e._h)  # noqa: E731
    assert wpb(small) == 1 and wpb(big) == 8
    t = backend.t
    for kw in (dict(mode="action"), dict(mode="ctrl", nsub=3)):
        uu = u if kw["mode"] == "action" else u * 40
        outs = [e.rollout(t(q), t(v), t(uu), qacc_warmstart=t(w), body_poses=True, **kw) for e in (small, big)]
        _bit_equal(outs[0], outs[1], ("qpos", "qvel", "status", "xpos", "xquat"), f"{kw}: 1-warp chunks vs 8-warp CTAs")
    z = big.rollout(t(np.zeros((0, m.nq))), t(np.zeros((0, m.nv))), t(np.zeros((0, 4, m.nu))), body_poses=True)
    assert z["qpos"].shape == (0, 4, m.nq) and z["status"].shape == (0, 4) and z["xquat"].shape == (0, 4, m.nbody, 4)


@pytest.mark.gpu_only
def test_production_launch_shapes(backend, monkeypatch):
    """5 000 rows x 4 action steps on a 4 096-env handle (two launches, the second ragged) against the same rows on 1-warp CTAs in
    chunks of 1 024: bit-identical."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q, v, w = _states(om, 64, seed=43, nair=8)
    idx = np.random.default_rng(44).integers(0, 64, 5000)
    q, v, w = q[idx], v[idx], w[idx]
    u = _controls(m, 5000, 4, "action", seed=45)
    t = backend.t
    got = backend.batch(cfg, 4096).rollout(t(q), t(v), t(u), qacc_warmstart=t(w), body_poses=True)
    monkeypatch.setenv("SMPLSIM_WPB", "1")
    small = backend.batch(cfg, 1024)
    monkeypatch.delenv("SMPLSIM_WPB", raising=False)
    ref = small.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), body_poses=True)
    _bit_equal(got, ref, ("qpos", "qvel", "status", "xpos", "xquat"), "4 096-env handle vs 1-warp chunks")


# ------------------------------------------------------------------ 6. per-env shapes and parameter records
def test_per_env_shapes_and_parameters(backend, tmp_path):
    """Row i uses env i's shape and parameter record: bit-identical with env i's own env path; n != num_envs is refused."""
    from smplsim_b200.abi import model_from_cfg
    from test_cta_shapes import _shape_variant
    path = _shape_variant(tmp_path, leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)
    cfg, om = make_models(control_mode="uhc_pd")
    cfg_b = make_models(control_mode="uhc_pd", **{"robot.xml_path": path})[0]
    m = om.model
    models = [model_from_cfg(cfg), model_from_cfg(cfg_b)]
    env_model = np.array([0, 1, 1, 0], dtype=np.int32)
    q, v, w = _states(om, 4, seed=51)
    u = _controls(m, 4, 2, "action", seed=52)
    t = backend.t
    kw = dict(models=models, env_model=env_model)
    env = backend.batch(cfg, 4, **kw)
    got = env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), body_poses=True)
    _bit_equal(got, _env_path(backend, cfg, q, v, w, u, "action", None, **kw), ("qpos", "qvel", "status", "xpos", "xquat"), "per-env shapes")
    same = backend.batch(cfg, 4).rollout(t(q), t(v), t(u), qacc_warmstart=t(w))
    assert torch.equal(same["qvel"][0], got["qvel"][0]) and not torch.equal(same["qvel"][1], got["qvel"][1])
    with pytest.raises(Exception, match="n must be the handle's num_envs"):
        env.rollout(t(q[:3]), t(v[:3]), t(u[:3]))
    prm = dict(friction=t(np.array([1.0, 0.6, 1.0, 1.2])), kp=t(np.tile(m.act_kp, (4, 1)) * np.array([[1.0], [1.3], [0.7], [1.0]])),
               body_mass_scale=t(np.ones((4, m.nbody)) * np.array([[1.0], [1.0], [1.2], [0.9]])))
    penv = backend.batch(cfg, 4)
    penv.set_env_params(**prm)
    got = penv.rollout(t(q), t(v), t(u), qacc_warmstart=t(w))
    ref_env = backend.batch(cfg, 4)
    ref_env.set_env_params(**prm)
    ref_env.set_state(t(q), t(v)); ref_env.qacc_warm.copy_(t(w))
    for s in range(2):
        ref_env.step(t(u[:, s]))
        assert torch.equal(got["qpos"][:, s], ref_env.qpos) and torch.equal(got["qvel"][:, s], ref_env.qvel), s
    with pytest.raises(Exception, match="n must be the handle's num_envs"):
        penv.rollout(t(q[:2]), t(v[:2]), t(u[:2]))


# ------------------------------------------------------------------ 7. bad rows stay local
def _over_cap_row(om, seed=61):
    """An airborne state with 20 hinges past their range (more joint-limit rows than the kernels hold), moving further out."""
    m = om.model
    q, v = airborne_states(m, 1, seed=seed)
    q, v = q[0], v[0] * 0.1
    rlo, rhi = np.asarray(m.dof_range)[6:, 0], np.asarray(m.dof_range)[6:, 1]
    for k in range(20):
        q[7 + k] = rhi[k] + 0.3
        v[6 + k] = 2.0
    assert _over_cap(_forward(om, q, v))
    return np.float32(q), np.float32(v)


def test_bad_rows_stay_local(backend):
    """A NaN start row and a row past the joint-limit row cap raise their own status bits (1, 8); the other rows are bit-identical with
    a call without them."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v, w = _states(make_models(control_mode="uhc_pd")[1], 4, seed=62)
    qc, vc = _over_cap_row(om)
    qb, vb, wb = q.copy(), v.copy(), w.copy()
    qb[1, 9] = np.nan
    qb[2], vb[2], wb[2] = qc, vc, 0
    u = _controls(m, 4, 2, "ctrl", seed=63)
    env = backend.batch(cfg, 4)
    t = backend.t
    bad = env.rollout(t(qb), t(vb), t(u), mode="ctrl", qacc_warmstart=t(wb))
    good = env.rollout(t(q), t(v), t(u), mode="ctrl", qacc_warmstart=t(w))
    st = bad["status"].cpu().numpy()
    assert st[1, 0] & 1 and st[2, 0] & 8, st
    for k in ("qpos", "qvel", "status"):
        for i in (0, 3):
            assert torch.equal(bad[k][i], good[k][i]), (k, i)


# ------------------------------------------------------------------ 8. arguments
def test_arguments(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    L, h, s = env._L(), env._h, env._stream()
    q, v = airborne_states(m, 4, seed=1)
    tq, tv, tu = backend.t(q), backend.t(v), backend.t(np.zeros((4, 2, m.nu)))
    oq, ov = backend.t(np.zeros((4, 2, m.nq))), backend.t(np.zeros((4, 2, m.nv)))
    xp, xq = backend.t(np.zeros((4, 2, m.nbody, 3))), backend.t(np.zeros((4, 2, m.nbody, 4)))
    p = lambda x: C.c_void_p(x.data_ptr())  # noqa: E731

    def call(hh=h, mode=0, nsub=0, q0=p(tq), u=p(tu), n=4, T=2, qo=p(oq), xpos=None, xquat=None):
        return L.smplsim_rollout(hh, mode, nsub, q0, p(tv), None, None, None, u, n, T, qo, p(ov), None, xpos, xquat, s)

    def err(rc, code, text):
        assert rc == code, (rc, code)
        assert L.smplsim_last_error().decode() == text

    first = "smplsim_rollout: null handle, n < 0 or nstep < 1"
    err(call(hh=None), -1, first)
    err(call(n=-1), -1, first)
    err(call(T=0), -1, first)
    err(call(mode=2), -1, "smplsim_rollout: unknown mode")
    err(call(mode=1, nsub=0), -1, "smplsim_rollout: SMPLSIM_ROLLOUT_CTRL needs nsub >= 1")
    err(call(mode=0, nsub=1), -1, "smplsim_rollout: SMPLSIM_ROLLOUT_ACTION takes nsub = 0 (an action step runs cfg.env.nsubsteps substeps)")
    err(call(xpos=p(xp)), -1, "smplsim_rollout: give both xpos and xquat, or neither")
    err(call(xquat=p(xq)), -1, "smplsim_rollout: give both xpos and xquat, or neither")
    null = "smplsim_rollout: null argument (qpos0, qvel0, control, qpos and qvel are required)"
    err(call(q0=None), -1, null)
    err(call(u=None), -1, null)
    err(call(qo=None), -1, null)
    assert L.smplsim_rollout(h, 0, 0, None, None, None, None, None, None, 0, 2, None, None, None, None, None, s) == 0
    assert call(mode=1, nsub=2, xpos=p(xp), xquat=p(xq)) == 0

    t = backend.t
    for kw, match in ((dict(mode="torque"), "mode"), (dict(nsub=2), "nsub is for mode='ctrl'"), (dict(mode="ctrl", nsub=0), "nsub"),
                      (dict(mode="ctrl", nsub=1.5), "nsub")):
        with pytest.raises(ValueError, match=match):
            env.rollout(tq, tv, tu, **kw)
    with pytest.raises(ValueError, match="control must have shape"):
        env.rollout(tq, tv, tu[:, :, :-1])
    with pytest.raises(ValueError, match="control must have shape"):
        env.rollout(tq, tv, tu[0])
    with pytest.raises(ValueError, match="at least one step"):
        env.rollout(tq, tv, tu[:, :0])
    with pytest.raises(ValueError, match="float32"):
        env.rollout(tq, tv, tu.double())
    with pytest.raises(ValueError, match="qacc_warmstart must have shape"):
        env.rollout(tq, tv, tu, qacc_warmstart=tv[:3])
    with pytest.raises(ValueError, match="qpos_fwd must have shape"):
        env.rollout(tq, tv, tu, qpos_fwd=tv)

    pcfg, _ = make_models(control_mode="simple_pid")
    penv = backend.batch(pcfg, 4)
    err(call(hh=penv._h), -3, "smplsim_rollout: control_mode simple_pid keeps its integral / last error in env state, which rollout rows do not have")
    assert call(hh=penv._h, mode=1, nsub=1) == 0
    scfg, _ = make_models(env="getup", control_mode="torque", self_collision=True)
    senv = backend.batch(scfg, 4)
    err(call(hh=senv._h), -3,
        "smplsim_rollout: the rollout on caller rows does not build geom-geom contacts (handle created with self_collision = 1)")
    with pytest.raises(Exception, match="self_collision"):
        senv.rollout(t(q), t(v), tu)


# ------------------------------------------------------------------ 9. single env
def test_single_env_rollout(backend):
    """envs.rollout (MuJoCo's signature, state [time, qpos, qvel]) equals HumanoidBatchB200.rollout in ctrl mode on the same rows."""
    from smplsim_b200.envs import HumanoidSpeed, rollout
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
    m = om.model
    q, v = airborne_states(m, 3, seed=71)
    x0 = np.concatenate([np.array([[0.5], [0.0], [1.25]]), q, v], axis=1)
    u = _controls(m, 3, 4, "ctrl", seed=72).astype(np.float64)
    state, sens = rollout(env.mj_model, env.mj_data, x0, u)
    assert state.shape == (3, 4, 1 + m.nq + m.nv) and sens.shape == (3, 4, 0)
    b = env._b
    want = b.rollout(backend.t(q), backend.t(v), backend.t(u), mode="ctrl")
    assert np.array_equal(state[:, :, 1:1 + m.nq], want["qpos"].cpu().numpy().astype(np.float64))
    assert np.array_equal(state[:, :, 1 + m.nq:], want["qvel"].cpu().numpy().astype(np.float64))
    h = env.mj_model.opt.timestep
    assert np.allclose(state[:, :, 0], x0[:, :1] + h * np.arange(1, 5))
    one, _ = rollout(env.mj_model, env.mj_data, x0[0], u[0, :2], nstep=2)   # one state, one control sequence
    assert np.array_equal(one, state[:1, :2])
    with pytest.raises(ValueError, match="nstep"):
        rollout(env.mj_model, env.mj_data, x0, u, nstep=3)
