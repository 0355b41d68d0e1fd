"""Parity tests: the kernels (through the C ABI) vs the fp64 oracle / reference-generated goldens.
Every test runs on the GPU (`-m gpu`: libsmplsim_b200.so on cuda:0 -- the parity claim) and, where the size allows, once more
on the host SIMT emulator (tests/emu: the same kernel sources compiled for the CPU; part of the `-m "not gpu"` suite).

Tolerances: north_star asks for 1e-4 relative (fp32) on qpos/qvel after one mj_step and bit-exact
floor-contact flags; relerr(a,b) = max|a-b| / max(1, max|b|).
"""
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from conftest import GOLDEN  # noqa: E402
from oracle import oracle as orc  # noqa: E402
from util_states import airborne_states, elem_relerr, make_models, relerr, rollout_states  # noqa: E402

TOL = 1e-4


@pytest.mark.gpu_only
def test_extension_loaded_and_symbols(backend):
    from smplsim_b200 import _lib
    L = _lib.lib()
    assert L.smplsim_version() >= 100
    maps = open("/proc/self/maps").read()
    assert "libsmplsim_b200.so" in maps


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_kinematics_matches_oracle(backend, robot):
    cfg, om = make_models(robot=robot)
    m = om.model
    q, _ = airborne_states(m, 64, seed=1)
    q[:, 0:2] *= 10
    env = backend.batch(cfg, 1)
    xpos, xquat = env.kinematics(backend.t(q))
    e = orc.OracleEnv(om)
    for i in range(q.shape[0]):
        e.qpos[:] = q[i]; e.kinematics()
        assert np.abs(xpos[i].cpu().numpy() - e.xpos).max() < 2e-5
        d = np.minimum(np.abs(xquat[i].cpu().numpy() - e.xquat).max(axis=1), np.abs(xquat[i].cpu().numpy() + e.xquat).max(axis=1))
        assert d.max() < 1e-5


@pytest.mark.parametrize("name,robot", [("smpl", "smpl_humanoid"), ("smplx", "smplx_humanoid")])
def test_self_obs_matches_reference_golden(backend, name, robot):
    g = np.load(os.path.join(GOLDEN, f"obs_{name}.npz"))
    for upright, rh in ((False, True), (False, False), (True, True)):
        cfg, om = make_models(robot=robot, **{"root_height_obs": rh, "robot.has_upright_start": upright})
        env = backend.batch(cfg, 1)
        tag = f"u{int(upright)}h{int(rh)}"
        o1 = env.self_obs(1, backend.t(g["xpos"]), backend.t(g["xquat"]), qvel=backend.t(g["qvel"])).cpu().numpy()
        o2 = env.self_obs(2, backend.t(g["xpos"]), backend.t(g["xquat"]), linvel=backend.t(g["linvel"]), angvel=backend.t(g["angvel"])).cpu().numpy()
        # xpos is absolute (|x| up to 20 m) in fp32 -> 2e-6 absolute resolution on local positions
        assert np.abs(o1 - g["v1_" + tag]).max() < 2e-5
        assert np.abs(o2 - g["v2_" + tag]).max() < 2e-5


def _oracle_one_step(om, q, v, w, ctrl):
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w; e.ctrl[:] = ctrl
    e.mj_step()
    return e


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_mj_step_airborne(backend, robot):
    """No contact: qacc = M^-1 (tau - c) through ABA vs the oracle's CRB + L'DL."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    n = 32
    q, v = airborne_states(m, n, seed=3)
    rng = np.random.default_rng(5)
    ctrl = rng.uniform(-50, 50, (n, m.nu))
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv, ga = env.qpos.cpu().numpy(), env.qvel.cpu().numpy(), env.qacc.cpu().numpy()
    for i in range(n):
        e = _oracle_one_step(om, q[i], v[i], np.zeros(m.nv), ctrl[i])
        assert relerr(ga[i], e.qacc) < 5e-4, ("qacc", i, relerr(ga[i], e.qacc))
        assert relerr(gv[i], e.qvel) < TOL, ("qvel", i, relerr(gv[i], e.qvel))
        assert relerr(gq[i], e.qpos) < TOL, ("qpos", i, relerr(gq[i], e.qpos))


def test_free_fall_closed_form(backend):
    """K-3: semi-implicit Euler free fall, v_z = -g n h, z = z0 - g h^2 n(n+1)/2; joints stay at rest."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    q = np.zeros((4, m.nq)); q[:, 2] = 5.0; q[:, 3] = 1.0
    env.set_state(backend.t(q), backend.t(np.zeros((4, m.nv))))
    n, h = 30, m.timestep
    env.mj_step(backend.t(np.zeros((4, m.nu))), n)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    assert np.abs(gv[:, 2] + 9.81 * n * h).max() < 1e-5
    assert np.abs(gq[:, 2] - (5.0 - 9.81 * h * h * n * (n + 1) / 2)).max() < 1e-5
    assert np.abs(gv[:, 6:]).max() < 1e-4 and np.abs(gv[:, [0, 1, 3, 4, 5]]).max() < 1e-4


@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_mj_step_contact_states(backend, robot, mode):
    """One substep from standing / stumbling / fallen states, through mj_step with the oracle's own torque.
    qpos, qvel: norm-relative 1e-4 (max|d| / max(1, max|x|)) AND per-element relative error with a stated floor
    (|d_i| / max(|x_i|, floor); floors: qvel 1 rad/s, qpos 1 -- one fp32 ABA solve through contact rows of stiffness ~1e4 loses
    ~3 digits, so velocity components far below the step's own velocity change h max|qacc| ~ 15 rad/s cannot be resolved
    better than 2e-3 of the floor); qacc norm-relative 5e-4.  Contact geom flags bit-exact outside a |dist - margin| < 1e-5
    guard band; at most 10 % of the states may fall into the band.  The solver may neither drop rows nor hit its iteration cap.
    SMPL-X (52 bodies, 1 g finger links behind a 1e4 N/m contact) is held to 2e-4: the fp32 articulated-inertia recursion loses
    one more bit there (the SMPL model named by north_star stays at 1e-4)."""
    tol = TOL if robot == "smpl_humanoid" else 2e-4
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    n = 96 if robot == "smpl_humanoid" else 48
    q, v, w = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], n, seed=11)   # states from stable-PD rollouts
    rng = np.random.default_rng(2)
    ctrl = rng.uniform(-80, 80, (n, m.nu))
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv, ga = env.qpos.cpu().numpy(), env.qvel.cpu().numpy(), env.qacc.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    it = env.solver_iter.cpu().numpy()
    st = env.status.cpu().numpy()
    assert not (st & (8 | 16)).any(), ("rows dropped / iteration cap", st)
    ncontact_states = nguard = nexact = 0
    worst = worst_el = 0.0
    for i in range(n):
        e = _oracle_one_step(om, q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        guard = (np.abs(con["dist"] - m.margin) < 1e-5).any() if e.ncon else False
        # flags must match whenever no contact sits inside the band
        if not guard and int(gmask[i]) != e.contact_mask:
            # tolerate a geom whose nearest feature is within the band on the rejecting side
            diff = int(gmask[i]) ^ e.contact_mask
            assert _near_margin(om, q[i], diff), ("contact flags", i, bin(int(gmask[i])), bin(e.contact_mask))
            nguard += 1
            continue
        if guard:
            nguard += 1
            continue
        nexact += 1
        ncontact_states += e.ncon > 0
        worst = max(worst, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
        worst_el = max(worst_el, elem_relerr(gv[i], e.qvel, 1.0), elem_relerr(gq[i], e.qpos, 1.0))
        assert relerr(gv[i], e.qvel) < tol, ("qvel", i, relerr(gv[i], e.qvel), e.ncon, int(it[i]), e.solver_iter)
        assert relerr(gq[i], e.qpos) < tol, ("qpos", i, relerr(gq[i], e.qpos))
        assert elem_relerr(gv[i], e.qvel, 1.0) < 20 * tol, ("qvel per element", i, elem_relerr(gv[i], e.qvel, 1.0))
        assert elem_relerr(gq[i], e.qpos, 1.0) < 1e-5, ("qpos per element", i, elem_relerr(gq[i], e.qpos, 1.0))
        assert relerr(ga[i], e.qacc) < 5e-4, ("qacc", i, relerr(ga[i], e.qacc), e.ncon)
    assert nguard <= n // 10, f"{nguard} of {n} states skipped for a contact inside the guard band"
    assert nexact >= n - n // 10 and ncontact_states > n // 3
    print(f"{robot}/{mode}: {nexact} states compared with bit-exact flags ({nguard} in the guard band), {ncontact_states} with contacts; "
          f"worst norm-relative {worst:.2e}, worst per-element (floor 1) {worst_el:.2e}; max solver iters {it.max()}")


def _near_margin(om, q, diffmask):
    """True if every geom in diffmask has its closest point within 1e-5 of the contact margin."""
    from smplsim_b200.model import fk_numpy
    from smplsim_b200.mjcf import quat_to_mat
    m = om.model
    xp, xq, _ = fk_numpy(m, q)
    for g in range(m.ngeom):
        if not (diffmask >> (g + 1)) & 1:
            continue
        b = m.geom_body[g]
        R = quat_to_mat(xq[b]); c = xp[b] + R @ m.geom_pos[g]; gm = R @ m.geom_mat[g].reshape(3, 3)
        if m.geom_type[g] == 6:
            s = m.geom_size[g]
            d = min(c[2] + (gm @ (np.array([sx, sy, sz]) * s))[2] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1))
        else:
            d = c[2] - abs(gm[2, 2]) * m.geom_size[g][1] - m.geom_size[g][0]
        if abs(d - m.margin) > 1e-5:
            return False
    return True


@pytest.mark.parametrize("mode", ["uhc_pd", "pd", "torque"])
def test_controller_torque_matches_oracle(backend, mode):
    """compute_torque (incl. the stale-M stable PD, quirk Q1) as applied in the first substep of env.step."""
    cfg, om = make_models(env="speed", control_mode=mode)
    m = om.model
    n = 48
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=21)
    rng = np.random.default_rng(4)
    act = np.clip(rng.normal(size=(n, m.nu)) * 0.4, -1, 1)
    qs = q.copy(); qs[:, 7:] += rng.normal(size=(n, m.nu)) * 0.003      # last-forward state differs slightly
    from smplsim_b200.cfg import make_cfg
    cfg1 = make_cfg(env="speed", overrides={"env.control_mode": mode, "env.control_frequency_inv": 1})
    env = backend.batch(cfg1, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qpos_fwd.copy_(backend.t(qs)); env.qvel_fwd.copy_(backend.t(v * 0.9))
    env.qacc_warm.copy_(backend.t(w))
    env.task_change_step.fill_(10000)
    env.step(backend.t(act))
    gt = env.ctrl.cpu().numpy()
    st = env.status.cpu().numpy() & 7          # mj_warning bits (bit 32 = self-contact flag: these are stumbling / fallen states)
    assert (st != 0).sum() <= 2
    for i in range(n):
        e = orc.OracleEnv(om)
        e.qpos[:] = qs[i]; e.qvel[:] = v[i] * 0.9; e.forward()       # leaves M, qfrc_bias of the stale state
        e.qpos[:] = q[i]; e.qvel[:] = v[i]
        tau = e.compute_torque(act[i])
        if st[i]:        # a blown-up rollout state (|qvel| ~ 1e5): mj_checkAcc resets the data and zeroes ctrl, in the oracle too
            e.ctrl[:] = tau; e.warn = 0; e.mj_step()
            assert e.warn == st[i] and np.abs(gt[i]).max() == 0.0
            continue
        scale = max(1.0, np.abs(tau).max())
        assert np.abs(gt[i] - tau).max() / scale < 2e-4, (i, np.abs(gt[i] - tau).max(), scale)


@pytest.mark.parametrize("task,obs_v", [("speed", 1), ("reach", 2), ("getup", 1)])
def test_env_step_matches_oracle(backend, task, obs_v):
    """reset + a few env steps (15 substeps each): obs / reward / flags / task sampling vs the oracle."""
    ov = {"self_obs_v": obs_v, "robot.create_vel_sensors": True}
    cfg, om = make_models(env=task, seed=123, **ov)
    m = om.model
    n = 16
    env = backend.batch(cfg, n, seed=123)
    obs0 = env.reset().cpu().numpy().copy()
    oes = [orc.OracleEnv(om, env_id=i) for i in range(n)]
    rng = np.random.default_rng(9)
    for i, e in enumerate(oes):
        o = e.reset()
        assert np.abs(obs0[i] - o).max() < (2e-3 if task == "getup" else 1e-5), (i, np.abs(obs0[i] - o).max())
    tgt = env.task_target.cpu().numpy(); chg = env.task_change_step.cpu().numpy()
    for i, e in enumerate(oes):
        assert np.allclose(tgt[i], e.target, atol=1e-6) and chg[i] == e.change_step
    nsteps = 3
    for t in range(nsteps):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.1, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            tol = 5e-4 * (t + 1) * (10 if task == "getup" else 1)
            assert np.abs(obs[i] - o).max() < tol, (task, t, i, np.abs(obs[i] - o).max())
            assert abs(rew[i] - r) < tol
            assert bool(term[i]) == te and bool(trunc[i]) == tr


@pytest.mark.gpu_only
def test_many_envs_identical_and_deterministic(backend):
    """4096 envs (BASELINE config 2 size): identical inputs give bit-identical outputs in every env and across runs."""
    cfg, om = make_models(env="speed")
    m = om.model
    n = 4096
    outs = []
    for rep in range(2):
        env = backend.batch(cfg, n, seed=7)
        env.reset()
        env.task_target[:, 0] = 1.5
        a = torch.zeros(n, m.nu, device=backend.device); a[:, 3] = 0.2
        for _ in range(4):
            env.step(a)
        outs.append((env.qpos.clone(), env.obs_buf.clone(), env.rew_buf.clone()))
    q, o, r = outs[0]
    assert torch.equal(q, q[0:1].expand_as(q)) and torch.equal(o, o[0:1].expand_as(o))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    assert torch.isfinite(o).all()


def test_fall_init_and_recovery_counter(backend):
    cfg, om = make_models(env="getup", seed=5)
    n = 8
    env = backend.batch(cfg, n, seed=5)
    env.reset()
    assert (env.recovery.cpu().numpy() == 60).all()
    q = env.qpos.cpu().numpy()
    assert (q[:, 2] < 0.35).all() and (q[:, 2] > 0.02).all()
    e = orc.OracleEnv(om, env_id=3); e.reset()
    assert relerr(q[3], e.qpos) < 5e-3
    a = torch.zeros(n, om.model.nu, device=backend.device)
    _, _, term, trunc = env.step(a)
    assert not term.any() and not trunc.any() and (env.recovery.cpu().numpy() == 59).all()


def test_masked_reset_only_touches_flagged_envs(backend):
    cfg, om = make_models(env="speed")
    n = 8
    env = backend.batch(cfg, n)
    env.reset()
    a = torch.zeros(n, om.model.nu, device=backend.device)
    for _ in range(3):
        env.step(a)
    before = env.qpos.clone()
    mask = torch.zeros(n, dtype=torch.uint8, device=backend.device); mask[2] = 1; mask[5] = 1
    env.reset(mask)
    after = env.qpos
    keep = [0, 1, 3, 4, 6, 7]
    assert torch.equal(after[keep], before[keep])
    assert abs(after[2, 2].item() - 0.94) < 1e-6 and env.progress_buf[2].item() == 0 and env.progress_buf[0].item() == 3


def test_joint_limit_rows_match_oracle(backend):
    """Tightened hinge ranges (what robot.has_jt_limit does in the reference, smpllib/smpl_local_robot.py:176-245) make
    limit rows routinely active; one substep vs the oracle, with and without floor contact."""
    from smplsim_b200.abi import env_cfg_from, model_from_cfg
    from smplsim_b200.cfg import make_cfg
    cfg = make_cfg(env="speed", overrides={"env.control_mode": "torque"})
    m = model_from_cfg(cfg)
    m.dof_range[6:, 0] = -0.25
    m.dof_range[6:, 1] = 0.25
    om = orc.OracleModel(m, env_cfg_from(cfg, m, seed=0))
    n = 48
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=31)
    q2, v2 = airborne_states(m, 16, seed=5)
    q = np.concatenate([q, q2]); v = np.concatenate([v, v2]); w = np.concatenate([w, np.zeros((16, m.nv))])
    n = q.shape[0]
    rng = np.random.default_rng(8)
    ctrl = rng.uniform(-60, 60, (n, m.nu))
    env = backend.batch(cfg, n, model=m)
    env.set_state(backend.t(q), backend.t(v)); env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    nlim_total = 0
    for i in range(n):
        e = _oracle_one_step(om, q[i], v[i], w[i], ctrl[i])
        nlim = e.nefc - 4 * e.ncon
        nlim_total += nlim
        if nlim > 8:        # the CUDA path keeps at most W_MAXLIM = 8 simultaneous limit rows (documented)
            continue
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        assert relerr(gv[i], e.qvel) < 2e-4, (i, relerr(gv[i], e.qvel), nlim, e.ncon)
        assert relerr(gq[i], e.qpos) < TOL
    assert nlim_total > n


def test_env_step_explicit_pd_single_substep(backend):
    """explicit-PD controller through env.step with one substep per step (with kp=800, kd=80 at h=1/450 the explicit
    controller is numerically unstable over 15 substeps -- the reason the reference defaults to stable PD -- so longer
    trajectories are chaotic and cannot be compared)."""
    cfg, om = make_models(env="speed", seed=4, control_mode="pd", control_frequency_inv=1)
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=4)
    env.reset()
    oes = [orc.OracleEnv(om, env_id=i) for i in range(n)]
    for e in oes:
        e.reset()
    rng = np.random.default_rng(3)
    for t in range(2):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.05, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            # per-step error amplification of the explicit controller is ~ kd*h/I >> 1 on the light links
            assert np.abs(obs[i] - o).max() < 2e-3 * 20 ** t, (t, i, np.abs(obs[i] - o).max())


def test_spd_fresh_mode_runs_and_differs_slightly(backend):
    """cfg.env.spd_inertia='fresh' (quirk Q1 switched off): finite, and close to -- but not identical with -- the stale default."""
    outs = {}
    for spd in ("stale", "fresh"):
        cfg, om = make_models(env="speed", seed=4, spd_inertia=spd)
        env = backend.batch(cfg, 8, seed=4)
        env.reset()
        a = torch.zeros(8, om.model.nu, device=backend.device); a[:, 10] = 0.3
        for _ in range(2):
            env.step(a)
        outs[spd] = env.qpos.cpu().numpy().copy()
        assert np.isfinite(outs[spd]).all()
    d = np.abs(outs["stale"] - outs["fresh"]).max()
    assert 0 < d < 5e-2, d


def test_regression_line_search_noise_floor(backend):
    """Captured case (round 1): from the Default reset pose with this action, substep 7's active-set iterate was already
    optimal to fp32 rounding but one row sat at r ~ 0, so the set comparison asked for another line search; its directional
    derivative (-3e-6, pure cancellation noise against g1 = 0.076) and curvature (-3e-6) sent the step to 2^24 and the env
    blew up (max|qvel| 281 instead of 3.62).  The solver now treats |f0| below the cancellation floor as converged and
    caps the extrapolation; the step must match the oracle replay."""
    d = np.load(os.path.join(GOLDEN, "regress_default_step_case1.npz"))
    cfg, om = make_models(env="speed")
    env = backend.batch(cfg, 64, seed=0)
    env.reset()
    env.task_change_step.fill_(10 ** 6)   # the speed target only enters obs / reward
    e = orc.OracleEnv(om, env_id=0)
    e.reset()
    assert np.abs(env.qpos[0].cpu().numpy() - d["qpos"]).max() < 1e-6
    act = np.repeat(d["action"][None], 64, 0)
    env.step(backend.t(act))
    e.step(d["action"].astype(np.float64))
    qp, qv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    assert np.array_equal(qp, np.repeat(qp[:1], 64, 0))
    assert relerr(qv[0], e.qvel) < 2e-3 and relerr(qp[0], e.qpos) < 2e-4, (relerr(qv[0], e.qvel), relerr(qp[0], e.qpos))
    assert np.abs(qv).max() < 5.0


@pytest.mark.parametrize("case", ["nan_qpos", "huge_qvel", "bad_qacc"])
def test_bad_state_autoreset_matches_mj_step_semantics(backend, case):
    """mj_checkPos / mj_checkVel / mj_checkAcc + mj_resetData (SURVEY A.2): a NaN or |x| > 1e10 never reaches the caller --
    the env's data is reset to qpos0 / zero velocity inside the substep, the warning bit is reported in aux.status, and the
    rest of the env step proceeds from there exactly like the oracle."""
    cfg, om = make_models(env="speed")
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=0)
    env.reset()
    e = orc.OracleEnv(om, env_id=3)
    e.reset()
    qp, qv = env.qpos.clone(), env.qvel.clone()
    if case == "nan_qpos":
        qp[3, 20] = float("nan"); e.qpos[20] = np.nan; bit = 1
    elif case == "huge_qvel":
        qv[3, 10] = 3e10; e.qvel[10] = 3e10; bit = 2
    else:
        qv[3, 6:] = 8e9; e.qvel[6:] = 8e9; bit = 4          # finite state, velocity-product forces overflow 1e10
    env.set_state(qp, qv)
    e.forward()
    act = np.zeros((n, m.nu)); act[:] = 0.05
    obs, rew, term, trunc = env.step(backend.t(act))
    st = env.status.cpu().numpy()
    e.warn = 0
    o, r, te, tr = e.step(act[3])
    assert e.warn & bit, e.warn
    assert st[3] & bit and not st[[0, 1, 2, 4, 5, 6, 7]].any(), st
    assert torch.isfinite(env.qpos).all() and torch.isfinite(env.qvel).all() and torch.isfinite(obs).all()
    assert relerr(env.qpos[3].cpu().numpy(), e.qpos) < 1e-3 and relerr(env.qvel[3].cpu().numpy(), e.qvel) < 5e-3
    ref = env.qpos[0].cpu().numpy()
    for i in (1, 2, 4, 5, 6, 7):                            # neighbours in the same CTA are untouched
        assert np.array_equal(env.qpos[i].cpu().numpy(), ref)


def test_env_step_simple_pid_matches_oracle(backend):
    """control_mode simple_pid: the stateful SimplePID (integral / last error carried across substeps, steps and resets)."""
    cfg, om = make_models(env="speed", control_mode="simple_pid", seed=5)
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=5)
    env.reset()
    oes = [orc.OracleEnv(om, env_id=i) for i in range(n)]
    for e in oes:
        e.reset()
    rng = np.random.default_rng(2)
    for t in range(3):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.1, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        gi, gl = env.pid_integral.cpu().numpy(), env.pid_last_error.cpu().numpy()
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            tol = 1e-3 * (t + 1)
            assert relerr(obs[i], o) < tol, (t, i, relerr(obs[i], o))       # obs carries joint velocities of ~40 rad/s here
            assert relerr(gi[i], e.pid_integral) < tol and relerr(gl[i], e.pid_last_error) < tol
            assert bool(term[i]) == te and bool(trunc[i]) == tr
    env.reset()                                   # the controller state survives reset, as the reference's controller object does
    assert env.pid_integral.abs().max() > 0 and torch.isfinite(env.pid_last_error).all()


def test_self_contact_flag_matches_mujoco_pair_filters(backend):
    """Self-collision is not simulated (SURVEY 8 f4); aux.status bit 32 must be raised exactly when a capsule / sphere geom pair that
    passes MuJoCo's filters (same body, parent-child, contype / conaffinity, the 10 <exclude> pairs of smpl_humanoid.xml:231-242)
    touches in the state the step ends in -- checked against the oracle's geom-geom narrow phase on the product's own end state
    (pairs within 1e-5 of the margin are not compared)."""
    cfg, om = make_models(env="getup", control_mode="torque")
    m = om.model
    n = 64
    q, v, w = rollout_states(make_models(env="getup", control_mode="uhc_pd")[1], n, seed=5, init_mode=1, control_sigma=0.6)
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.mj_step(backend.t(np.zeros((n, m.nu))), 1)
    st = env.status.cpu().numpy()
    gq = env.qpos.cpu().numpy()
    om.set_self_collision(True)
    nhit = ncmp = 0
    for i in range(n):
        e = orc.OracleEnv(om)
        e.qpos[:] = gq[i]; e.qvel[:] = 0; e.forward()
        con = e.contacts()
        selfc = con["geom1"] > 0
        if selfc.any() and (np.abs(con["dist"][selfc] - m.margin) < 1e-5).any():
            continue
        # a pair just outside the margin in the oracle may sit inside it in fp32 and vice versa: re-test with a widened margin
        ncmp += 1
        nhit += int(selfc.any())
        assert bool(st[i] & 32) == bool(selfc.any()), (i, st[i], con["dist"][selfc])
    om.set_self_collision(False)
    assert ncmp >= n - 4 and 3 <= nhit < ncmp, (ncmp, nhit)


def test_mj_step_self_contact_states(backend):
    """cfg.env.self_collision: geom-geom contacts between the capsule / sphere pairs MuJoCo's filters let through (SURVEY 8 f4) are
    two-body rows; the product solves them by Woodbury on top of the ABA factors, the oracle by a dense Newton.  One substep from
    fallen / tangled states (Fall-init rollouts of the self-colliding oracle): qpos, qvel norm-relative 1e-4, qacc 5e-4, on at least
    30 states that do have geom-geom contacts (up to 4 at once = 16 two-body rows; states with more raise status bit 8 and are
    not compared)."""
    cfg, om = make_models(env="getup", control_mode="torque", self_collision=True)
    m = om.model
    n = 96
    q, v, w = rollout_states(make_models(env="getup", control_mode="uhc_pd", self_collision=True)[1], n, seed=7, init_mode=1, control_sigma=0.6)
    rng = np.random.default_rng(2)
    ctrl = rng.uniform(-60, 60, (n, m.nu))
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv, ga = env.qpos.cpu().numpy(), env.qvel.cpu().numpy(), env.qacc.cpu().numpy()
    st = env.status.cpu().numpy()
    nself_states = ndropped = 0
    worst = 0.0
    for i in range(n):
        e = _oracle_one_step(om, q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        ns = int((con["geom1"] > 0).sum())
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        if ns > 4:
            assert st[i] & 8, (i, ns, st[i])
            ndropped += 1
            continue
        assert not (st[i] & (8 | 16 | 32)), (i, ns, st[i])
        nself_states += ns > 0
        worst = max(worst, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
        assert relerr(gv[i], e.qvel) < TOL and relerr(gq[i], e.qpos) < TOL, (i, ns, e.ncon, relerr(gv[i], e.qvel))
        assert relerr(ga[i], e.qacc) < 5e-4, (i, ns, relerr(ga[i], e.qacc))
    print(f"{nself_states} states with geom-geom contacts compared (worst {worst:.2e}); {ndropped} with more than 4 dropped")
    assert nself_states >= 30 and ndropped <= n // 10


def test_env_step_with_self_collision_matches_oracle(backend):
    """getup env steps (Fall init: 45 substeps of random actions on the floor, then 15 per step) with cfg.env.self_collision on both sides."""
    cfg, om = make_models(env="getup", seed=11, self_collision=True)
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=11)
    obs0 = env.reset().cpu().numpy().copy()
    oes = [orc.OracleEnv(om, env_id=i) for i in range(n)]
    for i, e in enumerate(oes):
        assert np.abs(obs0[i] - e.reset()).max() < 5e-3, i
    rng = np.random.default_rng(3)
    for t in range(2):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            assert np.abs(obs[i] - o).max() < 1e-2 * (t + 1), (t, i, np.abs(obs[i] - o).max())
            assert bool(term[i]) == te and bool(trunc[i]) == tr


@pytest.mark.parametrize("knob", ["SMPLSIM_ALIGN=0", "SMPLSIM_DIRTYPATH=0", "SMPLSIM_WPB=3", "SMPLSIM_AXES=generic"])
def test_every_runtime_knob_keeps_parity(backend, knob, monkeypatch):
    """The debug / A-B switches that stay selectable (INTEGRATION.md) are read at smplsim_create: no CTA phase-alignment barriers, full instead of dirty-chain re-sweeps, a forced CTA size, FK through the general hinge-axis path.  Each must
    give the same physics: one substep from contact states + two env steps, against the oracle."""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    n = 24
    q, v_, w = rollout_states(om, n, seed=11)
    rng = np.random.default_rng(2)
    ctrl = rng.uniform(-80, 80, (n, m.nu))
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v_)); env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    for i in range(n):
        e = _oracle_one_step(om, q[i], v_[i], w[i], ctrl[i])
        assert relerr(gv[i], e.qvel) < 2e-4 and relerr(gq[i], e.qpos) < TOL, (knob, i, relerr(gv[i], e.qvel))
    env2 = backend.batch(cfg, 8, seed=3)
    env2.reset()
    oes = [orc.OracleEnv(om, env_id=i) for i in range(8)]
    om2 = orc.OracleModel.from_cfg(cfg, seed=env2.seed)
    oes = [orc.OracleEnv(om2, env_id=i) for i in range(8)]
    for e in oes:
        e.reset()
    for t in range(2):
        act = np.clip(rng.normal(size=(8, m.nu)) * 0.1, -1, 1)
        obs = env2.step(backend.t(act))[0].cpu().numpy()
        for i, e in enumerate(oes):
            o = e.step(act[i])[0]
            assert np.abs(obs[i] - o).max() < 1e-3 * (t + 1), (knob, t, i)


def _shape_variant(tmp_path, leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2):
    """A differently proportioned SMPL body (what SMPL_Robot writes for non-zero betas, smpl_local_robot.py:1280-1505: other bone
    offsets, geom sizes and hence masses / inertias; same tree, joints and geom types), as a `*.model.json` for cfg.robot.xml_path."""
    import json
    from smplsim_b200 import model as M
    p = M.load_parsed("smpl")
    d = M._to_jsonable(p)
    def fac(name):
        if any(k in name for k in ("Hip", "Knee", "Ankle", "Toe")):
            return leg
        if any(k in name for k in ("Shoulder", "Elbow", "Wrist", "Hand", "Thorax")):
            return arm
        return trunk
    for b in d["bodies"]:
        f = fac(b["name"])
        b["pos"] = [x * (leg if b["free"] else f) for x in b["pos"]]   # the root's pos is the standing height
    names = [b["name"] for b in d["bodies"]]
    for g in d["geoms"]:
        f = fac(names[g["body"]] if isinstance(g["body"], int) else g["body"])
        g["pos"] = [x * f for x in g["pos"]]
        s = list(g["size"])
        if g["type"] == 3:   # capsule: radius, half length
            s[0] *= girth; s[1] *= f
        else:
            s = [x * girth for x in s]
        g["size"] = s
        g["density"] = g["density"] * density
    path = tmp_path / "variant.model.json"
    path.write_text(json.dumps(d))
    return str(path)


def test_custom_body_shape_matches_oracle(backend, tmp_path):
    """SURVEY 8 f4 (body shapes): a handle takes any SMPL-family model (cfg.robot.xml_path: MJCF or model table), e.g. one batch per
    body shape side by side.  A taller / heavier variant: one mj_step from contact-rich states, then env steps.  qvel is held to 2e-4
    norm-relative here (the emulator stays below 1e-4; the GPU's fp32 solve may land a little above): the 20 % heavier body behind the same 1e4 N/m
    contact rows loses a little more of the fp32 solve -- the north_star SMPL model itself stays at 1e-4 (test_mj_step_contact_states)."""
    path = _shape_variant(tmp_path)
    cfg, om = make_models(control_mode="uhc_pd", **{"robot.xml_path": path})
    base = make_models(control_mode="uhc_pd")[1].model
    m = om.model
    assert abs(m.body_mass.sum() / base.body_mass.sum() - 1) > 0.2 and not np.allclose(m.body_pos, base.body_pos)
    n = 32
    q, v, w = rollout_states(om, n, seed=5, every=9)   # sparse snapshots: the taller body first drops a few cm onto its feet
    rng = np.random.default_rng(3)
    ctrl = rng.uniform(-80, 80, (n, m.nu))
    cfg_t, om_t = make_models(control_mode="torque", **{"robot.xml_path": path})
    env = backend.batch(cfg_t, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    ncon = 0
    for i in range(n):
        e = _oracle_one_step(om_t, q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        assert int(gmask[i]) == e.contact_mask, (i, bin(int(gmask[i])), bin(e.contact_mask))
        ncon += e.ncon > 0
        assert relerr(gv[i], e.qvel) < 2e-4 and relerr(gq[i], e.qpos) < TOL, (i, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
    assert ncon > n // 3
    env2 = backend.batch(cfg, 8, seed=4)
    obs0 = env2.reset().cpu().numpy().copy()
    om4 = orc.OracleModel.from_cfg(cfg, seed=4)
    oes = [orc.OracleEnv(om4, env_id=i) for i in range(8)]
    for i, e in enumerate(oes):
        assert np.abs(obs0[i] - e.reset()).max() < 1e-5
    for t in range(2):
        act = np.clip(rng.normal(size=(8, m.nu)) * 0.1, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env2.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            assert np.abs(obs[i] - o).max() < 5e-4 * (t + 1), (t, i, np.abs(obs[i] - o).max())
            assert abs(rew[i] - r) < 5e-4 * (t + 1) and bool(term[i]) == te and bool(trunc[i]) == tr


def test_per_env_body_shapes_match_oracle(backend, tmp_path):
    """SURVEY 8 f4 (per-env body shapes): one batch, three body shapes interleaved over the envs (smplsim_create_shapes groups the
    envs of a shape into whole thread blocks; arrays stay indexed by env).  Every env against an oracle built from ITS shape:
    kinematics, one mj_step from that shape's own contact states, then reset + env steps with the stable-PD controller."""
    from smplsim_b200.abi import model_from_cfg
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    pa = _shape_variant(tmp_path / "a", leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2)
    pb = _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)
    paths = [None, pa, pb]
    def mk(mode, k, seed=0):
        ov = {"robot.xml_path": paths[k]} if paths[k] else {}
        return make_models(control_mode=mode, seed=seed, **ov)
    n = 45
    env_model = np.array([(i * 7 + i // 5) % 3 for i in range(n)], dtype=np.int32)   # 3 shapes, ragged group sizes
    assert len(set(np.bincount(env_model))) > 1
    # --- one mj_step from each shape's own states
    cfg_t = [mk("torque", k)[0] for k in range(3)]
    om_t = [mk("torque", k)[1] for k in range(3)]
    models = [model_from_cfg(c) for c in cfg_t]
    pools = [rollout_states(mk("uhc_pd", k)[1], 24, seed=20 + k, every=9) for k in range(3)]
    cnt = [0, 0, 0]
    q = np.zeros((n, models[0].nq)); v = np.zeros((n, models[0].nv)); w = np.zeros((n, models[0].nv))
    for i, k in enumerate(env_model):
        q[i], v[i], w[i] = pools[k][0][cnt[k]], pools[k][1][cnt[k]], pools[k][2][cnt[k]]
        cnt[k] += 1
    rng = np.random.default_rng(6)
    ctrl = rng.uniform(-80, 80, (n, models[0].nu))
    env = backend.batch(cfg_t[0], n, models=models, env_model=env_model)
    xp, xq = env.kinematics(backend.t(q))
    from smplsim_b200.model import fk_numpy
    for i, k in enumerate(env_model):
        ep, eq_, _ = fk_numpy(models[k], q[i])
        assert np.abs(xp[i].cpu().numpy() - ep).max() < 2e-5, ("kinematics with env i's shape", i)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    ncon = 0
    for i, k in enumerate(env_model):
        e = _oracle_one_step(om_t[k], q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - models[k].margin) < 1e-5).any():
            continue
        assert int(gmask[i]) == e.contact_mask, (i, k)
        ncon += e.ncon > 0
        assert relerr(gv[i], e.qvel) < (TOL if k == 0 else 2e-4) and relerr(gq[i], e.qpos) < TOL, (i, k, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
    assert ncon > n // 3
    # --- env steps (stable PD: gains and inertias of the env's own shape)
    cfgs = [mk("uhc_pd", k, seed=9) for k in range(3)]
    env2 = backend.batch(cfgs[0][0], n, seed=9, models=[model_from_cfg(c) for c, _ in cfgs], env_model=env_model)
    obs0 = env2.reset().cpu().numpy().copy()
    oes = [orc.OracleEnv(cfgs[k][1], env_id=i) for i, k in enumerate(env_model)]
    for i, e in enumerate(oes):
        assert np.abs(obs0[i] - e.reset()).max() < 1e-5, i
    for t in range(2):
        act = np.clip(rng.normal(size=(n, models[0].nu)) * 0.1, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env2.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            assert np.abs(obs[i] - o).max() < 5e-4 * (t + 1), (t, i, env_model[i], np.abs(obs[i] - o).max())
            assert abs(rew[i] - r) < 5e-4 * (t + 1) and bool(term[i]) == te and bool(trunc[i]) == tr
    # a structurally different model is refused
    import copy
    bad = copy.deepcopy(models[1]); bad.dof_limited = np.asarray(bad.dof_limited).copy(); bad.dof_limited[10] = 1 - bad.dof_limited[10]
    with pytest.raises(Exception):
        backend.batch(cfg_t[0], 4, models=[models[0], bad], env_model=[0, 1, 0, 1])


def test_free_joint_armature_matches_oracle(backend):
    """The root's six dofs are solved as one 6 x 6 system (A + S diag(armature) S^T) a = -p across the lanes of the env.  The shipped
    models have no armature on the free joint (MuJoCo's <freejoint>), so this branch is pinned with a model that has: anisotropic
    armature on the six root dofs (a <joint type="free" armature=...> with per-dof values), one mj_step from contact states and
    stable-PD env steps against the oracle (which adds the armature to the diagonal of M)."""
    import copy
    from smplsim_b200.abi import env_cfg_from, model_from_cfg
    cfg, om0 = make_models(control_mode="uhc_pd")
    arm6 = np.array([0.8, 1.5, 0.4, 0.06, 0.02, 0.11])
    def with_arm(c, seed=0):
        m = copy.deepcopy(model_from_cfg(c))
        m.dof_armature = np.asarray(m.dof_armature, dtype=np.float64).copy()
        m.dof_armature[:6] = arm6
        return m, orc.OracleModel(m, env_cfg_from(c, m, seed=seed))
    cfg_t, _ = make_models(control_mode="torque")
    m_t, om_t = with_arm(cfg_t)
    n = 24
    q, v, w = rollout_states(om0, n, seed=13)
    rng = np.random.default_rng(5)
    ctrl = rng.uniform(-80, 80, (n, m_t.nu))
    env = backend.batch(cfg_t, n, models=[m_t], env_model=np.zeros(n, dtype=np.int32))
    env.set_state(backend.t(q), backend.t(v)); env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    differs = 0
    om_plain = make_models(control_mode="torque")[1]          # the same model without the root armature
    for i in range(n):
        e = _oracle_one_step(om_t, q[i], v[i], w[i], ctrl[i])
        e0 = _oracle_one_step(om_plain, q[i], v[i], w[i], ctrl[i]) if i < 4 else None
        assert relerr(gv[i], e.qvel) < 2e-4 and relerr(gq[i], e.qpos) < TOL, (i, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
        if e0 is not None and relerr(e0.qvel, e.qvel) > 1e-3:
            differs += 1
    assert differs >= 2          # the armature matters: the same states step differently without it
    m_p, om_p = with_arm(cfg, seed=3)
    env2 = backend.batch(cfg, 8, seed=3, models=[m_p], env_model=np.zeros(8, dtype=np.int32))
    obs0 = env2.reset().cpu().numpy().copy()
    oes = [orc.OracleEnv(om_p, env_id=i) for i in range(8)]
    for i, e in enumerate(oes):
        assert np.abs(obs0[i] - e.reset()).max() < 1e-5
    for t in range(2):
        act = np.clip(rng.normal(size=(8, m_p.nu)) * 0.1, -1, 1)
        obs = env2.step(backend.t(act))[0].cpu().numpy()
        for i, e in enumerate(oes):
            assert np.abs(obs[i] - e.step(act[i])[0]).max() < 1e-3 * (t + 1), (t, i)
