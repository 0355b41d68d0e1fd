"""Mass matrix, bias forces and body Jacobians (smplsim_dynamics, HumanoidBatchB200.dynamics, the single-env mj_data.qM / qfrc_bias /
get_body_jac_by_id) against the fp64 oracle.

The oracle gives M (with armature) and qfrc_bias directly.  The Jacobian reference is test-side numpy built from the model tables and
the oracle's xpos / xquat; it is pinned to the oracle by the body-origin velocities (sensor) and by M = sum_b J_b^T I_b J_b + armature.
The kernel tests run on the H100 (-m gpu) and on the host emulator build of the same kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from smplsim_b200 import _lib
from smplsim_b200.cfg import make_cfg
from util_states import airborne_states, make_models, rollout_states

# Kernel against the oracle, worst case seen in test_dynamics_matches_oracle (M relative to max|M|, the bias relative to the
# humanoid's weight, J per column relative to the column's largest entry): emulator M 1.1e-7, bias 4.7e-7, J 1.0e-6;
# H100 M 9.4e-8, bias 3.9e-7, J 9.3e-7.  TOL keeps a margin of 20x.
TOL = 2e-5
G = 9.81


def _weight(m):
    return float(np.sum(m.body_mass)) * G


def _forward(om, q, v):
    """Oracle forward pass at the fp32-rounded state (what the kernel reads)."""
    e = orc.OracleEnv(om)
    e.qpos[:] = np.float32(q); e.qvel[:] = np.float32(v)
    e.forward()
    return e


# ------------------------------------------------------------------ test-side references
def _qmul(a, b):
    w1, x1, y1, z1 = a; w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def _qmat(q):
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _dof_body(m):
    return np.array([0] * 6 + [b for b in range(1, m.nbody) for _ in range(3)])


def _ancestors(m, b):
    out = set()
    while b >= 0:
        out.add(b)
        b = int(m.body_parent[b])
    return out


def ref_jac(m, q, xpos, xquat):
    """[nbody, 6, nv]: mj_jacBody at every body's origin.  World-frame dof axes: the root's rotation columns, each hinge's axis
    after the parent's orientation, the body quaternion and the body's earlier hinges; anchors at the body origin."""
    nv = m.nv
    ax, anc = np.zeros((nv, 3)), np.zeros((nv, 3))
    R0 = _qmat(xquat[0])
    for k in range(3):
        ax[3 + k], anc[3 + k] = R0[:, k], xpos[0]
    for b in range(1, m.nbody):
        qc = _qmul(xquat[int(m.body_parent[b])], np.asarray(m.body_quat[b], dtype=np.float64))
        for k in range(3):
            d = int(m.body_dofadr[b]) + k
            a = np.asarray(m.dof_axis[d], dtype=np.float64)
            ax[d], anc[d] = _qmat(qc) @ a, xpos[b]
            h = 0.5 * q[7 + d - 6]
            qc = _qmul(qc, np.r_[np.cos(h), np.sin(h) * a])
    db = _dof_body(m)
    J = np.zeros((m.nbody, 6, nv))
    for p in range(m.nbody):
        path = _ancestors(m, p)
        for d in range(nv):
            if db[d] not in path:
                continue
            if d < 3:
                J[p, d, d] = 1.0
            else:
                J[p, 0:3, d] = np.cross(ax[d], xpos[p] - anc[d])
                J[p, 3:6, d] = ax[d]
    return J


def ref_mass(m, J, xpos, xquat):
    """sum_b J_b^T I_b J_b + diag(armature), I_b the body's spatial inertia about its origin in world axes."""
    M = np.diag(np.asarray(m.dof_armature, dtype=np.float64))
    for b in range(m.nbody):
        R = _qmat(xquat[b])
        c = R @ np.asarray(m.body_ipos[b], dtype=np.float64)
        xx, yy, zz, xy, xz, yz = np.asarray(m.body_inertia[b], dtype=np.float64)
        Ic = R @ np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]]) @ R.T
        cx = np.array([[0, -c[2], c[1]], [c[2], 0, -c[0]], [-c[1], c[0], 0]])
        Jp, Jr = J[b, :3], J[b, 3:]
        Jc = Jp - cx @ Jr                                   # velocity of the centre of mass
        M += float(m.body_mass[b]) * Jc.T @ Jc + Jr.T @ Ic @ Jr
    return M


def _states(robot, n, seed):
    """Airborne states followed by stable-PD rollout states (standing, stumbling, lying)."""
    _, om = make_models(robot=robot, control_mode="uhc_pd")
    na = max(2, n // 4)
    qa, va = airborne_states(om.model, na, seed=seed)
    qc, vc, _ = rollout_states(om, n - na, seed=seed + 1)
    return np.concatenate([qa, qc]), np.concatenate([va, vc])


# ------------------------------------------------------------------ 1. the references hold the definitions (CPU, oracle only)
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_references_match_oracle(robot):
    """jacp / jacr reproduce the oracle's body-origin velocities, and sum J^T I J + armature its M, to 1e-9."""
    _, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    q, v = _states(robot, 8, seed=3)
    rng = np.random.default_rng(0)
    for i in range(len(q)):
        vel = rng.normal(size=m.nv) * 2.0
        e = _forward(om, q[i], vel)
        J = ref_jac(m, np.float32(q[i]).astype(np.float64), e.xpos.copy(), e.xquat.copy())
        lin, ang = J[:, :3] @ e.qvel, J[:, 3:] @ e.qvel
        sens = e.sensor.copy()
        assert np.abs(lin - sens[0]).max() < 1e-9 * max(1.0, np.abs(sens[0]).max()), i
        assert np.abs(ang - sens[1]).max() < 1e-9 * max(1.0, np.abs(sens[1]).max()), i
        Mr = ref_mass(m, J, e.xpos.copy(), e.xquat.copy())
        assert np.abs(Mr - e.M).max() < 1e-9 * np.abs(e.M).max(), i


# ------------------------------------------------------------------ 2. kernel against the oracle
def _check(m, om, q, v, out, tag):
    """Worst (M, bias, J) errors of kernel rows `out` against the oracle; also the structural properties of M and J."""
    wt, nb = _weight(m), m.nbody
    db = _dof_body(m)
    anc = np.array([[int(a in _ancestors(m, b)) for a in range(nb)] for b in range(nb)])
    pattern = (anc[db][:, db] + anc[db][:, db].T) > 0        # dof pairs where one is an ancestor of the other
    Mk = out["qM"].cpu().numpy()
    bk = out["qfrc_bias"].cpu().numpy().astype(np.float64)
    Jk = torch.cat([out["jacp"], out["jacr"]], dim=2).cpu().numpy()
    worst = np.zeros(3)
    for i in range(len(q)):
        e = _forward(om, q[i], v[i])
        M = Mk[i]
        assert np.array_equal(M, M.T) and np.all(M[~pattern] == 0.0), (tag, i)
        np.linalg.cholesky(M.astype(np.float64))
        em = np.abs(M - e.M).max() / np.abs(e.M).max()
        eb = np.abs(bk[i] - e.qfrc_bias).max() / max(wt, float(np.abs(e.qfrc_bias).max()))
        Jr = ref_jac(m, np.float32(q[i]).astype(np.float64), e.xpos.copy(), e.xquat.copy())
        for p in range(nb):
            off = anc[p][db] == 0
            assert np.all(Jk[i, p][:, off] == 0.0), (tag, i, p)
        scale = np.abs(Jr).max(axis=1)                       # [nbody, nv]: the largest entry of each reference column
        ej = float((np.abs(Jk[i] - Jr).max(axis=1)[scale > 0] / scale[scale > 0]).max())
        assert max(em, eb, ej) <= TOL, (tag, i, em, eb, ej)
        worst = np.maximum(worst, [em, eb, ej])
    return worst


@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_dynamics_matches_oracle(backend, robot, mode):
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    n = 24 if robot == "smpl_humanoid" else 10
    q, v = _states(robot, n, seed=11)
    env = backend.batch(cfg, 8)
    out = env.dynamics(backend.t(q), backend.t(v), jac_bodies=list(range(m.nbody)))
    worst = _check(m, om, q, v, out, robot)
    print(f"{robot} {mode}: worst M {worst[0]:.2e}, bias {worst[1]:.2e}, J {worst[2]:.2e}")


def test_world_body_jacobian_is_zero(backend):
    from smplsim_b200.envs import HumanoidSpeed
    cfg = make_cfg(env="speed", seed=4)

    class Env(HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    env = Env(cfg, device=backend.device)
    env.reset()
    nv = env.mj_model.nv
    jp, jr = np.ones((3, nv)), np.ones((3 * nv,))
    r = env.get_body_jac_by_id(0, jp, jr)
    assert r[0] is jp and r[1] is jr and not jp.any() and not jr.any()
    jp, jr = env.get_body_jac_by_id(0)
    assert jp.shape == (3, nv) and not jp.any() and not jr.any()


# ------------------------------------------------------------------ 4. consistency with the inverse
def test_inverse_is_M_a_plus_bias(backend):
    """Airborne, no rows (oracle nefc == 0): inverse(q, v, a) = M a + qfrc_bias for random a."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v = airborne_states(m, 8, seed=3)
    q[:, 7:] *= 0.2                                                    # inside the joint ranges
    a = np.random.default_rng(1).normal(size=v.shape) * 5.0
    env = backend.batch(cfg, 8)
    tq, tv, ta = backend.t(q), backend.t(v), backend.t(a)
    out = env.dynamics(tq, tv)
    inv = env.inverse(tq, tv, ta).cpu().numpy().astype(np.float64)
    M, b = out["qM"].cpu().numpy().astype(np.float64), out["qfrc_bias"].cpu().numpy().astype(np.float64)
    for i in range(len(q)):
        assert _forward(om, q[i], v[i]).nefc == 0
        want = M[i] @ np.float32(a[i]) + b[i]
        assert np.abs(inv[i] - want).max() / max(_weight(m), float(np.abs(want).max())) < 1e-5, i


# ------------------------------------------------------------------ 5. plumbing
def test_chunking_and_single_outputs(backend):
    """n = 2.5 num_envs equals three separate calls bit for bit; each output alone equals the all-outputs call bit for bit."""
    cfg, om = make_models(control_mode="uhc_pd")
    q, v = _states("smpl_humanoid", 20, seed=31)
    env = backend.batch(cfg, 8)
    jb = [0, "L_Hand", 18, 4, 4]
    tq, tv = backend.t(q), backend.t(v)
    full = env.dynamics(tq, tv, jac_bodies=jb)
    assert full["jacp"].shape == (20, 5, 3, om.model.nv) and full["jacp"].data_ptr() + 3 * om.model.nv * 4 == full["jacr"].data_ptr()
    for s in (slice(0, 8), slice(8, 16), slice(16, 20)):
        part = env.dynamics(backend.t(q[s]), backend.t(v[s]), jac_bodies=jb)
        for k in full:
            assert torch.equal(part[k], full[k][s]), k
    only = [env.dynamics(tq, tv, bias=False), env.dynamics(tq, tv, mass_matrix=False), env.dynamics(tq, mass_matrix=False, bias=False, jac_bodies=jb)]
    assert set(only[0]) == {"qM"} and set(only[1]) == {"qfrc_bias"} and set(only[2]) == {"jacp", "jacr"}
    for o in only:
        for k in o:
            assert torch.equal(o[k], full[k]), k
    e0 = env.dynamics(backend.t(np.zeros((0, om.model.nq))), backend.t(np.zeros((0, om.model.nv))), jac_bodies=[1])
    assert e0["qM"].shape == (0, om.model.nv, om.model.nv) and e0["jacr"].shape == (0, 1, 3, om.model.nv)


def test_per_env_shapes(backend, tmp_path):
    """Three body shapes interleaved: every row against the oracle of its own shape; n != num_envs is refused."""
    from smplsim_b200.abi import model_from_cfg
    from test_gpu_parity import _shape_variant
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a", leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2),
             _shape_variant(tmp_path / "b", leg=0.9, arm=1.1, trunk=0.95, girth=0.9, density=0.9)]
    mk = [make_models(control_mode="torque", **({"robot.xml_path": p} if p else {})) for p in paths]
    n = 12
    env_model = np.array([i % 3 for i in range(n)], dtype=np.int32)
    q, v = _states("smpl_humanoid", n, seed=17)
    env = backend.batch(mk[0][0], n, models=[model_from_cfg(c) for c, _ in mk], env_model=env_model)
    nb = mk[0][1].model.nbody
    out = env.dynamics(backend.t(q), backend.t(v), jac_bodies=list(range(nb)))
    for k in range(3):
        rows = np.nonzero(env_model == k)[0]
        _check(mk[k][1].model, mk[k][1], q[rows], v[rows], {key: t[rows] for key, t in out.items()}, f"shape {k}")
    with pytest.raises(_lib.SmplsimError, match="num_envs"):
        env.dynamics(backend.t(q[:4]), backend.t(v[:4]))


def test_self_collision_handle(backend):
    cfg, _ = make_models(env="getup", control_mode="torque", self_collision=True)
    _, om = make_models(control_mode="torque")
    q, v = _states("smpl_humanoid", 8, seed=5)
    env = backend.batch(cfg, 4)
    out = env.dynamics(backend.t(q), backend.t(v), jac_bodies=list(range(om.model.nbody)))
    _check(om.model, om, q, v, out, "self_collision")


def test_arguments(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    q, v = airborne_states(m, 4, seed=1)
    tq, tv = backend.t(q), backend.t(v)
    for bad in (dict(qpos=tq[:, :-1], qvel=tv), dict(qpos=tq, qvel=tv[:3])):
        with pytest.raises(ValueError, match="shape"):
            env.dynamics(**bad)
    with pytest.raises(ValueError, match="float32"):
        env.dynamics(tq, tv.double())
    with pytest.raises(ValueError, match="live on"):
        env.dynamics(tq, tv.to("meta"))
    with pytest.raises(ValueError, match="needs qvel"):
        env.dynamics(tq)
    for jb in ([m.nbody], [-1], ["no_such_body"], [1.0]):
        with pytest.raises(ValueError):
            env.dynamics(tq, tv, jac_bodies=jb)
    L, p = env._L(), lambda t: C.c_void_p(t.data_ptr())
    M, b, J = backend.t(np.zeros((4, m.nv, m.nv))), backend.t(np.zeros((4, m.nv))), backend.t(np.zeros((4, 2, 6, m.nv)))
    ok = (C.c_int32 * 2)(0, m.nbody - 1)
    bad = (C.c_int32 * 2)(0, m.nbody)
    s = env._stream()
    assert L.smplsim_dynamics(env._h, p(tq), p(tv), 4, p(M), p(b), ok, 2, p(J), s) == 0
    assert L.smplsim_dynamics(env._h, p(tq), p(tv), 4, None, None, bad, 2, p(J), s) == -1          # body index
    assert L.smplsim_dynamics(env._h, p(tq), p(tv), 4, None, None, ok, 2, None, s) == -1           # njac > 0 without jac
    assert L.smplsim_dynamics(env._h, p(tq), None, 4, p(M), p(b), None, 0, None, s) == -1          # bias without qvel
    assert L.smplsim_dynamics(env._h, p(tq), p(tv), 4, None, None, None, 0, None, s) == -1         # no output
    assert L.smplsim_dynamics(env._h, p(tq), p(tv), -1, p(M), None, None, 0, None, s) == -1
    assert L.smplsim_dynamics(None, p(tq), p(tv), 4, p(M), None, None, 0, None, s) == -1
    assert L.smplsim_dynamics(env._h, p(tq), None, 4, p(M), None, None, 0, None, s) == 0            # M without qvel


# ------------------------------------------------------------------ 5b. no effect on the stepper
def test_dynamics_leaves_the_stepper_alone(backend):
    """step -> dynamics -> step and step -> step from the same state: every output and every state row bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_dyn in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_dyn and t == 0:     # every scratch row of the handle
                qq = env.qpos.repeat(3, 1)[: 2 * n + n // 2]
                qq[:, 7:] += torch.as_tensor(rin.normal(size=(qq.shape[0], m.nu)) * 0.5, dtype=torch.float32, device=qq.device)
                vv = torch.as_tensor(rin.normal(size=(qq.shape[0], m.nv)), dtype=torch.float32, device=qq.device)
                env.dynamics(qq, vv, jac_bodies=[0, 5, 23])
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


# ------------------------------------------------------------------ 6. single-env surface (B1)
def _b1_env(backend, **ov):
    from smplsim_b200.envs import HumanoidSpeed
    cfg = make_cfg(env="speed", seed=4, overrides={f"env.{k}": x for k, x in ov.items()})

    class Env(HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    return Env(cfg, device=backend.device)


def test_mj_data_qM_and_velocities(backend):
    from smplsim_b200.envs import mj_fullM
    env = _b1_env(backend)
    env.reset()
    rng = np.random.default_rng(3)
    for _ in range(2):
        env.step(np.clip(rng.normal(size=env.get_action_size()) * 0.3, -1, 1).astype(np.float32))
    mm, d = env.mj_model, env.mj_data
    assert mm.nM == 1221 and len(d.qM) == mm.nM and mm.dof_Madr[-1] < mm.nM and mm.dof_parentid[0] == -1
    M = np.zeros((mm.nv, mm.nv))
    mj_fullM(mm, M, d.qM)
    b = env._b
    want = b.dynamics(b.qpos_fwd, b.qvel_fwd)
    assert np.array_equal(M, want["qM"][0].cpu().numpy().astype(np.float64))
    assert np.array_equal(d.qfrc_bias, want["qfrc_bias"][0].cpu().numpy().astype(np.float64))
    qvel = env.get_qvel()
    for name in ("Pelvis", "L_Hand", "Head"):
        jp = np.zeros((3, mm.nv)); jr = np.zeros((3, mm.nv))
        env.get_body_jac_by_id(env.mj_body_names.index(name), jp, jr)
        assert np.array_equal(env.get_body_jacp_by_name(name), jp)
        assert np.allclose(env.get_body_xvelp(name), jp @ qvel, rtol=0, atol=1e-12)
        assert np.allclose(env.get_body_xvelr(name), jr @ qvel, rtol=0, atol=1e-12)


def test_stable_pd_from_mj_data(backend):
    """controllers.py:142-190 (StablePDController._compute_torque + the clip of control()) fed from env.mj_data with mj_fullM
    reproduces the torque the kernel applies in the next step (control_frequency_inv = 1: one substep per env step)."""
    from scipy.linalg import cho_factor, cho_solve
    from smplsim_b200.envs import mj_fullM
    env = _b1_env(backend, control_frequency_inv=1, control_mode="uhc_pd")
    env.reset()
    mm = env.mj_model
    nv, dt = mm.nv, mm.opt.timestep
    rng = np.random.default_rng(5)
    ncmp = 0
    for t in range(6):
        act = np.clip(rng.normal(size=env.get_action_size()) * 0.5, -1, 1).astype(np.float32)
        d = env.mj_data
        qpos, qvel = d.qpos.copy(), d.qvel.copy()
        setpoint = act * env._pd_action_scale + env._pd_action_offset
        k_p, k_d = np.zeros(nv), np.zeros(nv)
        k_p[6:], k_d[6:] = env.jkp, env.jkd
        qpos_err = np.concatenate((np.zeros(6), qpos[7:] + qvel[6:] * dt - setpoint))
        qvel_err = qvel
        M = np.zeros((nv, nv))
        mj_fullM(mm, M, d.qM)
        Cb = d.qfrc_bias.copy()
        K_p, K_d = np.diag(k_p), np.diag(k_d)
        q_accel = cho_solve(cho_factor(M + K_d * dt), -Cb[:, None] - K_p.dot(qpos_err[:, None]) - K_d.dot(qvel_err[:, None])).squeeze()
        qvel_err = qvel_err + q_accel * dt
        torque = np.clip(-env.jkp * qpos_err[6:] - env.jkd * qvel_err[6:], -env.torque_lim, env.torque_lim)
        _, _, died, timed_out, _ = env.step(act)
        if died or timed_out:
            break
        got = env._b.ctrl[0].cpu().numpy().astype(np.float64)
        assert np.abs(got - torque).max() / max(1.0, float(np.abs(torque).max())) < 2e-3, t
        ncmp += 1
    assert ncmp >= 3
