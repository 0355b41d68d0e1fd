"""Known-answer tests of the fp64 wrench oracle (tests/xfrc_oracle.c): mj_data.xfrc_applied as MuJoCo's mj_xfrcAccumulate applies it."""
import copy

import numpy as np

from oracle import oracle as orc
from smplsim_b200.mjcf import quat_to_mat
from smplsim_b200.model import fk_numpy
from test_oracle_witness import _integrate
from util_states import airborne_states, make_models, relerr, rollout_states
from xfrc_oracle import XfrcOracleEnv


def _com_frames(m, q):
    xp, xq, _ = fk_numpy(m, q)
    R = np.array([quat_to_mat(x) for x in xq])
    return xp + np.einsum("bij,bj->bi", R, np.asarray(m.body_ipos)), R


def _numeric_qfrc(m, q, xfrc, eps=1e-6):
    """sum_b Jp_b(xipos_b)^T f_b + Jr_b^T t_b with the Jacobians as central differences of each body's COM position and orientation."""
    out = np.zeros(m.nv)
    for i in range(m.nv):
        dq = np.zeros(m.nv); dq[i] = 1.0
        cp, Rp = _com_frames(m, _integrate(m, q, dq, eps))
        cm, Rm = _com_frames(m, _integrate(m, q, dq, -eps))
        jp = (cp - cm) / (2 * eps)
        W = np.einsum("bij,bkj->bik", Rp, Rm)          # R(+eps) R(-eps)^T = exp(2 eps [w]x)
        jr = np.stack([W[:, 2, 1] - W[:, 1, 2], W[:, 0, 2] - W[:, 2, 0], W[:, 1, 0] - W[:, 0, 1]], axis=1) / (4 * eps)
        out[i] = np.sum(jp * xfrc[:, :3]) + np.sum(jr * xfrc[:, 3:])
    return out


def _wrench(m, rng, fscale=2.0, tscale=20.0):
    mass = np.asarray(m.body_mass)[:, None]
    f = rng.uniform(-1, 1, (m.nbody, 3)) * fscale * 9.81 * mass
    return np.concatenate([f, rng.uniform(-1, 1, (m.nbody, 3)) * tscale], axis=1)


def test_qfrc_applied_is_jacobian_transpose_of_the_wrench():
    """Witness: on the contact states of test_oracle_witness.py and random wrenches, qfrc_applied equals J^T w with numerical
    Jacobians (1e-7 relative)."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], 40, seed=17, every=4)
    rng = np.random.default_rng(1)
    for i in range(len(q)):
        e = XfrcOracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]
        e.xfrc_applied[:] = _wrench(m, rng)
        e.forward()
        ref = _numeric_qfrc(m, e.qpos.copy(), e.xfrc_applied)
        assert np.abs(e.qfrc_applied - ref).max() <= 1e-7 * np.abs(ref).max(), (i, np.abs(e.qfrc_applied - ref).max())


def _gravity_off(om):
    m2 = copy.deepcopy(om.model)
    m2.gravity = np.zeros(3)
    return orc.OracleModel(m2, om.envcfg)


def test_gravity_compensation():
    """f_b = -m_b g on every body cancels gravity: at rest |qacc| < 1e-9; moving, qacc equals that of the model without gravity."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    om0 = _gravity_off(om)
    g = np.asarray(m.gravity)
    xf = np.zeros((m.nbody, 6)); xf[:, :3] = -np.asarray(m.body_mass)[:, None] * g[None, :]
    q, v = airborne_states(m, 12, seed=8)
    q[:, 7:] *= 0.1                      # inside the joint ranges: no limit rows
    for i in range(len(q)):
        e = XfrcOracleEnv(om)
        e.qpos[:] = q[i]; e.xfrc_applied[:] = xf
        e.forward()
        assert e.nefc == 0 and np.abs(e.qacc).max() < 1e-9, (i, e.nefc, np.abs(e.qacc).max())
        e.qvel[:] = v[i]
        e.forward()
        z = orc.OracleEnv(om0)
        z.qpos[:] = q[i]; z.qvel[:] = v[i]
        z.forward()
        assert relerr(e.qacc, z.qacc) < 1e-9, (i, relerr(e.qacc, z.qacc))


def test_wrench_leaves_qfrc_bias_and_stable_pd_torque_alone():
    """The wrench enters qfrc_smooth, not qfrc_bias: the stable-PD torque (which reads qfrc_bias, quirk Q1) is identical with and
    without it, while qacc changes."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q, v, w = rollout_states(om, 12, seed=5)
    rng = np.random.default_rng(2)
    for i in range(len(q)):
        a = np.clip(rng.normal(size=m.nu) * 0.3, -1, 1)
        es = []
        for xf in (np.zeros((m.nbody, 6)), _wrench(m, rng)):
            e = XfrcOracleEnv(om)
            e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]; e.xfrc_applied[:] = xf
            e.forward()
            es.append((e.qfrc_bias.copy(), e.compute_torque(a), e.qacc.copy()))
        assert np.array_equal(es[0][0], es[1][0]) and np.array_equal(es[0][1], es[1][1])
        assert np.abs(es[0][2] - es[1][2]).max() > 1e-3


def test_zero_wrench_is_the_oracle_bit_for_bit():
    cfg, om = make_models(control_mode="uhc_pd")
    q, v, w = rollout_states(om, 6, seed=9)
    for i in range(len(q)):
        e, o = XfrcOracleEnv(om), orc.OracleEnv(om)
        for x in (e, o):
            x.qpos[:] = q[i]; x.qvel[:] = v[i]; x.qacc_warm[:] = w[i]
            x.mj_step()
        assert np.array_equal(e.qpos, o.qpos) and np.array_equal(e.qvel, o.qvel) and np.array_equal(e.qacc, o.qacc)


def test_auto_reset_clears_the_wrench():
    """mj_checkVel (huge qvel) resets the data: the wrench is zeroed with it and the substep runs as the plain oracle's."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    e, o = XfrcOracleEnv(om), orc.OracleEnv(om)
    for x in (e, o):
        x.qpos[2] = 1.5
        x.qvel[10] = 3e10
    e.xfrc_applied[:] = _wrench(m, np.random.default_rng(3))
    e.mj_step(); o.mj_step()
    assert e.warn & 2 and o.warn & 2
    assert not e.xfrc_applied.any()
    assert np.array_equal(e.qpos, o.qpos) and np.array_equal(e.qvel, o.qvel)
