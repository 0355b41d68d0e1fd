"""Per-body contact wrenches (aux.contact_wrench, HumanoidBatchB200(contact_wrench=True)) against a reference built from the fp64 oracle.

The reference is test-side: the oracle's contact list (point, frame, geoms), its constraint forces (joint-limit rows first, then four
pyramid rows per contact) and the forward pass's body poses.  Row b = [F ; t]: the world-frame force the contacts apply to body b and
its torque about the body's centre of mass (xipos), the convention of xfrc_applied.  The kernel tests run on the H100 (-m gpu) and on
the host emulator build of the same kernels."""
import numpy as np
import pytest

from oracle import oracle as orc
from smplsim_b200.cfg import make_cfg
from util_states import airborne_states, make_models, rollout_states
from xfrc_oracle import XfrcOracleEnv

# per-env max |kernel - reference| over the [nbody, 6] block, in units of the humanoid's weight m_total g, or of the env's largest
# reference component where that is larger (deeply interpenetrating self-collision states carry ~2e6 N, where fp32 rounding alone is
# a few N).  Worst case seen over the states below: 1.2e-4 on the emulator (self-collision states), 1.5e-4 on an H100 (SMPL floor
# contacts); TOL keeps a margin above 10x.
TOL = 2e-3
G = 9.81


def _rot(q, v):
    """Rotate v [.., 3] by the unit quaternions q [.., 4] (w, x, y, z)."""
    w, u = q[..., :1], q[..., 1:]
    t = 2.0 * np.cross(u, v)
    return v + w * t + np.cross(u, t)


def ref_wrench(m, con, force, xpos, xquat):
    """[nbody, 6] reference wrench from an oracle forward pass: con = OracleEnv.contacts(), force = its efc force rows past the
    joint-limit rows ([ncon, 4]), xpos / xquat the body poses of that pass."""
    gb = np.asarray(m.geom_body)
    mu = float(np.asarray(m.friction)[0])
    xipos = xpos + _rot(xquat, np.asarray(m.body_ipos, dtype=np.float64))
    out = np.zeros((m.nbody, 6))
    for c in range(len(con["geom"])):
        n, t1, t2 = con["frame"][c]
        f = force[c]
        F = f[0] * (n + mu * t1) + f[1] * (n - mu * t1) + f[2] * (n + mu * t2) + f[3] * (n - mu * t2)
        p = con["pos"][c]
        for g, sg in ((con["geom"][c], 1.0), (con["geom1"][c], -1.0)):
            if g <= 0:              # 0: the floor
                continue
            b = gb[g - 1]
            out[b, :3] += sg * F
            out[b, 3:] += sg * np.cross(p - xipos[b], F)
    return out


def oracle_wrench(e, xpos=None, xquat=None):
    """ref_wrench of the oracle env's last forward pass (poses: its own xpos / xquat unless given)."""
    con = e.contacts()
    nc = len(con["geom"])
    nlim = e.nefc - 4 * nc
    force = e.efc()["force"][nlim:].reshape(nc, 4)
    return ref_wrench(e.m, con, force, e.xpos.copy() if xpos is None else xpos, e.xquat.copy() if xquat is None else xquat)


def _weight(m):
    return float(np.sum(m.body_mass)) * G


def _guard_band(e):
    con = e.contacts()
    return e.ncon > 0 and bool((np.abs(con["dist"] - e.m.margin) < 1e-5).any())


def _self_states(n, seed=7):
    cfg, om = make_models(env="getup", control_mode="torque", self_collision=True)
    q, v, w = rollout_states(make_models(env="getup", control_mode="uhc_pd", self_collision=True)[1], n, seed=seed, init_mode=1,
                             control_sigma=0.6)
    return cfg, om, q, v, w


# ------------------------------------------------------------------ 1. the reference holds the definition (CPU, oracle only)
@pytest.mark.parametrize("kind", ["rollout", "self_collision", "airborne"])
def test_reference_wrench_reproduces_contact_forces(kind):
    """J^T of the reference wrench (through the wrench oracle's qfrc_applied) equals qfrc_constraint without the joint-limit rows."""
    if kind == "self_collision":
        _, om, q, v, w = _self_states(24, seed=3)
    else:
        _, om = make_models(control_mode="torque")
        if kind == "rollout":
            q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], 48, seed=5)
        else:
            q, v = airborne_states(om.model, 8, seed=2)
            w = np.zeros_like(v)
    m = om.model
    rng = np.random.default_rng(1)
    nself = ncontact = 0
    for i in range(len(q)):
        e = XfrcOracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]; e.ctrl[:] = rng.uniform(-50, 50, m.nu)
        e.forward()
        W = oracle_wrench(e)
        con = e.contacts()
        nself += int((con["geom1"] > 0).sum() > 0)
        ncontact += e.ncon > 0
        if kind == "airborne":
            assert e.ncon == 0 and np.all(W == 0.0), i
            continue
        efc = e.efc()
        nlim = e.nefc - 4 * e.ncon
        want = e.qfrc_constraint - efc["J"][:nlim].T @ efc["force"][:nlim]
        e2 = XfrcOracleEnv(om)
        e2.qpos[:] = q[i]; e2.qvel[:] = v[i]; e2.xfrc_applied[:] = W
        e2.forward()
        scale = max(1.0, float(np.abs(e.qfrc_constraint).max()))
        assert np.abs(e2.qfrc_applied - want).max() / scale < 1e-9, (i, np.abs(e2.qfrc_applied - want).max(), scale)
        # the free joint's translational dofs are world-frame: their constraint force is the total contact force
        assert np.abs(W[:, :3].sum(0) - e.qfrc_constraint[:3]).max() / scale < 1e-9
    if kind == "rollout":
        assert ncontact >= len(q) // 4
    if kind == "self_collision":
        assert nself >= 4


# ------------------------------------------------------------------ kernel against the reference
def _mj_step_compare(backend, cfg, om, q, v, w, ctrl, xf=None, nsub=1, skip_guard=True):
    """mj_step(ctrl, nsub) on the batch with contact_wrench=True; per env the reference of the oracle's last forward pass (stepped
    nsub - 1 times, then forward() with the same ctrl).  Returns (kernel wrench, list of (i, oracle env) compared, worst error)."""
    m = om.model
    n = len(q)
    env = backend.batch(cfg, n, contact_wrench=True)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    if xf is not None:
        env.xfrc_applied = backend.t(xf)
    env.mj_step(backend.t(ctrl), nsub)
    gw = env.contact_wrench.cpu().numpy().astype(np.float64)
    st = env.status.cpu().numpy()
    assert gw.shape == (n, m.nbody, 6)
    wt = _weight(m)
    worst, done = 0.0, []
    for i in range(n):
        e = XfrcOracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]; e.ctrl[:] = ctrl[i]
        if xf is not None:
            e.xfrc_applied[:] = xf[i]
        for _ in range(nsub - 1):
            e.mj_step()
        e.forward()
        if (skip_guard and _guard_band(e)) or st[i] & (1 | 2 | 4 | 8 | 16):
            continue
        ref = oracle_wrench(e)
        if e.ncon == 0:
            assert np.all(gw[i] == 0.0), ("airborne env with a nonzero wrench", i)
        scale = max(wt, float(np.abs(ref).max()))
        err = np.abs(gw[i] - ref).max() / scale
        assert err < TOL, (i, err, e.ncon, np.abs(gw[i] - ref).max(axis=1))
        # sum of the contact forces: the free joint's translational constraint force (world frame)
        assert np.abs(gw[i, :, :3].sum(0) - e.qfrc_constraint[:3]).max() / scale < TOL, (i, gw[i, :, :3].sum(0), e.qfrc_constraint[:3])
        worst = max(worst, err)
        done.append((i, e))
    return gw, done, worst


@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_mj_step_contact_wrench_matches_reference(backend, robot, mode):
    """One mj_step from airborne states and stable-PD rollout contact states, a random xfrc_applied on half of them."""
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    na = 8
    qa, va = airborne_states(m, na, seed=4)
    nc = 48 if robot == "smpl_humanoid" else 24
    qc, vc, wc = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], nc, seed=11)
    q = np.concatenate([qa, qc]); v = np.concatenate([va, vc]); w = np.concatenate([np.zeros((na, m.nv)), wc])
    n = len(q)
    rng = np.random.default_rng(7)
    ctrl = rng.uniform(-50, 50, (n, m.nu))
    mass = np.asarray(m.body_mass)[None, :, None]
    xf = np.concatenate([rng.uniform(-1, 1, (n, m.nbody, 3)) * 9.81 * mass, rng.uniform(-1, 1, (n, m.nbody, 3)) * 5.0], axis=2)
    xf[::2] = 0.0
    gw, done, worst = _mj_step_compare(backend, cfg, om, q, v, w, ctrl, xf)
    ncontact = sum(e.ncon > 0 for _, e in done)
    print(f"{len(done)} envs compared ({ncontact} with contacts), worst {worst:.2e}")
    assert len(done) >= n - n // 10 and ncontact > nc // 2
    assert all(np.all(gw[i] == 0.0) for i in range(na))


def test_contact_wrench_is_the_last_substeps(backend):
    """mj_step(ctrl, nsub=5): the wrench is the one of the fifth forward pass (oracle stepped four times, then forward())."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], 48, seed=13)
    ctrl = np.random.default_rng(3).uniform(-30, 30, (len(q), m.nu))
    gw, done, worst = _mj_step_compare(backend, cfg, om, q, v, w, ctrl, nsub=5)
    print(f"{len(done)} envs compared ({sum(e.ncon > 0 for _, e in done)} with contacts), worst {worst:.2e}")
    assert len(done) >= 40 and sum(e.ncon > 0 for _, e in done) >= 8
    # not the first forward pass: at least one env's wrench moved by more than the tolerance over the call
    e1 = [oracle_wrench(_forward(om, q[i], v[i], w[i], ctrl[i])) for i, _ in done]
    assert max(np.abs(gw[i] - r).max() for (i, _), r in zip(done, e1)) / _weight(m) > 10 * TOL


def _forward(om, q, v, w, ctrl):
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w; e.ctrl[:] = ctrl
    e.forward()
    return e


def test_self_collision_contact_wrench_matches_reference(backend):
    """cfg.env.self_collision: fallen / tangled states; each geom-geom contact puts equal and opposite wrenches on its two bodies."""
    cfg, om, q, v, w = _self_states(48)
    m = om.model
    ctrl = np.random.default_rng(2).uniform(-60, 60, (len(q), m.nu))
    gw, done, worst = _mj_step_compare(backend, cfg, om, q, v, w, ctrl)
    nself = sum(int((e.contacts()["geom1"] > 0).any()) for _, e in done)
    print(f"{len(done)} envs compared, {nself} with geom-geom contacts, worst {worst:.2e}")
    assert nself >= 8 and len(done) >= len(q) - len(q) // 5


def test_env_step_contact_wrench_matches_reference(backend):
    """Full env step (speed task, stable PD) with control_frequency_inv = 1: the last forward pass is at the input state."""
    cfg, om = make_models(control_mode="uhc_pd", control_frequency_inv=1)
    m = om.model
    n = 32
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=21)
    act = np.clip(np.random.default_rng(4).normal(size=(n, m.nu)) * 0.4, -1, 1)
    env = backend.batch(cfg, n, contact_wrench=True)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.task_change_step.fill_(10000)
    env.step(backend.t(act))
    gw = env.contact_wrench.cpu().numpy().astype(np.float64)
    st = env.status.cpu().numpy()
    wt = _weight(m)
    ncmp = 0
    for i in range(n):
        e = orc.OracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.forward()        # the stable-PD torque reads M / qfrc_bias of this state
        e.qacc_warm[:] = w[i]; e.change_step = 10000
        k = orc.OracleEnv(om)
        k.qpos[:] = q[i]; k.kinematics()                        # body poses of the forward pass (the env step ends on mj_kinematics)
        e.step(act[i])
        if _guard_band(e) or st[i] & 7:
            continue
        err = np.abs(gw[i] - oracle_wrench(e, k.xpos.copy(), k.xquat.copy())).max() / wt
        assert err < TOL, (i, err, e.ncon)
        ncmp += e.ncon > 0
    assert ncmp >= n // 4


def test_reading_the_wrench_changes_nothing(backend):
    """Env steps (15 substeps) with contact_wrench on and off: obs, reward, flags and state bit-identical; airborne envs read zeros."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for on in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=on)
        env.reset()
        q = env.qpos.clone(); q[::4, 2] += 3.0                  # every fourth env starts 3 m up
        env.set_state(q, env.qvel.clone())
        rng = np.random.default_rng(1)
        rows = []
        for t in range(3):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status)]
        res.append(rows)
        if on:
            cw = env.contact_wrench.cpu().numpy()
            assert np.all(cw[::4] == 0.0)
            assert cw[:, :, 2].sum(1).max() > 0.3 * _weight(m)      # feet on the floor carry (a good part of) the weight
        else:
            assert env.contact_wrench is None
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_reset_zeroes_the_rows_of_reset_envs(backend):
    cfg, om = make_models(env="speed", seed=2)
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=2, contact_wrench=True, with_aux=False)
    env.reset()
    assert np.all(env.contact_wrench.cpu().numpy() == 0.0)
    rng = np.random.default_rng(0)
    for _ in range(2):
        env.step(backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.1, -1, 1)))
    before = env.contact_wrench.cpu().numpy().copy()
    touching = np.abs(before).reshape(n, -1).max(1) > 0
    assert touching.sum() >= n // 2
    mask = np.zeros(n, dtype=np.uint8); mask[np.flatnonzero(touching)[:3]] = 1
    env.reset(backend.t(mask, dtype=__import__("torch").uint8))
    after = env.contact_wrench.cpu().numpy()
    assert np.all(after[mask == 1] == 0.0)
    assert np.array_equal(after[mask == 0], before[mask == 0])


def test_per_env_shapes_contact_wrench_match_each_shape(backend, tmp_path):
    """A per-env-shapes handle: each env's wrench against a reference built from its own body shape."""
    from smplsim_b200.abi import model_from_cfg
    from test_gpu_parity import _shape_variant
    pa = _shape_variant(tmp_path, leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2)
    mk = [make_models(control_mode="torque"), make_models(control_mode="torque", **{"robot.xml_path": pa})]
    models = [model_from_cfg(c) for c, _ in mk]
    n = 24
    env_model = np.array([(i * 5) % 3 % 2 for i in range(n)], dtype=np.int32)
    states = [rollout_states(make_models(control_mode="uhc_pd", **({"robot.xml_path": pa} if k else {}))[1], n, seed=17, every=7)
              for k in range(2)]
    q = np.stack([states[k][0][i] for i, k in enumerate(env_model)])
    v = np.stack([states[k][1][i] for i, k in enumerate(env_model)])
    w = np.stack([states[k][2][i] for i, k in enumerate(env_model)])
    ctrl = np.random.default_rng(8).uniform(-50, 50, (n, models[0].nu))
    env = backend.batch(mk[0][0], n, models=models, env_model=env_model, contact_wrench=True)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gw = env.contact_wrench.cpu().numpy().astype(np.float64)
    ncmp = 0
    for i, k in enumerate(env_model):
        om = mk[k][1]
        e = orc.OracleEnv(om)
        e.qpos[:] = q[i]; e.qvel[:] = v[i]; e.qacc_warm[:] = w[i]; e.ctrl[:] = ctrl[i]
        e.mj_step()
        if _guard_band(e):
            continue
        err = np.abs(gw[i] - oracle_wrench(e)).max() / _weight(om.model)
        assert err < TOL, (i, k, err)
        ncmp += e.ncon > 0
    assert ncmp >= n // 4


def test_contact_wrench_off_by_default(backend):
    cfg, _ = make_models(env="speed")
    env = backend.batch(cfg, 2)
    assert env.contact_wrench is None and env._aux.contact_wrench is None
