"""Per-env physics parameters (HumanoidBatchB200.set_env_params): friction, gravity, controller gains / torque limits and body mass
scales per env.  The reference for env e is the fp64 oracle of the model with those fields replaced (dataclasses.replace of the
nominal ModelDesc: masses and inertias scaled, gains, friction and gravity replaced, invweight0 and the mean inertia left as they are,
which is MuJoCo's behaviour for in-place MjModel edits without mj_setConst).  Every kernel test runs on the GPU and on the emulator."""
import ctypes
import dataclasses
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import oracle as orc
from smplsim_b200.abi import env_cfg_from, model_from_cfg
from util_states import make_models, relerr, rollout_states

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
TOL = 1e-4


def draw(m, n, seed, gain=0.4):
    """Independent draws per env, float32 (the values the kernels see; the oracle takes the same numbers in fp64): friction
    U(0.4, 1.6), gains and torque limits x U(1 - gain, 1 + gain), mass scales U(0.7, 1.3), gravity + U(-0.5, 0.5)."""
    rng = np.random.default_rng(seed)
    g = lambda: rng.uniform(1 - gain, 1 + gain, (n, m.nu))  # noqa: E731
    P = {"friction": rng.uniform(0.4, 1.6, n), "gravity": m.gravity + rng.uniform(-0.5, 0.5, (n, 3)),
         "kp": m.act_kp * g(), "kd": m.act_kd * g(), "torque_limit": m.act_torque_lim * g(),
         "body_mass_scale": rng.uniform(0.7, 1.3, (n, m.nbody))}
    return {k: v.astype(np.float32) for k, v in P.items()}


def variant(m, P, e):
    s = P["body_mass_scale"][e].astype(np.float64)
    fr = np.array(m.friction, dtype=np.float64).copy()
    fr[0] = P["friction"][e]
    return dataclasses.replace(m, body_mass=m.body_mass * s, body_inertia=m.body_inertia * s[:, None], friction=fr,
                               gravity=P["gravity"][e].astype(np.float64), act_kp=P["kp"][e].astype(np.float64),
                               act_kd=P["kd"][e].astype(np.float64), act_torque_lim=P["torque_limit"][e].astype(np.float64))


def oracle_for(cfg, m, P, e, seed=0, self_collision=False):
    """fp64 oracle of env e's variant model; the mean inertia stays the nominal model's (no mj_setConst)."""
    om = orc.OracleModel(variant(m, P, e), env_cfg_from(cfg, m, seed=seed))
    M0, _ = orc.mass_matrix_numpy(m, m.qpos0)
    orc.lib().orc_set_meaninertia(om.ptr, float(np.mean(np.diag(M0))))
    if self_collision:
        om.set_self_collision(True)
    return om


def set_all(env, backend, P, env_ids=None):
    env.set_env_params(env_ids, **{k: backend.t(v) for k, v in P.items()})


def one_step(om, q, v, w, ctrl):
    e = orc.OracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w; e.ctrl[:] = ctrl
    e.mj_step()
    return e


def check_mj_step(backend, cfg, n, seed, robot="smpl_humanoid", self_collision=False, contact_wrench=False, models=None, env_model=None,
                  min_con=None):
    """One mj_step (torque-mode handle: raw ctrl) from states of a stable-PD rollout, every env with its own draws."""
    m = model_from_cfg(cfg) if models is None else models[0]
    q, v, w = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], n, seed=seed, every=9)
    rng = np.random.default_rng(seed + 1)
    ctrl = rng.uniform(-80, 80, (n, m.nu))
    kw = dict(contact_wrench=contact_wrench)
    if models is not None:
        kw.update(models=models, env_model=env_model)
    env = backend.batch(cfg, n, **kw)
    P = draw(m, n, seed + 2)
    set_all(env, backend, P)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    cw = env.contact_wrench.cpu().numpy() if contact_wrench else None
    ncon, worst = 0, 0.0
    for i in range(n):
        mi = m if models is None else models[env_model[i]]
        e = one_step(oracle_for(cfg, mi, P, i, self_collision=self_collision), q[i], v[i], w[i], ctrl[i])
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue   # a contact on the margin: the float32 and fp64 passes may disagree on it
        assert int(gmask[i]) == e.contact_mask, i
        ncon += e.ncon > 0
        worst = max(worst, relerr(gv[i], e.qvel))
        assert relerr(gv[i], e.qvel) < 2e-4 and relerr(gq[i], e.qpos) < TOL, (i, relerr(gv[i], e.qvel), relerr(gq[i], e.qpos))
        if contact_wrench:   # against a one-env batch of env i's variant model without records
            one = backend.batch(cfg, 1, contact_wrench=True, model=variant(mi, P, i))
            one.set_state(backend.t(q[i:i + 1]), backend.t(v[i:i + 1]))
            one.qacc_warm.copy_(backend.t(w[i:i + 1]))
            one.mj_step(backend.t(ctrl[i:i + 1]), 1)
            ref = one.contact_wrench[0].cpu().numpy()
            scale = max(1.0, float(np.abs(ref).max()))
            assert np.abs(cw[i] - ref).max() / scale < 1e-3, (i, np.abs(cw[i] - ref).max())
    assert ncon >= (min_con if min_con is not None else max(2, n // 8)), ncon
    return env, P


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_mj_step_matches_variant_oracle(backend, robot):
    """One mj_step from contact-rich states, every env with its own friction, gravity and mass scales, against its variant oracle."""
    cfg, _ = make_models(robot=robot, control_mode="torque")
    check_mj_step(backend, cfg, 32 if robot == "smpl_humanoid" else 16, seed=40, robot=robot)


# The explicit pd controller runs one substep per env step, with the error growth per step of test_gpu_parity's explicit-pd test: at
# its shipped gains it is unstable over 15 substeps, and the oracle and the kernels part within one env step even without records.
# With one substep the stable-PD Fall init is three controlled substeps, so the reset kernel's gravity, gains and masses are held to a
# tight bound there.  Fall init with simple_pid (45 substeps on the floor) parts like the explicit pd and is not compared; the
# controllers' torques themselves, with the clamp, are compared in test_controller_torque_matches_variant_oracle.
@pytest.mark.parametrize("mode,init,nsub", [("uhc_pd", 0, 15), ("simple_pid", 0, 15), ("uhc_pd", 1, 15), ("uhc_pd", 1, 1), ("pd", 0, 1)])
def test_env_steps_match_variant_oracle(backend, mode, init, nsub):
    """reset (Default / Fall init: the Fall init runs the controller for three env steps) and two env steps under every controller
    (torque mode: the per-env torque limit is the clamp), against per-env oracles with the env's gains, torque limits, masses,
    friction and gravity."""
    cfg, om = make_models(control_mode=mode, seed=5, state_init=["Default", "Fall"][init], control_frequency_inv=nsub)
    m = om.model
    n = 6
    env = backend.batch(cfg, n, seed=5)
    P = draw(m, n, 70 + init)
    # Fall init: 45 substeps of random actions on the floor before the first observation, where float32 and fp64 trajectories part
    # (the oracle tests of the Fall init hold 5e-3 / 1e-2 per step with nominal parameters)
    tol0, tol = (1e-4, 1e-3) if init == 0 else (1e-3, 1e-3) if nsub == 1 else (5e-2, 5e-2)
    grow = 20 if mode == "pd" else 1   # explicit pd: error amplification per step ~ kd h / I on the light links
    set_all(env, backend, P)
    obs0 = env.reset(init_mode=init).cpu().numpy().copy()
    oes = [orc.OracleEnv(oracle_for(cfg, m, P, i, seed=env.seed), env_id=i) for i in range(n)]
    for i, e in enumerate(oes):
        assert np.abs(obs0[i] - e.reset(init)).max() < tol0, i
    rng = np.random.default_rng(3)
    for t in range(2):
        act = np.clip(rng.normal(size=(n, m.nu)) * (0.05 if mode == "pd" else 0.1), -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            o, r, te, tr = e.step(act[i])
            assert np.abs(obs[i] - o).max() < tol * (t + 1) * grow ** t, (t, i, np.abs(obs[i] - o).max())
            assert abs(rew[i] - r) < tol * (t + 1) * grow ** t and bool(term[i]) == te and bool(trunc[i]) == tr, (t, i)


@pytest.mark.parametrize("mode", ["uhc_pd", "pd", "torque"])
def test_controller_torque_matches_variant_oracle(backend, mode):
    """The torque each controller applies in the first substep of an env step (aux ctrl), with per-env gains and torque limits low
    enough that the clamp acts, against the variant oracle's compute_torque (stale-M stable PD: the env's kd and masses on both
    sides of quirk Q1)."""
    from smplsim_b200.cfg import make_cfg
    cfg, om = make_models(env="speed", control_mode=mode)
    m = om.model
    n = 24
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=21)
    rng = np.random.default_rng(4)
    act = np.clip(rng.normal(size=(n, m.nu)) * 0.4, -1, 1)
    qs = q.copy(); qs[:, 7:] += rng.normal(size=(n, m.nu)) * 0.003      # last-forward state differs slightly
    P = draw(m, n, 31)
    P["torque_limit"] = (m.act_torque_lim * rng.uniform(0.02, 0.1, (n, m.nu))).astype(np.float32)   # 20-100 Nm: the clamp acts
    cfg1 = make_cfg(env="speed", overrides={"env.control_mode": mode, "env.control_frequency_inv": 1})
    env = backend.batch(cfg1, n)
    set_all(env, backend, P)
    env.set_state(backend.t(q), backend.t(v))
    env.qpos_fwd.copy_(backend.t(qs)); env.qvel_fwd.copy_(backend.t(v * 0.9))
    env.qacc_warm.copy_(backend.t(w))
    env.task_change_step.fill_(10000)
    env.step(backend.t(act))
    gt = env.ctrl.cpu().numpy()
    st = env.status.cpu().numpy() & 7
    clamped = 0
    for i in range(n):
        if st[i]:
            continue   # a blown-up rollout state: mj_checkAcc resets the data and zeroes ctrl
        e = orc.OracleEnv(oracle_for(cfg, m, P, i))
        e.qpos[:] = qs[i]; e.qvel[:] = v[i] * 0.9; e.forward()
        e.qpos[:] = q[i]; e.qvel[:] = v[i]
        tau = e.compute_torque(act[i])
        clamped += int((np.abs(np.abs(tau) - P["torque_limit"][i]) < 1e-3).sum())
        scale = max(1.0, np.abs(tau).max())
        assert np.abs(gt[i] - tau).max() / scale < 2e-4, (i, np.abs(gt[i] - tau).max(), scale)
    assert (st != 0).sum() <= 2 and clamped > n


def test_params_compose_with_per_env_shapes(backend, tmp_path):
    """Per-env body shapes plus records: the mass scale multiplies env e's own shape."""
    from test_gpu_parity import _shape_variant
    (tmp_path / "a").mkdir()
    pa = _shape_variant(tmp_path / "a", leg=1.15, arm=0.9, trunk=1.05, girth=1.1, density=1.15)
    cfg0, _ = make_models(control_mode="torque")
    cfg1, _ = make_models(control_mode="torque", **{"robot.xml_path": pa})
    models = [model_from_cfg(cfg0), model_from_cfg(cfg1)]
    n = 20
    env_model = np.array([(i * 3) % 2 for i in range(n)], dtype=np.int32)
    check_mj_step(backend, cfg0, n, seed=50, models=models, env_model=env_model, min_con=n // 4)


def test_params_with_self_collision_and_contact_wrench(backend):
    """A self-collision handle with records (friction enters the geom-geom rows too) and the per-body contact wrench output."""
    cfg, _ = make_models(control_mode="torque", self_collision=True)
    check_mj_step(backend, cfg, 16, seed=60, self_collision=True, min_con=3)
    cfg2, _ = make_models(control_mode="torque")
    check_mj_step(backend, cfg2, 16, seed=61, contact_wrench=True, min_con=3)


def _variant_batch(backend, cfg, m, P, i):
    return backend.batch(cfg, 1, model=variant(m, P, i))


def test_dynamics_and_inverse_match_variant_models(backend):
    """qM, qfrc_bias, body Jacobians and qfrc_inverse with records against one-env batches built from each env's variant model (no
    records).  n != num_envs is rejected while records exist."""
    cfg, _ = make_models(control_mode="torque")
    m = model_from_cfg(cfg)
    n = 6
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=80, every=7)
    qacc = np.random.default_rng(1).normal(size=(n, m.nv)) * 3.0
    env = backend.batch(cfg, n)
    P = draw(m, n, 81)
    set_all(env, backend, P)
    d = env.dynamics(backend.t(q), backend.t(v), jac_bodies=[0, 5, m.nbody - 1])
    inv = env.inverse(backend.t(q), backend.t(v), backend.t(qacc)).cpu().numpy()
    for i in range(n):
        ref = _variant_batch(backend, cfg, m, P, i)
        dr = ref.dynamics(backend.t(q[i:i + 1]), backend.t(v[i:i + 1]), jac_bodies=[0, 5, m.nbody - 1])
        M, Mr = d["qM"][i].cpu().numpy(), dr["qM"][0].cpu().numpy()
        assert np.abs(M - Mr).max() / np.abs(Mr).max() < 2e-5, i
        wt = float(np.sum(m.body_mass * P["body_mass_scale"][i]) * 9.81)
        assert np.abs(d["qfrc_bias"][i].cpu().numpy() - dr["qfrc_bias"][0].cpu().numpy()).max() / wt < 2e-5, i
        assert np.abs(d["jacp"][i].cpu().numpy() - dr["jacp"][0].cpu().numpy()).max() < 2e-5, i
        ir = ref.inverse(backend.t(q[i:i + 1]), backend.t(v[i:i + 1]), backend.t(qacc[i:i + 1])).cpu().numpy()[0]
        assert np.abs(inv[i] - ir).max() / max(1.0, np.abs(ir).max()) < 2e-5, (i, np.abs(inv[i] - ir).max())
    # the masses and gravity do change M and the bias
    nom = backend.batch(cfg, n).dynamics(backend.t(q), backend.t(v))
    assert np.abs(nom["qM"].cpu().numpy() - d["qM"].cpu().numpy()).max() > 1e-2
    from smplsim_b200._lib import SmplsimError
    with pytest.raises(SmplsimError):
        env.dynamics(backend.t(q[:2]), backend.t(v[:2]))
    with pytest.raises(SmplsimError):
        env.inverse(backend.t(q[:2]), backend.t(v[:2]), backend.t(qacc[:2]))


def test_trackcom_camera_follows_mass_scaled_com(backend):
    """A TRACKCOM camera with records sits at the mass-scaled robot COM (numpy) + its offset: the image equals a FIXED camera there."""
    from smplsim_b200 import camera as cam
    cfg, _ = make_models(control_mode="torque")
    m = model_from_cfg(cfg)
    n = 4
    q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=90, every=11)
    env = backend.batch(cfg, n)
    P = draw(m, n, 91)
    P["body_mass_scale"][:, 0] = 3.0   # a heavy pelvis moves the COM visibly
    set_all(env, backend, P)
    xp, xq = env.kinematics(backend.t(q))
    mat = cam.xyaxes_mat((1, 0, 0, 0, 0, 1))   # looking along +y
    off = np.array([0.0, -3.0, 0.5])
    tc = cam.Camera(cam.TRACKCOM, off, mat, fovy=45.0)
    img = env.render(tc, 48, 32, depth=True, rgb=False, xpos=xp, xquat=xq)["depth"].cpu().numpy()
    from smplsim_b200.model import fk_numpy
    for i in range(n):
        xpos, xquat = fk_numpy(m, q[i])[:2]
        w_, x_, y_, z_ = np.asarray(xquat, dtype=np.float64).reshape(m.nbody, 4).T
        R = np.stack([1 - 2 * (y_ * y_ + z_ * z_), 2 * (x_ * y_ - w_ * z_), 2 * (x_ * z_ + w_ * y_),
                      2 * (x_ * y_ + w_ * z_), 1 - 2 * (x_ * x_ + z_ * z_), 2 * (y_ * z_ - w_ * x_),
                      2 * (x_ * z_ - w_ * y_), 2 * (y_ * z_ + w_ * x_), 1 - 2 * (x_ * x_ + y_ * y_)], 1).reshape(m.nbody, 3, 3)
        ms = m.body_mass * P["body_mass_scale"][i].astype(np.float64)
        com = (ms[:, None] * (np.asarray(xpos) + np.einsum("bij,bj->bi", R, m.body_ipos))).sum(0) / ms.sum()
        fx = cam.Camera(cam.FIXED, com + off, mat, fovy=45.0)
        ref = env.render(fx, 48, 32, depth=True, rgb=False, xpos=xp[i:i + 1], xquat=xq[i:i + 1])["depth"].cpu().numpy()[0]
        close = np.abs(img[i] - ref) < 1e-3
        assert close.mean() > 0.97, (i, close.mean())
    nom = backend.batch(cfg, n).render(tc, 48, 32, depth=True, rgb=False, xpos=xp, xquat=xq)["depth"].cpu().numpy()
    assert (np.abs(nom - img) > 1e-3).any()


def _same(a, b):
    """Rollouts equal bit for bit."""
    return all(np.array_equal(u, v) for x, y in zip(a, b) for u, v in zip(x, y))


def _roll(backend, env, steps, seed=7):
    rng = np.random.default_rng(seed)
    out = []
    env.reset()
    for _ in range(steps):
        act = np.clip(rng.normal(size=(env.num_envs, env.num_actions)) * 0.3, -1, 1)
        o, r, te, tr = env.step(backend.t(act))
        out.append([x.cpu().numpy().copy() for x in (env.qpos, env.qvel, o, r, env.contact_mask)])
    return out


def test_nominal_records_mask_readback_and_clear(backend):
    """Records holding the model's values give bit-identical results to a batch without records; a masked set changes only the
    masked envs; env_params reads back what was set; after clear_env_params the stateless calls match a batch that never had records."""
    import torch
    cfg, _ = make_models(control_mode="uhc_pd", seed=2)
    n = 6
    ref = _roll(backend, backend.batch(cfg, n, seed=2), 3)
    env = backend.batch(cfg, n, seed=2)
    nominal = env.env_params
    m = env.model
    assert np.allclose(nominal["kp"].cpu().numpy(), m.act_kp.astype(np.float32)[None])
    assert (nominal["body_mass_scale"].cpu().numpy() == 1.0).all()
    env.set_env_params(**nominal)
    got_nom = _roll(backend, env, 3)
    # bit-identical on the GPU.  The host emulator's compiler contracts the two instances' arithmetic into FMAs differently, and its
    # 1e-7 differences grow over 45 contact-rich substeps; there one substep from contact states is held to 1e-6 instead (below).
    if backend.name == "gpu":
        assert _same(ref, got_nom)
    else:
        q, v, w = rollout_states(make_models(control_mode="uhc_pd")[1], n, seed=12, every=9)
        ctrl = np.random.default_rng(13).uniform(-80, 80, (n, m.nu))
        outs = []
        for rec in (False, True):
            b = backend.batch(make_models(control_mode="torque")[0], n)
            if rec:
                b.set_env_params(**b.env_params)
            b.set_state(backend.t(q), backend.t(v)); b.qacc_warm.copy_(backend.t(w)); b.mj_step(backend.t(ctrl), 1)
            outs.append((b.qpos.cpu().numpy(), b.qvel.cpu().numpy(), b.contact_mask.cpu().numpy()))
        assert np.array_equal(outs[0][2], outs[1][2])
        assert relerr(outs[1][0], outs[0][0]) < 1e-6 and relerr(outs[1][1], outs[0][1]) < 1e-6, (relerr(outs[1][0], outs[0][0]), relerr(outs[1][1], outs[0][1]))
    # masked set: only envs 1 and 4 change
    P = draw(m, n, 5)
    mask = np.zeros(n, dtype=bool); mask[[1, 4]] = True
    env.set_env_params(backend.t(np.array([1, 4]), dtype=__import__("torch").int64), friction=backend.t(P["friction"]),
                       kp=backend.t(P["kp"]))
    rb = env.env_params
    for k in ("friction", "kp"):
        exp = np.where(mask.reshape((n,) + (1,) * (P[k].ndim - 1)), P[k], nominal[k].cpu().numpy())
        assert np.array_equal(rb[k].cpu().numpy(), exp), k
    for k in ("gravity", "kd", "torque_limit", "body_mass_scale"):
        assert np.array_equal(rb[k].cpu().numpy(), nominal[k].cpu().numpy()), k
    got = _roll(backend, env, 3)
    for i in range(n):
        same = all(np.array_equal(a[0][i], b[0][i]) for a, b in zip(got_nom, got))
        assert same == (not mask[i]), i
    # cleared: the stateless calls give what a batch that never had records gives, bit for bit (a rollout would not: the env's task
    # random stream and working-set memory have moved on)
    env.clear_env_params()
    fresh = backend.batch(cfg, n, seed=2)
    q, v = env.qpos.clone(), env.qvel.clone()
    a_ = torch.zeros_like(v)
    for x, y in ((env.dynamics(q, v, jac_bodies=[3]), fresh.dynamics(q, v, jac_bodies=[3])),
                 ({"inv": env.inverse(q, v, a_)}, {"inv": fresh.inverse(q, v, a_)})):
        for k in x:
            assert np.array_equal(x[k].cpu().numpy(), y[k].cpu().numpy()), k
    xp, xq = env.kinematics(q)
    from smplsim_b200 import camera as cam
    tc = cam.Camera(cam.TRACKCOM, np.array([0.0, -3.0, 0.5]), cam.xyaxes_mat((1, 0, 0, 0, 0, 1)), fovy=45.0)
    assert np.array_equal(env.render(tc, 16, 8, depth=True, rgb=False, xpos=xp, xquat=xq)["depth"].cpu().numpy(),
                          fresh.render(tc, 16, 8, depth=True, rgb=False, xpos=xp, xquat=xq)["depth"].cpu().numpy())


def test_argument_errors(backend):
    import torch
    cfg, _ = make_models(control_mode="pd")
    n = 4
    env = backend.batch(cfg, n)
    m = env.model
    good = {k: backend.t(v) for k, v in draw(m, n, 1).items()}
    for k, t in good.items():
        with pytest.raises(ValueError):
            env.set_env_params(**{k: t[:-1]})                       # shape
        with pytest.raises(ValueError):
            env.set_env_params(**{k: t.double()})                   # dtype
        with pytest.raises(ValueError):
            env.set_env_params(**{k: t.cpu().numpy()})              # not a tensor
        bad = t.clone(); bad.view(-1)[0] = float("nan")
        with pytest.raises(ValueError):
            env.set_env_params(**{k: bad})                          # non-finite
    for k, v in (("friction", 1e-6), ("kp", -1.0), ("kd", -1.0), ("torque_limit", 0.0), ("body_mass_scale", 0.0)):
        bad = good[k].clone(); bad.view(-1)[-1] = v
        with pytest.raises(ValueError):
            env.set_env_params(**{k: bad})
        env.set_env_params(torch.tensor([0], device=bad.device), **{k: bad})   # the bad row is not selected: accepted
    if backend.name == "gpu":
        with pytest.raises(ValueError):
            env.set_env_params(friction=good["friction"].cpu())     # device


def test_ctypes_struct_matches_header():
    from smplsim_b200.abi import SmplsimEnvParamsC
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "smplsim.h"\nint main(){printf("%zu %zu %zu\\n", sizeof(SmplsimEnvParams), '
           'offsetof(SmplsimEnvParams, torque_limit), offsetof(SmplsimEnvParams, body_mass_scale));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    assert got == [ctypes.sizeof(SmplsimEnvParamsC), SmplsimEnvParamsC.torque_limit.offset, SmplsimEnvParamsC.body_mass_scale.offset]
