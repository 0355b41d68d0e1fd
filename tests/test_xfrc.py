"""External body wrenches (mj_data.xfrc_applied) through the step kernel against the fp64 wrench oracle (tests/xfrc_oracle.c).
Each test runs on the H100 (-m gpu) and on the host emulator build of the same kernels."""
import numpy as np
import pytest

from oracle import oracle as orc
from smplsim_b200.cfg import make_cfg
from util_states import airborne_states, make_models, relerr, rollout_states
from xfrc_oracle import XfrcOracleEnv

TOL = 1e-4


def _wrenches(m, n, rng, fscale=2.0, tscale=20.0):
    """[n, nbody, 6]: forces up to fscale m_b g, torques up to tscale N m, on every body."""
    mass = np.asarray(m.body_mass)[None, :, None]
    f = rng.uniform(-1, 1, (n, m.nbody, 3)) * fscale * 9.81 * mass
    return np.concatenate([f, rng.uniform(-1, 1, (n, m.nbody, 3)) * tscale], axis=2)


def _oracle_step(om, q, v, w, ctrl, xf):
    e = XfrcOracleEnv(om)
    e.qpos[:] = q; e.qvel[:] = v; e.qacc_warm[:] = w; e.ctrl[:] = ctrl; e.xfrc_applied[:] = xf
    e.mj_step()
    return e


@pytest.mark.parametrize("robot,mode", [("smpl_humanoid", "torque"), ("smpl_humanoid", "uhc_pd"), ("smplx_humanoid", "torque")])
def test_mj_step_with_wrench_matches_oracle(backend, robot, mode):
    """One mj_step with a wrench on every body, from airborne states and from stable-PD rollout contact states.  Tolerances as
    test_mj_step_airborne / test_mj_step_contact_states: qpos / qvel 1e-4 norm-relative (SMPL-X 2e-4), qacc 5e-4, contact flags
    bit-exact outside the |dist - margin| < 1e-5 guard band."""
    tol = TOL if robot == "smpl_humanoid" else 2e-4
    cfg, om = make_models(robot=robot, control_mode=mode)
    m = om.model
    na = 16
    qa, va = airborne_states(m, na, seed=4)
    nc = 48 if robot == "smpl_humanoid" else 24
    qc, vc, wc = rollout_states(make_models(robot=robot, control_mode="uhc_pd")[1], nc, seed=11)
    q = np.concatenate([qa, qc]); v = np.concatenate([va, vc]); w = np.concatenate([np.zeros((na, m.nv)), wc])
    n = len(q)
    rng = np.random.default_rng(7)
    ctrl = rng.uniform(-50, 50, (n, m.nu))
    xf = _wrenches(m, n, rng)
    env = backend.batch(cfg, n)
    env.set_state(backend.t(q), backend.t(v))
    env.qacc_warm.copy_(backend.t(w))
    env.xfrc_applied = backend.t(xf)
    env.mj_step(backend.t(ctrl), 1)
    gq, gv, ga = env.qpos.cpu().numpy(), env.qvel.cpu().numpy(), env.qacc.cpu().numpy()
    gmask = env.contact_mask.cpu().numpy().astype(np.uint64)
    st = env.status.cpu().numpy()
    assert not (st & (8 | 16)).any(), ("rows dropped / iteration cap", st)
    nexact = ncontact = 0
    for i in range(n):
        e = _oracle_step(om, q[i], v[i], w[i], ctrl[i], xf[i])
        con = e.contacts()
        if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
            continue
        assert int(gmask[i]) == e.contact_mask, ("contact flags", i)
        nexact += 1
        ncontact += e.ncon > 0
        assert relerr(gv[i], e.qvel) < tol, ("qvel", i, relerr(gv[i], e.qvel), e.ncon)
        assert relerr(gq[i], e.qpos) < tol, ("qpos", i, relerr(gq[i], e.qpos))
        assert relerr(ga[i], e.qacc) < 5e-4, ("qacc", i, relerr(ga[i], e.qacc), e.ncon)
    assert nexact >= n - n // 10 and ncontact > nc // 3
    # the wrench mattered: the same step without it lands elsewhere
    e0 = orc.OracleEnv(om)
    e0.qpos[:] = q[0]; e0.qvel[:] = v[0]; e0.ctrl[:] = ctrl[0]
    e0.mj_step()
    assert relerr(gv[0], e0.qvel) > 100 * tol


def test_env_step_with_wrench_on_some_envs_matches_oracle(backend):
    """speed task, uhc_pd, 15 substeps: a wrench on half the envs (zero rows for the others, in the same batch), held over every
    substep; tolerances as test_env_step_matches_oracle."""
    cfg, om = make_models(env="speed", seed=123)
    m = om.model
    n = 16
    env = backend.batch(cfg, n, seed=123)
    env.reset()
    oes = [XfrcOracleEnv(om, env_id=i) for i in range(n)]
    for e in oes:
        e.reset()
    rng = np.random.default_rng(9)
    xf = _wrenches(m, n, rng, fscale=0.5, tscale=5.0)
    xf[::2] = 0.0
    xf[1::2, 0, :3] += [150.0, -80.0, 0.0]          # a push on the pelvis
    env.xfrc_applied = backend.t(xf)
    for t in range(3):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.1, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            e.xfrc_applied[:] = xf[i]
            o, r, te, tr = e.step(act[i])
            tol = 5e-4 * (t + 1)
            assert np.abs(obs[i] - o).max() < tol, (t, i, np.abs(obs[i] - o).max())
            assert abs(rew[i] - r) < tol
            assert bool(term[i]) == te and bool(trunc[i]) == tr
    assert np.array_equal(env.xfrc_applied.cpu().numpy(), backend.t(xf).cpu().numpy())      # the caller's tensor is never written


def test_env_step_with_wrench_and_self_collision_matches_oracle(backend):
    """getup with self-collision on fallen states (Fall init), a wrench on some envs; tolerances as
    test_env_step_with_self_collision_matches_oracle."""
    cfg, om = make_models(env="getup", seed=11, self_collision=True)
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=11)
    env.reset()
    oes = [XfrcOracleEnv(om, env_id=i) for i in range(n)]
    for e in oes:
        e.reset()
    rng = np.random.default_rng(3)
    xf = _wrenches(m, n, rng, fscale=0.5, tscale=5.0)
    xf[[0, 3, 4]] = 0.0
    env.xfrc_applied = backend.t(xf)
    for t in range(2):
        act = np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1)
        obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
        for i, e in enumerate(oes):
            e.xfrc_applied[:] = xf[i]
            o, r, te, tr = e.step(act[i])
            assert np.abs(obs[i] - o).max() < 1e-2 * (t + 1), (t, i, np.abs(obs[i] - o).max())
            assert bool(term[i]) == te and bool(trunc[i]) == tr


def test_stable_pd_torque_does_not_see_the_wrench(backend):
    """control_frequency_inv = 1, uhc_pd: the torque of the step (aux ctrl) is the same with and without a wrench, the velocity is not."""
    cfg = make_cfg(env="speed", overrides={"env.control_frequency_inv": 1})
    _, om = make_models(control_mode="uhc_pd")
    m = om.model
    n = 8
    q, v, w = rollout_states(om, n, seed=21)
    act = np.clip(np.random.default_rng(4).normal(size=(n, m.nu)) * 0.4, -1, 1)
    out = []
    for xf in (None, _wrenches(m, n, np.random.default_rng(5))):
        env = backend.batch(cfg, n)
        env.set_state(backend.t(q), backend.t(v))
        env.qacc_warm.copy_(backend.t(w))
        env.task_change_step.fill_(10000)
        env.xfrc_applied = None if xf is None else backend.t(xf)
        env.step(backend.t(act))
        out.append((env.ctrl.cpu().numpy().copy(), env.qvel.cpu().numpy().copy()))
    assert np.array_equal(out[0][0], out[1][0])
    assert np.abs(out[0][1] - out[1][1]).max() > 1e-2


def test_zero_wrench_equals_no_wrench(backend):
    """None and an all-zero tensor: identical obs, reward, flags and state, bit for bit (the wrench instance adds exact zeros)."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for zero in (False, True):
        env = backend.batch(cfg, n, seed=5)
        env.reset()
        if zero:
            env.xfrc_applied = backend.t(np.zeros((n, m.nbody, 6)))
        rng = np.random.default_rng(1)
        rows = []
        for t in range(3):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_reset_ignores_the_wrench(backend):
    """Fall init (45 substeps of random actions) gives the same state with a wrench set as without."""
    cfg, om = make_models(env="getup", seed=2)
    m = om.model
    n = 8
    res = []
    for xf in (None, _wrenches(m, n, np.random.default_rng(0))):
        env = backend.batch(cfg, n, seed=2)
        env.xfrc_applied = None if xf is None else backend.t(xf)
        obs = env.reset().cpu().numpy().copy()
        res.append((obs, env.qpos.cpu().numpy().copy(), env.qvel.cpu().numpy().copy()))
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_per_env_shapes_with_wrench_match_each_shape(backend, tmp_path):
    """A per-env-shapes handle: each env's wrench (env-indexed rows) against an oracle of its own body shape."""
    from smplsim_b200.abi import model_from_cfg
    from test_gpu_parity import _shape_variant
    pa = _shape_variant(tmp_path, leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2)
    mk = [make_models(control_mode="torque"), make_models(control_mode="torque", **{"robot.xml_path": pa})]
    models = [model_from_cfg(c) for c, _ in mk]
    n = 12
    env_model = np.array([(i * 5) % 3 % 2 for i in range(n)], dtype=np.int32)
    q, v = airborne_states(models[0], n, seed=6)
    rng = np.random.default_rng(8)
    ctrl = rng.uniform(-50, 50, (n, models[0].nu))
    xf = _wrenches(models[0], n, rng)
    env = backend.batch(mk[0][0], n, models=models, env_model=env_model)
    env.set_state(backend.t(q), backend.t(v))
    env.xfrc_applied = backend.t(xf)
    env.mj_step(backend.t(ctrl), 1)
    gq, gv = env.qpos.cpu().numpy(), env.qvel.cpu().numpy()
    for i, k in enumerate(env_model):
        e = _oracle_step(mk[k][1], q[i], v[i], np.zeros(models[0].nv), ctrl[i], xf[i])
        assert relerr(gv[i], e.qvel) < TOL and relerr(gq[i], e.qpos) < TOL, (i, k, relerr(gv[i], e.qvel))


def test_bad_wrench_tensor_is_refused(backend):
    import torch
    cfg, om = make_models(env="speed")
    m = om.model
    env = backend.batch(cfg, 4)
    for bad in (torch.zeros(4, m.nbody, 3, device=backend.device), torch.zeros(3, m.nbody, 6, device=backend.device),
                torch.zeros(4, m.nbody, 6, dtype=torch.float64, device=backend.device),
                torch.zeros(4, 6, m.nbody, device=backend.device).transpose(1, 2), np.zeros((4, m.nbody, 6), dtype=np.float32)):
        with pytest.raises(ValueError):
            env.xfrc_applied = bad
    other = "cpu" if backend.name == "gpu" else "meta"
    with pytest.raises(ValueError):
        env.xfrc_applied = torch.zeros(4, m.nbody, 6, device=other)
    assert env.xfrc_applied is None


def test_single_env_mj_data_xfrc_applied(backend):
    """B1: env.mj_data.xfrc_applied is one persistent [nbody + 1, 6] float64 array in MuJoCo indexing; a push written into it moves
    the env, an all-zero array is no wrench at all."""
    from smplsim_b200.envs import HumanoidSpeed
    cfg = make_cfg(env="speed", seed=4)

    class Env(HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    res = []
    for push in (False, True):
        env = Env(cfg, device=backend.device)
        x = env.mj_data.xfrc_applied
        assert x is env.mj_data.xfrc_applied and x.shape == (env.num_rigid_bodies + 1, 6) and x.dtype == np.float64
        env.reset()
        a = np.zeros(env.get_action_size(), dtype=np.float32)
        env.step(a)
        assert env._b.xfrc_applied is None
        if push:
            env.mj_data.xfrc_applied[1] = [300.0, 0, 0, 0, 0, 0]       # MuJoCo body 1 = the pelvis
        env.step(a)
        assert (env._b.xfrc_applied is not None) == push
        res.append(env.get_qvel())
        if push:
            env.mj_data.xfrc_applied[:] = 0.0
            env.step(a)
            assert env._b.xfrc_applied is None
    assert res[1][0] - res[0][0] > 0.1          # 300 N on the ~70 kg body for one env step (1/30 s): ~0.14 m/s along +x


def test_auto_reset_drops_the_wrench_for_the_rest_of_the_call(backend):
    """mj_checkVel: an env whose qvel blows past 1e10 is reset inside the first substep (mj_resetData also zeroes xfrc_applied) and
    runs the remaining substeps without the wrench, like the oracle; the other envs keep theirs and the tensor is left as it was."""
    cfg, om = make_models(env="speed")
    m = om.model
    n = 8
    env = backend.batch(cfg, n, seed=0)
    env.reset()
    e = XfrcOracleEnv(om, env_id=3)
    e.reset()
    qv = env.qvel.clone()
    qv[3, 10] = 3e10; e.qvel[10] = 3e10
    env.set_state(env.qpos.clone(), qv)
    e.forward()
    xf = _wrenches(m, n, np.random.default_rng(6), fscale=0.5, tscale=5.0)
    env.xfrc_applied = backend.t(xf)
    e.xfrc_applied[:] = xf[3]
    act = np.zeros((n, m.nu)); act[:] = 0.05
    obs, rew, term, trunc = [x.cpu().numpy() for x in env.step(backend.t(act))]
    e.warn = 0
    o, r, te, tr = e.step(act[3])
    assert e.warn & 2 and env.status.cpu().numpy()[3] & 2
    assert not e.xfrc_applied.any()
    assert np.abs(obs[3] - o).max() < 5e-4, np.abs(obs[3] - o).max()
    assert np.array_equal(env.xfrc_applied.cpu().numpy(), backend.t(xf).cpu().numpy())
