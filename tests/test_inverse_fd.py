"""Finite-difference inverse-dynamics derivatives (smplsim_inverse_fd, HumanoidBatchB200.inverse_fd, envs.mjd_inverseFD) against the
fp64 oracle, against the forward derivatives of transition_fd, and against inverse() itself.

States: rollouts of the speed task (floor contacts, joint-limit rows) and airborne states.  The kernel tests run on the H100 (-m gpu)
and on the host emulator build of the same kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from smplsim_b200.abi import SmplsimInverseFdCfgC
from test_forward_fd import _oracle_env, _perturb, _small_and_production, _states
from test_forward_fd_paths import _past_cap
from test_inverse import _forward, _over_cap, ref_inverse
from util_states import airborne_states, make_models, relerr

EPS = (1e-3, 1e-2, 1.0)   # the defaults
KINK, SOLVER = 1, 2
# dfrc against a centered fp64 oracle FD of ref_inverse at the same eps: per column max|k - o| / max(1, max|o|) over the column's
# block, and per block (dq / qvel / qacc) ||K - O||_F / max(1, ||O||_F), on columns neither side flags.  Worst seen on the emulator:
# column 2.2e-4, block 2.6e-4 (SMPL), column 3.4e-4, block 6.1e-4 (SMPL-X).
COL_TOL, BLOCK_TOL = 2e-3, 3e-3
MAX_EXCLUDED = 0.05


def _blocks(nv):
    return {"dq": slice(0, nv), "qvel": slice(nv, 2 * nv), "qacc": slice(2 * nv, 3 * nv)}


def _row_set(e, qacc):
    """The inverse's row set at the oracle env's state: contacts and the sign pattern of the row residuals."""
    _, _, r = ref_inverse(e, qacc)
    return (e.ncon, e.nefc, tuple(e.contacts()["geom"]), tuple(r < 0))


def _perturb3(m, q, v, a, col, s):
    """(qpos, qvel, qacc) in fp64 with column col of [dq, qvel, qacc] moved by s."""
    a = a.astype(np.float64).copy()
    if col < 2 * m.nv:
        q, v, _ = _perturb(m, q, v, np.zeros(m.nu), col, s)
    else:
        q, v = q.astype(np.float64), v.astype(np.float64)
        a[col - 2 * m.nv] += s
    return q, v, a


def oracle_dfrc(om, q, v, a, eps):
    """Centered fp64 FD of ref_inverse at the fp32 state; and per column whether the oracle's row set switched."""
    m = om.model
    nv = m.nv
    D = np.zeros((nv, 3 * nv)); switched = np.zeros(3 * nv, bool)
    for j in range(3 * nv):
        e = eps[j // nv]
        r = []
        for s in (e, -e):
            qq, vv, aa = _perturb3(m, q, v, a, j, s)
            o = _oracle_env(om, qq, vv, np.zeros(m.nu))
            o.forward()
            r.append((ref_inverse(o, aa)[0], _row_set(o, aa)))
        D[:, j] = (r[0][0] - r[1][0]) / (2 * e)
        switched[j] = r[0][1] != r[1][1]
    return D, switched


def dfrc_errors(nv, K, O, keep):
    """(worst column, worst block) error on the kept columns, as test_forward_fd's dqacc_errors."""
    col = blk = 0.0
    for s in _blocks(nv).values():
        k = np.zeros_like(keep); k[s] = keep[s]
        if k.any():
            d = K[:, k] - O[:, k]
            col = max(col, np.abs(d).max() / max(1.0, np.abs(O[:, s]).max()))
            blk = max(blk, np.linalg.norm(d) / max(1.0, np.linalg.norm(O[:, k])))
    return col, blk


def _inv_states(robot, n, seed, nair=1):
    """_states of test_forward_fd with qacc = the oracle's forward qacc under the random ctrl (rows on and off the set)."""
    cfg, om, q, v, u = _states(robot, n, seed=seed, nair=nair)
    a = np.float32([_forward(om, q[i], v[i], u[i]).qacc.copy() for i in range(n)])   # copied while the oracle env lives
    return cfg, om, q, v, a, u


# ------------------------------------------------------------------ 1. against the fp64 oracle
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_dfrc_matches_oracle(backend, robot):
    n = 4 if robot == "smpl_humanoid" else 2
    cfg, om, q, v, a, _ = _inv_states(robot, n, seed=11)
    nv = om.model.nv
    env = backend.batch(cfg, 64)
    fd = env.inverse_fd(backend.t(q), backend.t(v), backend.t(a))
    K, F = fd["dfrc"].cpu().numpy().astype(np.float64), fd["flags"].cpu().numpy()
    excluded = total = 0
    worst = [0.0, 0.0]
    for i in range(n):
        O, sw = oracle_dfrc(om, q[i], v[i], a[i], EPS)
        keep = (F[i] == 0) & ~sw
        excluded += int((~keep).sum()); total += keep.size
        col, blk = dfrc_errors(nv, K[i], O, keep)
        worst = [max(worst[0], col), max(worst[1], blk)]
    print(f"{robot}: {excluded}/{total} columns excluded, worst column {worst[0]:.2e}, worst block {worst[1]:.2e}")
    assert excluded <= MAX_EXCLUDED * total
    assert worst[0] <= COL_TOL and worst[1] <= BLOCK_TOL


# ------------------------------------------------------------------ 2. exact structure of the qacc block
def test_qacc_block_structure(backend):
    """d qfrc_inverse / d qacc = M + J^T diag(D [r < 0]) J of the oracle on unflagged columns; on airborne rows without limit rows it is
    dynamics()["qM"] to fp32 rounding."""
    cfg, om, q, v, a, _ = _inv_states("smpl_humanoid", 4, seed=13)
    m = om.model
    nv = m.nv
    env = backend.batch(cfg, 64)
    fd = env.inverse_fd(backend.t(q), backend.t(v), backend.t(a))
    K, F = fd["dfrc"].cpu().numpy().astype(np.float64)[:, :, 2 * nv:], fd["flags"].cpu().numpy()[:, 2 * nv:]
    rows, worst = 0, 0.0
    for i in range(len(q)):
        e = _forward(om, q[i], v[i])
        efc = e.efc()
        _, _, r = ref_inverse(e, a[i].astype(np.float64))
        W = efc["D"] * (r < 0)
        H = e.M + efc["J"].T @ (W[:, None] * efc["J"])
        keep = F[i] == 0
        assert keep.mean() >= 0.95, i
        # worst seen on the emulator: 1.8e-5
        assert relerr(K[i][:, keep], H[:, keep]) <= 1e-4, (i, relerr(K[i][:, keep], H[:, keep]))
        worst = max(worst, relerr(K[i][:, keep], H[:, keep]))
        rows += e.nefc > 0
    assert rows >= 2
    q2, v2 = airborne_states(m, 3, seed=19)
    q2[:, 7:] *= 0.2
    q2, v2 = np.float32(q2), np.float32(v2)
    a2 = np.float32(np.random.default_rng(4).normal(size=v2.shape) * 3.0)
    fd = env.inverse_fd(backend.t(q2), backend.t(v2), backend.t(a2))
    M = env.dynamics(backend.t(q2), backend.t(v2))["qM"].cpu().numpy().astype(np.float64)
    K = fd["dfrc"].cpu().numpy().astype(np.float64)[:, :, 2 * nv:]
    print(f"contact rows: worst {worst:.2e}; airborne: worst {max(relerr(K[i], M[i]) for i in range(3)):.2e}")
    for i in range(3):
        assert _forward(om, q2[i], v2[i]).nefc == 0
        assert not fd["flags"][i].any()
        # fp32 rounding of qfrc_inverse over 2 eps_qacc; worst seen on the emulator: 9.5e-7
        assert relerr(K[i], M[i]) <= 5e-6, (i, relerr(K[i], M[i]))


# ------------------------------------------------------------------ 3. against the forward derivatives
def test_consistent_with_transition_fd(backend):
    """At qacc* = forward(q, v, u): f(q, v, qacc*(q, v, u)) = [0_6 ; u], so DfDa dqacc_ctrl = [0 ; I], DfDq + DfDa dqacc_q = 0 and
    DfDv + DfDa dqacc_v = 0, on columns neither call flags (rows whose DfDa has no flagged column).  Frobenius norms relative to [0 ; I]
    and to DfDq / DfDv."""
    cfg, om, q, v, u = _states("smpl_humanoid", 6, seed=17, nair=2)
    m = om.model
    nv, nu = m.nv, m.nu
    env = backend.batch(cfg, 64)
    tq, tv, tu = backend.t(q), backend.t(v), backend.t(u)
    fwd = env.transition_fd(tq, tv, tu, dqacc=True)
    inv = env.inverse_fd(tq, tv, fwd["qacc"], eps_qpos=1e-2, eps_qvel=1e-1)   # the steps of transition_fd's defaults
    G, Fg = fwd["dqacc"].cpu().numpy().astype(np.float64), fwd["flags"].cpu().numpy()
    K, Fk = inv["dfrc"].cpu().numpy().astype(np.float64), inv["flags"].cpu().numpy()
    I = np.r_[np.zeros((6, nu)), np.eye(nu)]
    worst = {"ctrl": 0.0, "q": 0.0, "v": 0.0}
    rows = 0
    for i in range(len(q)):
        if Fk[i, 2 * nv:].any():
            continue
        Da = K[i][:, 2 * nv:]
        kc = Fg[i, 2 * nv:] == 0
        worst["ctrl"] = max(worst["ctrl"], np.linalg.norm((Da @ G[i][:, 2 * nv:] - I)[:, kc]) / np.linalg.norm(I[:, kc]))
        for name, s in (("q", slice(0, nv)), ("v", slice(nv, 2 * nv))):
            k = (Fg[i, s] == 0) & (Fk[i, s] == 0)
            R = K[i][:, s] + Da @ G[i][:, s]
            worst[name] = max(worst[name], np.linalg.norm(R[:, k]) / max(1.0, np.linalg.norm(K[i][:, s][:, k])))
        rows += 1
    print(rows, {k: f"{x:.2e}" for k, x in worst.items()})
    assert rows >= 4
    # worst seen on the emulator: ctrl 4.1e-2 (fp32 rounding of qacc ~ 1e3 over eps_ctrl = 1 in dqacc, times the large entries of M),
    # q 6.3e-3, v 4.5e-4
    assert worst["ctrl"] <= 0.2 and worst["q"] <= 3e-2 and worst["v"] <= 2.5e-3


# ------------------------------------------------------------------ 4. bit-identity
def test_column_equals_inverse_difference(backend):
    """Root-translation, hinge, qvel and qacc columns: (inverse(x+) - inverse(x-)) / (x+ - x-) bit for bit; the nominal output is
    inverse() bit for bit."""
    cfg, om, q, v, a, _ = _inv_states("smpl_humanoid", 4, seed=19)
    nv = om.model.nv
    env = backend.batch(cfg, 32)
    t = [backend.t(x) for x in (q, v, a)]
    fd = env.inverse_fd(*t)
    assert torch.equal(fd["qfrc_inverse"], env.inverse(*t))
    for col in (2, 6, 40, nv - 1, nv + 3, nv + 20, 2 * nv - 1, 2 * nv, 2 * nv + 5, 2 * nv + 33, 3 * nv - 1):
        k, e = (0, col + 1 if col >= 6 else col) if col < nv else (1, col - nv) if col < 2 * nv else (2, col - 2 * nv)
        tp, tm = [x.clone() for x in t], [x.clone() for x in t]
        tp[k][:, e] += EPS[col // nv]; tm[k][:, e] -= EPS[col // nv]
        want = (env.inverse(*tp) - env.inverse(*tm)) / (tp[k][:, e] - tm[k][:, e])[:, None]
        assert torch.equal(fd["dfrc"][:, :, col], want), col


def test_launch_shapes(backend, monkeypatch):
    """3 rows: chunked by 32 slots on a 1-warp handle, one launch on the production 8-warp handle; bit-identical.  n = 0 returns empty
    outputs."""
    cfg, om, q, v, a, _ = _inv_states("smpl_humanoid", 3, seed=23)
    small, big = _small_and_production(backend, cfg, monkeypatch)
    outs = [e.inverse_fd(backend.t(q), backend.t(v), backend.t(a)) for e in (small, big)]
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), k
    m = om.model
    z = [backend.t(np.zeros((0, w))) for w in (m.nq, m.nv, m.nv)]
    f0 = big.inverse_fd(*z)
    assert f0["dfrc"].shape == (0, m.nv, 3 * m.nv) and f0["flags"].shape == (0, 3 * m.nv)


# ------------------------------------------------------------------ 5. flags
def _at_margin(om, seed):
    """A standing state lowered or raised so that its lowest contact sits exactly at the contact margin."""
    _, _, q, v, a, _ = _inv_states("smpl_humanoid", 1, seed=seed, nair=0)
    q, v, a = q[0].astype(np.float64), v[0], a[0]
    e = _forward(om, q, v)
    assert e.ncon > 0
    q[2] += e.m.margin - e.contacts()["dist"].min()   # contacts are generated below the margin
    return np.float32(q), v, a


def test_flags(backend):
    """A foot at the contact margin: KINK on the root-height column, which moves it across; nothing with centered=False.  A state with
    more joint-limit rows than the kernels hold: SOLVER on every column."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    nv = m.nv
    q, v, a = _at_margin(om, 29)
    qc, vc = _past_cap(m, 5)
    assert _over_cap(_forward(om, qc, vc))
    Q, V, A = np.float32([q, qc]), np.float32([v, vc]), np.float32([a, np.zeros(nv)])
    env = backend.batch(cfg, 64)
    c = env.inverse_fd(backend.t(Q), backend.t(V), backend.t(A))
    f = env.inverse_fd(backend.t(Q), backend.t(V), backend.t(A), centered=False)
    Fc, Ff = c["flags"].cpu().numpy(), f["flags"].cpu().numpy()
    assert Fc[0, 2] & KINK
    assert not (Fc[0] & SOLVER).any()
    assert not Ff[0].any()
    assert (Fc[1] & SOLVER).all() and (Ff[1] & SOLVER).all()
    assert torch.equal(c["qfrc_inverse"], f["qfrc_inverse"])


# ------------------------------------------------------------------ 6. isolation
def test_stepper_cannot_tell(backend):
    """step -> inverse_fd -> step and step -> step from the same state: every output and state row bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 16
    res = []
    for with_fd in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng, rin = np.random.default_rng(1), np.random.default_rng(2)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_fd and t == 0:        # every scratch row of the handle
                vv = torch.as_tensor(rin.normal(size=(2, m.nv)), dtype=torch.float32, device=env.qpos.device)
                env.inverse_fd(env.qpos[:2].clone(), vv, vv * 10.0)
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_nan_row_leaves_other_rows_alone(backend):
    """A NaN in one row's qpos: every column of that row has SOLVER, the other rows are bit-identical with a call without the NaN."""
    cfg, om, q, v, a, _ = _inv_states("smpl_humanoid", 3, seed=31)
    env = backend.batch(cfg, 64)
    ref = env.inverse_fd(backend.t(q), backend.t(v), backend.t(a))
    q2 = q.copy(); q2[1, 9] = np.nan
    got = env.inverse_fd(backend.t(q2), backend.t(v), backend.t(a))
    assert bool((got["flags"][1] & SOLVER).all())
    for k in ref:
        assert torch.equal(got[k][[0, 2]], ref[k][[0, 2]]), k


# ------------------------------------------------------------------ 7. arguments
def test_arguments(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 4)
    L, h, s = env._L(), env._h, env._stream()
    q, v = airborne_states(m, 4, seed=1)
    tq, tv = backend.t(q), backend.t(v)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    qf = backend.t(np.zeros((4, m.nv)))
    D = backend.t(np.zeros((4, m.nv, 3 * m.nv)))
    good = SmplsimInverseFdCfgC(1e-2, 1e-1, 1.0, 1, 0)

    def err(rc, code, text):
        assert rc == code, (rc, code)
        assert L.smplsim_last_error().decode() == text

    fd = lambda hh, cfg_, n, a=p(tv), qfrc=p(qf), dfrc=p(D), fl=None: L.smplsim_inverse_fd(hh, cfg_, p(tq), p(tv), a, n, qfrc, dfrc, fl, s)  # noqa: E731
    err(fd(None, C.byref(good), 4), -1, "smplsim_inverse_fd: null handle / cfg or n < 0")
    err(fd(h, None, 4), -1, "smplsim_inverse_fd: null handle / cfg or n < 0")
    err(fd(h, C.byref(good), -1), -1, "smplsim_inverse_fd: null handle / cfg or n < 0")
    err(fd(h, C.byref(good), 4, a=None), -1, "smplsim_inverse_fd: null argument (qpos, qvel, qacc and qfrc_inverse are required)")
    err(fd(h, C.byref(good), 4, qfrc=None), -1, "smplsim_inverse_fd: null argument (qpos, qvel, qacc and qfrc_inverse are required)")
    err(fd(h, C.byref(good), 4, dfrc=None), -1, "smplsim_inverse_fd: no derivative output requested (dfrc and flags both NULL)")
    for bad in ((0.0, 1e-1, 1.0), (1e-2, -1.0, 1.0), (1e-2, 1e-1, float("nan")), (float("inf"), 1e-1, 1.0)):
        err(fd(h, C.byref(SmplsimInverseFdCfgC(*bad, 1, 0)), 4), -1,
            "smplsim_inverse_fd: eps_qpos, eps_qvel and eps_qacc must be finite and > 0")
    assert L.smplsim_inverse_fd(h, C.byref(good), None, None, None, 0, None, None, None, s) == 0
    for name in ("eps_qpos", "eps_qvel", "eps_qacc"):
        with pytest.raises(ValueError, match=name):
            env.inverse_fd(tq, tv, tv, **{name: 0.0})
    with pytest.raises(ValueError, match="shape"):
        env.inverse_fd(tq, tv, tv[:, :-1])

    from smplsim_b200 import _lib
    env.set_env_params(friction=backend.t(np.full(4, 0.8)))
    text = "smplsim_inverse_fd: not available while the handle has per-env parameter records (smplsim_clear_env_params)"
    err(fd(h, C.byref(good), 4), -3, text)
    with pytest.raises(_lib.SmplsimError, match="parameter records"):
        env.inverse_fd(tq, tv, tv)

    from smplsim_b200.abi import model_from_cfg
    shapes = backend.batch(cfg, 4, models=[model_from_cfg(cfg)] * 2, env_model=np.array([0, 1, 0, 1], dtype=np.int32))
    err(fd(shapes._h, C.byref(good), 4), -3,
        "smplsim_inverse_fd: not available with per-env body shapes (the column slots of a row span CTAs of any shape)")

    scfg, _ = make_models(env="getup", control_mode="torque", self_collision=True)
    senv = backend.batch(scfg, 4)
    err(fd(senv._h, C.byref(good), 4), -3,
        "smplsim_inverse_fd: the inverse does not build geom-geom contacts (handle created with self_collision = 1)")
    with pytest.raises(_lib.SmplsimError, match="geom-geom"):
        senv.inverse_fd(tq, tv, tv)


# ------------------------------------------------------------------ 8. single env
def test_single_env_mjd_inverseFD(backend):
    from smplsim_b200.envs import HumanoidSpeed, mjd_inverseFD
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
    env.step(np.zeros(env.get_action_size(), dtype=np.float32))
    nv = om.model.nv
    d = env.mj_data
    b = env._b
    row = lambda x: torch.as_tensor(np.float32(x)[None], device=b.device)  # noqa: E731
    want = b.inverse_fd(row(d.qpos), row(d.qvel), row(d.qacc))["dfrc"][0].cpu().numpy().astype(np.float64)
    outs = []
    for flg in (0, 1):
        Dq, Dv, Da = np.zeros((nv, nv)), np.zeros((nv, nv)), np.zeros((nv, nv))
        mjd_inverseFD(env.mj_model, d, None, flg, Dq, Dv, Da, None, None, None, None)
        outs.append((Dq, Dv, Da))
        for k, X in enumerate((Dq, Dv, Da)):
            assert np.array_equal(X, want[:, k * nv:(k + 1) * nv].T), (flg, k)
    for x, y in zip(*outs):
        assert np.array_equal(x, y)
    w1 = b.inverse_fd(row(d.qpos), row(d.qvel), row(d.qacc), 1e-3, 1e-3, 1e-3)["dfrc"][0].cpu().numpy().astype(np.float64)
    Da = np.zeros((nv, nv))
    mjd_inverseFD(env.mj_model, d, 1e-3, 0, None, None, Da, None, None, None, None)
    assert np.array_equal(Da, w1[:, 2 * nv:].T)
    for i in range(4):
        extra = [None] * 4
        extra[i] = np.zeros((1, 1))
        with pytest.raises(NotImplementedError, match="DmDq"):
            mjd_inverseFD(env.mj_model, d, None, 0, Dq, Dv, Da, *extra)
