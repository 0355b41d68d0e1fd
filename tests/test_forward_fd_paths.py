"""Forward dynamics (smplsim_forward) and the finite-difference transition derivatives (smplsim_transition_fd) on every launch path
of k_fwd5 and at their edges, against the fp64 oracle and against 1-warp CTAs.

test_forward_fd holds the two calls to the oracle on small SMPL batches in 1-warp CTAs.  Here the same kernel runs where production
runs it and where its rarer branches live:

- forward at the production CTA shapes (8-warp SMPL with a ragged second launch, 4-warp SMPL-X), where l_solve's CTA-wide iteration
  loop holds every warp to the slowest env of its CTA;
- forward through the instance that reads per-env parameter records (k_fwd5<P>) and on per-env body shapes (the slot map);
- rows with non-finite inputs and rows past the joint-limit row cap, next to good rows in the same CTAs and launches;
- the column pass split over launches of num_envs slots, a row's columns straddling two launches;
- SMPL-X A / B against whole oracle steps, both branches of the root-rotation assembly (series and closed form of R(th)^T, J_r(th)),
  and the kink flag against the oracle's own active-set switches.

As in test_cta_shapes, the GPU reaches the production CTA shapes by env count alone and the emulator forces them with SMPLSIM_WPB at a
few dozen envs; every test asserts the CTA shape it ran."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
from smplsim_b200 import _lib  # noqa: E402
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from test_contact_wrench import oracle_wrench  # noqa: E402
from test_cta_shapes import (CHUNK, EPW, N_DYN, N_SHAPES, N_SMPL, N_SMPLX, _bit_equal, _dups_equal, _one_warp_chunks,  # noqa: E402
                             _pool, _production, _tiled, _wpb)
from test_env_params import draw, oracle_for, variant  # noqa: E402
from test_forward_fd import (EPS, QACC_TOL, _oracle_env, _perturb, _rollout, _states, dqacc_errors, oracle_AB,  # noqa: E402
                             oracle_dqacc)
from test_gpu_parity import _shape_variant  # noqa: E402
from test_inverse import _forward, _near_switch, _over_cap, _weight  # noqa: E402
from util_states import airborne_states, make_models, relerr, rollout_states  # noqa: E402

WRENCH_TOL = 2e-3     # contact wrench: max |kernel - oracle| in units of the body weight (or the largest component), test_inverse's TOL
ROT_TOL = 1e-5        # rotation rows of A / B against their fp64 restatement from the kernel's own dqacc, qacc and qvel (relative, F);
                      # worst seen: 1.3e-7 on the emulator, 1.2e-7 on an H100
# SMPL-X A / B against whole oracle steps (the method of test_AB_matches_full_step_oracle, whose SMPL bounds are 1e-2, 1e-3, 1e-4).
# SMPL-X qacc runs to ~3e3 at these states, and the fp32 rounding of the two solves, divided by 2 eps, puts a relative error of a few
# 1e-3 into A - I on the contact row's unflagged columns; an oracle FD at the kernel's own eps (no truncation error) gives the same.
# On the contact row the kernel flags the root-rotation columns, so that the rotation rows' reference norm is small (~5e-3) and their
# relative error large.  Worst seen: A - I 6.9e-3, B 3.2e-4, rotation rows 5.3e-4 on the emulator; 6.7e-3, 2.6e-4, 5.3e-4 on an H100.
SMPLX_AB_TOL = {"A - I": 2e-2, "B": 1e-3, "rot rows": 2e-3}
THETAS = (0.02, 0.0999, 0.1001, 0.3, 1.0)   # |th| = |h v'_nom[3:6]|: the kernel's series branch below 0.1, closed form above
# those rows against oracle_AB: the bounds of test_AB_matches_full_step_oracle (A - I, B, rotation rows) up to |th| = 0.3.  At |th| = 1
# (450 rad/s) qacc reaches ~2e5 and the fp32 rounding of the two solves, divided by 2 eps, grows with it.  Worst seen, |th| <= 0.3:
# 1.4e-3, 4.3e-4, 3.4e-5 on the emulator, 1.4e-3, 4.5e-4, 3.6e-5 on an H100; |th| = 1: 4.3e-4, 4.2e-3, 9.3e-5 on the emulator, 4.2e-4,
# 4.1e-3, 8.8e-5 on an H100.
SPIN_AB_TOL = {0.3: {"A - I": 1e-2, "B": 1e-3, "rot rows": 1e-4}, 1.0: {"A - I": 1e-2, "B": 1e-2, "rot rows": 3e-4}}


def _fwd(env, t, q, v, u, w):
    out = env.forward(t(q), t(v), t(u), qacc_warmstart=t(w), contact_wrench=True)
    return {k: x.cpu().numpy().copy() for k, x in out.items()}


def _bits(d):
    """float32 outputs as their bit patterns, so that bit identity includes the NaN a column gets where its perturbation vanishes in
    fp32 (den = 0: qvel 8e9 + eps_qvel of the overflowing pool state; the column carries SMPLSIM_FD_SOLVER)."""
    return {k: x.view(np.int32) if x.dtype == np.float32 else x for k, x in d.items()}


def _check_forward(e, r, i, wt):
    """Row i of forward outputs r against the oracle forward pass e at the same state, ctrl and warm start: qacc to QACC_TOL, contact
    mask exact, contact wrench to WRENCH_TOL of the weight wt.  Returns (qacc error, wrench error)."""
    err = relerr(r["qacc"][i], e.qacc)
    assert err <= QACC_TOL, ("qacc", i, err, e.ncon, e.nefc)
    assert int(r["contact_mask"][i]) == e.contact_mask, ("contact mask", i, bin(int(r["contact_mask"][i])), bin(e.contact_mask))
    W = oracle_wrench(e)
    werr = float(np.abs(r["contact_wrench"][i] - W).max() / max(wt, float(np.abs(W).max())))
    assert werr <= WRENCH_TOL, ("contact wrench", i, werr)
    if e.ncon == 0:
        assert np.all(r["contact_wrench"][i] == 0.0), i
    return err, werr


def _skip(e):
    """Not compared: joint-limit rows past the cap (dropped by design) or a contact / row inside the guard band (fp32 may set it
    either way)."""
    return _over_cap(e) or _near_switch(e, e.qacc)


# ------------------------------------------------------------------ 1. forward at the production CTA shapes
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_forward_at_production_shape(backend, monkeypatch, robot):
    """The _pool states tiled over the rows, each with its pool warm start: SMPL on an 8-warp handle with num_envs rows plus a ragged
    second launch, SMPL-X on a 4-warp handle with a ragged last CTA.  Against the oracle per pool state, bit-identical with 1-warp
    CTAs and across rows of the same pool state."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    if robot == "smpl_humanoid":
        nenv, extra = N_DYN[backend.name]
        env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
        assert extra % (8 * EPW) != 0
    else:
        nenv, extra = N_SMPLX[backend.name], 0
        env = _production(backend, monkeypatch, cfg, nenv, 4)
    n = nenv + extra
    q, v, w, kinds, ctrl, idx = _tiled(robot, n)
    t = backend.t

    def run(env, s):
        return _fwd(env, t, q[idx[s]], v[idx[s]], ctrl[idx[s]], w[idx[s]])

    got = run(env, slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), run), "production vs 1-warp CTAs")
    _dups_equal(got, idx, "same pool state")
    wt = _weight(m)
    ncmp = nrows = 0
    worst = [0.0, 0.0]
    for k in range(len(q)):
        st = int(got["status"][k])
        if kinds[k] == "bad":
            assert st & 4, (k, st)
            continue
        assert not st & (1 | 2 | 4), (k, kinds[k], st)
        e = _forward(om, q[k], v[k], ctrl[k], w[k])
        if _skip(e):
            continue
        err = _check_forward(e, got, k, wt)
        worst = [max(a, b) for a, b in zip(worst, err)]
        ncmp += 1
        nrows += e.nefc > 0
    assert got["solver_iter"].max() >= 4 and got["solver_iter"].min() == 0    # CTAs mix long solves with airborne envs
    print(f"{robot}: {ncmp}/{len(q)} pool states compared ({nrows} with rows), worst qacc {worst[0]:.2e}, wrench {worst[1]:.2e}")
    # compared: 28 of 30 pool states (SMPL and SMPL-X; the rest are the bad state and a guard-band state).  Worst qacc / wrench error:
    # 4.6e-5 / 6.0e-5 on the emulator, 8.1e-5 / 1.3e-4 on an H100
    assert ncmp >= len(q) - 8 and nrows >= len(q) // 2, (ncmp, nrows)


# ------------------------------------------------------------------ 2. forward with per-env parameter records (k_fwd5<P>)
def test_forward_with_parameter_records(backend, monkeypatch):
    """An SMPL handle with draw() records on every env, n == num_envs: each pool state against the oracle of its env's variant model,
    at the 8-warp production shape and bit-identical with 1-warp CTAs."""
    robot = "smpl_humanoid"
    cfg, _ = make_models(robot=robot, control_mode="torque")
    m = model_from_cfg(cfg)
    n = N_SMPL[backend.name]
    q, v, w, kinds, ctrl, idx = _tiled(robot, n, seed=8)
    P = len(q)
    prm = draw(m, P, 83)
    t = backend.t

    def run(env, s):
        env.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        return _fwd(env, t, q[idx[s]], v[idx[s]], ctrl[idx[s]], w[idx[s]])

    got = run(_production(backend, monkeypatch, cfg, n, 8), slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), "records: 8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "records: same pool state")
    ncmp = ncon = 0
    for k in range(P):
        if kinds[k] == "bad":
            assert got["status"][k] & 4, k
            continue
        e = _forward(oracle_for(cfg, m, prm, k), q[k], v[k], ctrl[k], w[k])
        if _skip(e):
            continue
        _check_forward(e, got, k, float(np.sum(variant(m, prm, k).body_mass)) * 9.81)
        ncmp += 1
        ncon += e.ncon > 0
    assert ncmp >= P - 8 and ncon >= P // 3, (ncmp, ncon)


@pytest.mark.parametrize("mode", ["torque", "uhc_pd"])
def test_forward_record_fields(backend, mode):
    """Records with the model's values give what the handle without records gives (bit for bit on the GPU; 1e-6 on the emulator,
    whose compiler contracts the two instances' arithmetic into FMAs differently, the rule of test_nominal_records_mask_readback_and_
    clear).  ctrl is raw torque: records that change only kp / kd / torque_limit leave qacc bit-identical to nominal records on the
    same instance.  Records that change friction, gravity and masses change qacc on every row with contacts: they are read."""
    robot = "smpl_humanoid"
    cfg, _ = make_models(robot=robot, control_mode=mode)
    m = model_from_cfg(cfg)
    q, v, w, kinds, ctrl, _ = _tiled(robot, 30, seed=9)
    P = len(q)
    t = backend.t
    env = backend.batch(cfg, P)
    ref = _fwd(env, t, q, v, ctrl, w)
    env.set_env_params(**env.env_params)
    nom = _fwd(env, t, q, v, ctrl, w)
    if backend.name == "gpu":
        _bit_equal(nom, ref, "nominal records vs no records")
    else:
        for k in ("contact_mask", "status"):
            assert np.array_equal(nom[k], ref[k]), k
        assert max(relerr(nom["qacc"][i], ref["qacc"][i]) for i in range(P)) < 1e-6
    D = draw(m, P, 85)
    env.set_env_params(**{k: t(D[k]) for k in ("kp", "kd", "torque_limit")})
    gains = _fwd(env, t, q, v, ctrl, w)
    _bit_equal(gains, nom, "kp / kd / torque_limit records vs nominal records")
    env.set_env_params(**{k: t(D[k]) for k in ("friction", "gravity", "body_mass_scale")})
    phys = _fwd(env, t, q, v, ctrl, w)
    rows = (nom["contact_mask"] != 0) & (nom["status"] == 0)
    assert rows.sum() >= P // 3, rows.sum()
    moved = np.abs(phys["qacc"] - nom["qacc"]).max(axis=1) > 1e-3 * np.maximum(1.0, np.abs(nom["qacc"]).max(axis=1))
    assert moved[rows].all(), np.flatnonzero(rows & ~moved)


# ------------------------------------------------------------------ 3. forward on per-env body shapes
def test_forward_per_env_shapes(backend, monkeypatch, tmp_path):
    """Three body shapes interleaved in ragged groups (every shape's last CTA has empty slots) at the 8-warp production shape: each row
    against its own shape's oracle, contact wrench included; bit-identical with 1-warp CTAs; n != num_envs is refused."""
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]

    def mk(mode, k):
        return make_models(control_mode=mode, **({"robot.xml_path": paths[k]} if paths[k] else {}))
    n = N_SHAPES[backend.name]
    env_model = np.array([(i * 7 + i // 5) % 3 for i in range(n)], dtype=np.int32)
    assert (np.bincount(env_model) % (8 * EPW) != 0).all()
    oms = [mk("torque", k)[1] for k in range(3)]
    cfg0 = mk("torque", 0)[0]
    models = [model_from_cfg(mk("torque", k)[0]) for k in range(3)]
    pools = [rollout_states(mk("uhc_pd", k)[1], 12, seed=30 + k, every=9) for k in range(3)]
    pidx = np.zeros(n, dtype=np.int64)
    seen = [0, 0, 0]
    for i, k in enumerate(env_model):
        pidx[i] = seen[k] % 12
        seen[k] += 1
    q, v, w = (np.array([pools[k][j][pidx[i]] for i, k in enumerate(env_model)]) for j in range(3))
    ctrl = np.random.default_rng(6).uniform(-80, 80, (12, models[0].nu))[pidx]
    t = backend.t

    def run(env, s):
        return _fwd(env, t, q[s], v[s], ctrl[s], w[s])

    env = _production(backend, monkeypatch, cfg0, n, 8, models=models, env_model=env_model)
    got = run(env, slice(0, n))
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg0, s.stop - s.start, models=models, env_model=env_model[s]), run,
                           chunk=CHUNK - 12)
    _bit_equal(got, ref, "per-env shapes: 8-warp vs 1-warp CTAs")
    key = env_model * 12 + pidx
    _dups_equal(got, np.unique(key, return_inverse=True)[1], "same shape and state")
    ncmp = ncon = 0
    for kk in np.unique(key):
        i = int(np.flatnonzero(key == kk)[0])
        k = env_model[i]
        assert not got["status"][i] & (1 | 2 | 4), (i, got["status"][i])
        e = _forward(oms[k], q[i], v[i], ctrl[i], w[i])
        if _skip(e):
            continue
        _check_forward(e, got, i, _weight(models[k]))
        ncmp += 1
        ncon += e.ncon > 0
    assert ncmp >= 30 and ncon >= ncmp // 3, (ncmp, ncon)
    with pytest.raises(_lib.SmplsimError, match="num_envs"):
        env.forward(t(q[:8]), t(v[:8]), t(ctrl[:8]))


# ------------------------------------------------------------------ 4. bad rows: non-finite inputs, joint-limit rows past the cap
def _past_cap(m, seed):
    """An airborne state with 20 hinges past their range (more joint-limit rows than the kernels hold), moving further out."""
    q, v = airborne_states(m, 1, seed=seed)
    q, v = q[0], v[0]
    q[7:] *= 0.2
    rng = np.random.default_rng(seed)
    lo, hi = np.asarray(m.dof_range)[6:, 0], np.asarray(m.dof_range)[6:, 1]
    d = rng.choice(m.nu, 20, replace=False)
    up = rng.random(20) < 0.5
    q[7 + d] = np.where(up, hi[d] + 0.05, lo[d] - 0.05)
    v[6 + d] = np.where(up, 1.0, -1.0)
    return q, v


def test_bad_rows_leave_other_rows_alone(backend, monkeypatch):
    """Forward on an 8-warp handle with num_envs rows plus a ragged second launch: a NaN in qpos, an inf in qvel, a NaN in ctrl, a NaN
    in the warm start and a row with 20 hinges past their range, all inside CTA 0.  Each bad row reports its status bit (1, 2, 4, 8;
    the NaN warm start, which only seeds the working set, none: that row still gives the clean row's qacc), every other row is
    bit-identical with the clean call.  transition_fd on the same kinds of rows, the first of them holding the first launch boundary
    (slot num_envs), so that bad and good rows share CTAs and launches: every column of a bad or over-cap row has SMPLSIM_FD_SOLVER,
    every other row is bit-identical with a call without the bad rows."""
    robot = "smpl_humanoid"
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    nenv, extra = N_DYN[backend.name]
    n = nenv + extra
    env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
    q, v, w, kinds, ctrl, idx = _tiled(robot, n)
    assert kinds[0] == "lying"
    q, v, w, ctrl = q[idx], v[idx], w[idx], ctrl[idx]
    t = backend.t
    clean = _fwd(env, t, q, v, ctrl, w)
    qc, vc = _past_cap(m, 5)
    assert _over_cap(_forward(om, qc, vc))
    bad = {3: 1, 9: 2, 12: 4, 20: 8}               # row -> the status bit it must report
    wrow = 30                                      # NaN warm start: the lying state (contacts, several active-set iterations)
    assert max(*bad, wrow) < 8 * EPW and clean["contact_mask"][wrow] != 0 and clean["solver_iter"][wrow] >= 2
    q2, v2, u2, w2 = q.copy(), v.copy(), ctrl.copy(), w.copy()
    q2[3, 9] = np.nan; v2[9, 0] = np.inf; u2[12, 40] = np.nan; w2[wrow, 17] = np.nan
    q2[20], v2[20] = qc, vc
    got = _fwd(env, t, q2, v2, u2, w2)
    keep = np.setdiff1d(np.arange(n), [*bad, wrow])
    _bit_equal({k: x[keep] for k, x in got.items()}, {k: x[keep] for k, x in clean.items()}, "forward: rows next to bad rows")
    for r, bit in bad.items():
        assert got["status"][r] & bit, (r, got["status"][r], bit)
    assert not got["status"][20] & 7 and np.isfinite(got["qacc"][20]).all()
    # the warm start only seeds the contact rows' working set: a NaN there is no bad state, the solve ends where the clean row's does
    assert got["status"][wrow] == 0 and got["contact_mask"][wrow] == clean["contact_mask"][wrow]
    assert relerr(got["qacc"][wrow], clean["qacc"][wrow]) <= QACC_TOL
    # transition_fd: rows b .. b + 5 around the row b that holds the first launch boundary (slot num_envs), the bad rows among them
    ncol = 2 * m.nv + m.nu
    b = nenv // ncol
    nf = b + 6
    assert nenv % ncol != 0 and nf * ncol > nenv
    qf, vf, uf = q[:nf].copy(), v[:nf].copy(), ctrl[:nf].copy()
    qf[b, 9] = np.nan; vf[b + 1, 0] = np.inf; uf[b + 3, 40] = np.nan
    qf[b + 4], vf[b + 4] = qc, vc
    badf = [b, b + 1, b + 3, b + 4]
    good = np.setdiff1d(np.arange(nf), badf)
    fd = env.transition_fd(t(qf), t(vf), t(uf), dqacc=True)
    ref = env.transition_fd(t(qf[good]), t(vf[good]), t(uf[good]), dqacc=True)
    fd = {k: x.cpu().numpy() for k, x in fd.items()}
    _bit_equal(_bits({k: x[good] for k, x in fd.items()}), _bits({k: x.cpu().numpy() for k, x in ref.items()}),
               "transition_fd: rows next to bad rows")
    for r in badf:
        assert (fd["flags"][r] & 2).all(), (r, np.flatnonzero(~(fd["flags"][r] & 2).astype(bool))[:8])


# ------------------------------------------------------------------ 5. column-mode launch shapes
# (num_envs, rows, warps per CTA, rows whose columns straddle a launch boundary); launches are of num_envs slots each
FD_LAUNCH = {"gpu": {"smpl_humanoid": (4096, 41, 8, [18, 37]),        # 8 979 slots: 4 096 + 4 096 + 787 (ragged)
                     "smplx_humanoid": (2049, 9, 4, [4, 8])},         # 4 239 slots: 2 049 + 2 049 + 141
             "emu": {"smpl_humanoid": (40, 2, 8, [0, 1]),             # 438 slots in 11 launches of 40 (the last 38)
                     "smplx_humanoid": (17, 2, 4, [0, 1])}}           # 942 slots in 56 launches of 17 (the last 7)
ONE_WARP_ENVS = {"gpu": CHUNK, "emu": 24}


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_fd_launch_shapes(backend, monkeypatch, robot):
    """transition_fd on a production handle, whose launches of num_envs slots split rows, against a 1-warp handle whose launches split
    them elsewhere: qacc, A, B, dqacc and flags bit-identical."""
    nenv, n, wpb, split = FD_LAUNCH[backend.name][robot]
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    ncol = 2 * m.nv + m.nu
    bounds = range(nenv, n * ncol, nenv)
    assert all(s % ncol for s in bounds)                          # every launch boundary falls inside a row
    assert sorted({s // ncol for s in bounds}) == split
    q, v, _, _, ctrl, _ = _tiled(robot, 30, seed=12)
    idx = np.arange(n) % len(q)
    q, v, ctrl = (x[idx] for x in (q, v, ctrl))
    t = backend.t
    big = _production(backend, monkeypatch, cfg, nenv, wpb, ragged=nenv % (wpb * EPW) != 0)
    small = backend.batch(cfg, ONE_WARP_ENVS[backend.name])
    assert _wpb(small) == 1
    outs = [{k: x.cpu().numpy() for k, x in e.transition_fd(t(q), t(v), t(ctrl), dqacc=True).items()} for e in (big, small)]
    _bit_equal(_bits(outs[0]), _bits(outs[1]), f"{wpb}-warp launches of {nenv} slots vs 1-warp launches")
    assert (outs[0]["flags"] == 0).mean() > 0.5


# ------------------------------------------------------------------ 6. SMPL-X A / B against whole oracle steps
def test_smplx_AB_matches_full_step_oracle(backend):
    """test_AB_matches_full_step_oracle on SMPL-X: a row with floor contacts and an airborne row, the root spun up as there.  A - I
    and B against an fp64 FD of whole oracle steps (Frobenius, relative, on columns neither side flags); the root-rotation rows on
    their own."""
    robot = "smplx_humanoid"
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    nv = m.nv
    qc, vc, _ = _rollout(robot, 6, 14)
    c = next(i for i in range(len(qc)) if _forward(om, qc[i], vc[i]).ncon > 0)
    qa, va = airborne_states(m, 1, seed=14)
    qa[:, 7:] *= 0.2
    q, v = np.float32(np.concatenate([qc[c:c + 1], qa])), np.float32(np.concatenate([vc[c:c + 1], va]))
    u = np.float32(np.random.default_rng(15).uniform(-30, 30, (2, m.nu)))
    v[:, 3:6] += np.float32([4.0, -6.0, 5.0])
    assert _forward(om, q[0], v[0], u[0]).ncon > 0 and _forward(om, q[1], v[1], u[1]).nefc == 0
    env = backend.batch(cfg, 64)
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u))
    A, B, F, qn = (fd[k].cpu().numpy().astype(np.float64) for k in ("A", "B", "flags", "qacc"))
    I = np.eye(2 * nv)
    worst = {}
    for i in range(2):
        Ao, Bo = oracle_AB(om, q[i], v[i], u[i], qn[i])
        ka, kb = F[i, :2 * nv] == 0, F[i, 2 * nv:] == 0
        assert ka.mean() > 0.8 and kb.mean() > 0.8, (i, ka.mean(), kb.mean())
        for name, K, O, keep in (("A - I", A[i] - I, Ao - I, ka), ("B", B[i], Bo, kb)):
            err = np.linalg.norm((K - O)[:, keep]) / max(1e-12, np.linalg.norm(O[:, keep]))
            worst[name] = max(worst.get(name, 0.0), err)
        rot = np.linalg.norm((A[i] - Ao)[3:6][:, ka]) / np.linalg.norm(Ao[3:6][:, ka])
        worst["rot rows"] = max(worst.get("rot rows", 0.0), rot)
    print("SMPL-X A / B:", {k: f"{x:.2e}" for k, x in worst.items()})
    assert all(worst[k] <= SMPLX_AB_TOL[k] for k in SMPLX_AB_TOL), worst


# ------------------------------------------------------------------ 7. both branches of the root-rotation assembly
def _skew(x):
    return np.array([[0.0, -x[2], x[1]], [x[2], 0.0, -x[0]], [-x[1], x[0], 0.0]])


def _rot_rows(m, h, dqacc, qacc, qvel):
    """Rows 3:6 of A and B in fp64 from the kernel's own dqacc [nv, ncol], nominal qacc and qvel: column j is R(th)^T e_k (root-rotation
    columns only) + J_r(th) h dv'[3:6], with dv' = h dqacc_j + [qvel column], th = h (v + h qacc)[3:6]."""
    nv = m.nv
    th = h * (qvel[3:6] + h * qacc[3:6])
    t = np.linalg.norm(th)
    S = _skew(th)
    Rt = np.eye(3) - np.sin(t) / t * S + (1 - np.cos(t)) / t ** 2 * S @ S
    Jr = np.eye(3) - (1 - np.cos(t)) / t ** 2 * S + (t - np.sin(t)) / t ** 3 * S @ S
    dv = h * dqacc[3:6].copy()
    dv[:, nv + 3:nv + 6] += np.eye(3)
    r = Jr @ (h * dv)
    r[:, 3:6] += Rt
    return r[:, :2 * nv], r[:, 2 * nv:]


def test_rotation_rows_both_branches(backend):
    """Airborne SMPL rows (no constraint rows, no kinks) with the root spun so that |th| = |h (v + h qacc_nom)[3:6]| is 0.02, 0.0999,
    0.1001, 0.3 and 1.0 (about 9 to 450 rad/s).  (a) A[:, 3:6] and B[:, 3:6] equal their fp64 restatement from the kernel's own
    dqacc, qacc and qvel to ROT_TOL on both sides of the series / closed-form switch at |th| = 0.1; (b) against oracle_AB, which checks
    the definition (the tangent of q (x) exp)."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    nv, h = m.nv, m.timestep
    k = len(THETAS)
    q, v = airborne_states(m, k, seed=41)
    q[:, 7:] *= 0.2
    q = np.float32(q)
    rng = np.random.default_rng(42)
    u = np.float32(rng.uniform(-30, 30, (k, m.nu)))
    d = rng.normal(size=(k, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    env = backend.batch(cfg, 8)
    target = np.array(THETAS)

    def theta(s):
        v[:, 3:6] = s[:, None] * d
        v32 = np.float32(v)
        qa = env.forward(backend.t(q), backend.t(v32), backend.t(u))["qacc"].cpu().numpy().astype(np.float64)
        return np.linalg.norm(h * (v32[:, 3:6] + h * qa[:, 3:6]), axis=1), v32

    # secant on the spin rate per row: qacc (gyroscopic terms) depends on it
    s0, s1 = target / h, 1.02 * target / h
    f0, f1 = theta(s0)[0] - target, theta(s1)[0] - target
    for _ in range(12):
        s2 = np.where(f1 != f0, s1 - f1 * (s1 - s0) / np.where(f1 != f0, f1 - f0, 1.0), s1)
        s0, f0, s1 = s1, f1, s2
        f1 = theta(s1)[0] - target
    th, v = theta(s1)
    assert np.all(np.abs(th - target) <= 2e-5 * target), th
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), dqacc=True)
    A, B, K, F, qn = (fd[x].cpu().numpy().astype(np.float64) for x in ("A", "B", "dqacc", "flags", "qacc"))
    assert (F == 0).all()
    tk = np.linalg.norm(h * (v[:, 3:6].astype(np.float64) + h * qn[:, 3:6]), axis=1)
    assert (tk ** 2 < 1e-2).tolist() == [x < 0.1 for x in THETAS], tk    # the rows on each side of the kernel's switch
    I = np.eye(2 * nv)
    worst = {"assembly A": 0.0, "assembly B": 0.0, "A - I": 0.0, "B": 0.0, "rot rows": 0.0}
    for i in range(k):
        Ar, Br = _rot_rows(m, h, K[i], qn[i], v[i].astype(np.float64))
        ea = np.linalg.norm(A[i, 3:6] - Ar) / np.linalg.norm(Ar)
        eb = np.linalg.norm(B[i, 3:6] - Br) / np.linalg.norm(Br)
        assert ea <= ROT_TOL and eb <= ROT_TOL, (THETAS[i], ea, eb)
        Ao, Bo = oracle_AB(om, q[i], v[i], u[i], qn[i])
        errs = {"A - I": np.linalg.norm(A[i] - Ao) / np.linalg.norm(Ao - I), "B": np.linalg.norm(B[i] - Bo) / np.linalg.norm(Bo),
                "rot rows": np.linalg.norm((A[i] - Ao)[3:6]) / np.linalg.norm(Ao[3:6])}
        print(f"|th| = {tk[i]:.5f}, max|qacc| {np.abs(qn[i]).max():.1e}: assembly A {ea:.1e}, B {eb:.1e}; oracle "
              + ", ".join(f"{x} {y:.1e}" for x, y in errs.items()))
        tol = SPIN_AB_TOL[0.3 if THETAS[i] <= 0.3 else 1.0]
        assert all(errs[x] <= tol[x] for x in tol), (THETAS[i], errs)
        worst = {x: max(worst[x], y) for x, y in {"assembly A": ea, "assembly B": eb, **errs}.items()}
    print({x: f"{y:.2e}" for x, y in worst.items()})


# ------------------------------------------------------------------ 8. the kink flag against the oracle's active-set switches
def _band(om, q, v, u, eps):
    """Per column: either perturbed oracle state has a contact or a row inside the guard band (_near_switch)."""
    m = om.model
    ncol = 2 * m.nv + m.nu
    out = np.zeros(ncol, bool)
    for j in range(ncol):
        e = eps[0] if j < m.nv else eps[1] if j < 2 * m.nv else eps[2]
        for s in (e, -e):
            o = _oracle_env(om, *_perturb(m, q, v, u, j, s))
            o.forward()
            out[j] |= _near_switch(o, o.qacc)
    return out


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_kink_flags_match_oracle_switches(backend, robot):
    """SMPLSIM_FD_KINK against the oracle's own active-set switches (oracle_dqacc's `switched`) on the states of
    test_dqacc_matches_oracle plus _pool's lying state and two of its limit states, in both directions: outside the guard band every
    switched column carries bit 1, and every bit-1 column switched or lies inside the band.  Columns with SMPLSIM_FD_SOLVER are not
    compared."""
    n = 4 if robot == "smpl_humanoid" else 2
    cfg, om, q, v, u = _states(robot, n, seed=11, nair=1)
    m = om.model
    qp, vp, _, kinds = _pool(robot)
    pick = [kinds.index("lying")] + [i for i, kd in enumerate(kinds) if kd == "limit"][:2]
    q = np.concatenate([q, np.float32(qp[pick])])
    v = np.concatenate([v, np.float32(vp[pick])])
    u = np.concatenate([u, np.float32(np.random.default_rng(12).uniform(-30, 30, (len(pick), m.nu)))])
    env = backend.batch(cfg, 64)
    fd = env.transition_fd(backend.t(q), backend.t(v), backend.t(u), dqacc=True)
    F = fd["flags"].cpu().numpy()
    K = fd["dqacc"].cpu().numpy().astype(np.float64)
    tot = {"switched": 0, "flagged": 0, "band": 0, "solver": 0, "switched outside the band": 0}
    for i in range(len(q)):
        e = _forward(om, q[i], v[i], u[i])
        O, sw = oracle_dqacc(om, q[i], v[i], u[i], EPS)
        band = _band(om, q[i], v[i], u[i], EPS)
        kink, solver = (F[i] & 1) != 0, (F[i] & 2) != 0
        cmp = ~solver
        miss = np.flatnonzero(cmp & sw & ~band & ~kink)
        extra = np.flatnonzero(cmp & kink & ~sw & ~band)
        assert not len(miss), (i, "switched columns without bit 1", miss[:8])
        assert not len(extra), (i, "bit-1 columns the oracle does not switch", extra[:8])
        if e.ncon > 0:
            assert (sw & ~band & cmp).sum() >= 1, (i, "no switched column outside the band")
        # unflagged columns still hold test_dqacc_matches_oracle's accuracy
        col, blk = dqacc_errors(m, K[i], O, (F[i] == 0) & ~sw)
        assert col <= 1e-2 and blk <= 2e-2, (i, col, blk)
        tot = {"switched": tot["switched"] + int(sw.sum()), "flagged": tot["flagged"] + int(kink.sum()),
               "band": tot["band"] + int(band.sum()), "solver": tot["solver"] + int(solver.sum()),
               "switched outside the band": tot["switched outside the band"] + int((sw & ~band & cmp).sum())}
    # both backends: SMPL 33 switched columns of 7 x 219, all flagged, none in the band; SMPL-X 29 of 5 x 471, all flagged, 22 outside
    # the band
    print(f"{robot}: {len(q)} rows x {F.shape[1]} columns: {tot}")
