"""Batched rollouts (smplsim_rollout, k_roll5) and the inverse-dynamics FD derivatives (smplsim_inverse_fd, k_invfd5) on every launch
path and at their edges, against the fp64 oracle, against the env path and against 1-warp CTAs.

test_rollout and test_inverse_fd hold the two calls to the oracle on a few rows in 1-warp CTAs, from well-behaved states.  Here the
same kernels run where production runs them and where their rarer branches live:

- rollouts at the production CTA shapes (8-warp SMPL with a ragged second launch, 4-warp SMPL-X) from the mixed state pool: the lying
  state whose contact entries overflow to global scratch, the state whose qacc overflows (mj_checkAcc resets it inside the substep,
  and in ctrl mode hands the caller's ctrl back to the next substep), states past their joint limits;
- long horizons under stale-inertia stable PD, each step boundary crossing the scratch rows and l_spd_prologue, with an auto-reset in
  the middle; the fresh-inertia, unclipped-action and ctrl-mode branches on every controller; the outputs a caller may leave out and
  handle state the rollout must not take; per-env parameter records (k_roll5<WithPrm>) and body shapes at the production size;
- inverse_fd's forward differences (their own minuend and denominator), its column launches split over launches of num_envs slots,
  SMPL-X, bad rows next to good ones, each output alone at the C ABI and non-default eps.

As in test_cta_shapes, the GPU reaches the production CTA shapes by env count alone and the emulator forces them with SMPLSIM_WPB at a
few dozen envs; every test asserts the CTA shape it ran."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from smplsim_b200.abi import SmplsimInverseFdCfgC, model_from_cfg  # noqa: E402
from test_cta_shapes import (CHUNK, EPW, N_DYN, N_SHAPES, N_SMPL, N_SMPLX, NCS, _bit_equal, _check_row, _dups_equal,  # noqa: E402
                             _one_warp_chunks, _oracle_step, _pool, _production, _tiled, _wpb)
from test_env_params import draw, oracle_for  # noqa: E402
from test_forward_fd import _oracle_env  # noqa: E402
from test_forward_fd_paths import ONE_WARP_ENVS, _bits, _past_cap  # noqa: E402
from test_gpu_parity import _shape_variant  # noqa: E402
from test_inverse import _forward, _over_cap, ref_inverse  # noqa: E402
from test_inverse_fd import (BLOCK_TOL, COL_TOL, EPS, KINK, SOLVER, _inv_states, _perturb3, _row_set, dfrc_errors,  # noqa: E402
                             oracle_dfrc)
from test_rollout import _env_path  # noqa: E402
from test_xfrc import _wrenches  # noqa: E402
from util_states import make_models, relerr, rollout_states  # noqa: E402

ROBOT = "smpl_humanoid"
T_PROD = {"gpu": 3, "emu": 2}                  # steps of the production-shape rollouts
N_LONG, T_LONG = {"gpu": 1024, "emu": 7}, 28    # rows and action steps of the long horizon
N_BRANCH = {"gpu": 600, "emu": 9}              # rows of the configuration-branch rollouts (the pool's first kinds, bad state included)


def _np(d):
    return {k: x.cpu().numpy().copy() for k, x in d.items()}


def _controls(m, P, T, mode, seed, scale=None):
    """Per pool state: ctrl-mode torques U(-80, 80) (those of _tiled), action-mode actions N(0, 0.4) (or U(-scale, scale))."""
    rng = np.random.default_rng(seed)
    if mode == "ctrl":
        return np.float32(rng.uniform(-80, 80, (P, T, m.nu)))
    if scale is not None:
        return np.float32(rng.uniform(-scale, scale, (P, T, m.nu)))
    return np.float32(rng.normal(size=(P, T, m.nu)) * 0.4)


def _roll(env, t, q, v, w, u, mode, nsub, poses=False, **kw):
    kw = dict(kw, mode=mode, body_poses=poses)
    if mode == "ctrl":
        kw["nsub"] = nsub
    return _np(env.rollout(t(q), t(v), t(u), qacc_warmstart=t(w), **kw))


def _env_ref(backend, cfg, q, v, w, u, mode, nsub, keys, **kw):
    ref = _np(_env_path(backend, cfg, q, v, w, u, mode, nsub, **kw))
    return {k: ref[k] for k in keys}


def _check_steps(backend, fenv, got, q, v, w, U, first, oracle_of, kinds, tol, m, check=_check_row):
    """Every recorded step t of a ctrl-mode rollout (nsub = 1) of rows `first` against one oracle mj_step from the kernel's own state at
    t - 1 (test_rollout's test_steps_match_oracle), held to _check_row: state, status and guard band of that step, with the step's
    contact mask and qacc from a kernel forward pass at the same state, ctrl and warm start (fenv: a handle that takes all n rows).
    The overflowing state raises bit 4, resets and is an ordinary row from the next step on.  Returns the number of compared steps
    and the worst norm-relative qvel error of the ordinary rows."""
    t_ = backend.t
    ncmp, worst = 0, 0.0
    for t in range(U.shape[1]):
        q0 = q if t == 0 else got["qpos"][:, t - 1]
        v0 = v if t == 0 else got["qvel"][:, t - 1]
        w0 = w if t == 0 else np.zeros_like(v0)
        f = _np(fenv.forward(t_(q0), t_(v0), t_(U[:, t]), qacc_warmstart=t_(w0)))
        r = {"qpos": got["qpos"][:, t], "qvel": got["qvel"][:, t], "status": got["status"][:, t], "contact_mask": f["contact_mask"],
             "qacc": f["qacc"]}
        for i in first:
            e = _oracle_step(oracle_of(i), q0[i], v0[i], w0[i], U[i, t])
            kind = kinds[i] if t == 0 else "reset" if kinds[i] == "bad" else kinds[i]
            if check(e, r, i, tol, m, kind):
                ncmp += 1
                if kind != "bad":
                    worst = max(worst, relerr(r["qvel"][i], e.qvel))
    return ncmp, worst


# ------------------------------------------------------------------ 1. rollouts at the production CTA shapes
@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_rollout_at_production_shape(backend, monkeypatch, robot):
    """The _pool states tiled over the rows, each with its pool warm start and its own control rows: SMPL on an 8-warp handle with
    num_envs rows plus a ragged second launch, SMPL-X on a 4-warp handle with a ragged last CTA.  Ctrl mode with nsub = 1 and 3 and
    action mode under stable PD with stale inertia (poses on), each (a) bit-identical with 1-warp CTAs and across rows of the same pool
    state, (b) bit-identical with the env path (set_state + T step / mj_step calls); (c) ctrl mode with nsub = 1 against one oracle
    mj_step per recorded step from the kernel's own state, per pool state."""
    cfg, om = make_models(robot=robot, control_mode="uhc_pd")
    m = om.model
    if robot == ROBOT:
        nenv, extra = N_DYN[backend.name]
        env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
        assert extra % (8 * EPW) != 0
    else:
        nenv, extra = N_SMPLX[backend.name], 0
        env = _production(backend, monkeypatch, cfg, nenv, 4)
    n = nenv + extra
    q, v, w, kinds, _, idx = _tiled(robot, n)
    P, T = len(q), T_PROD[backend.name]
    t = backend.t
    bad = [k for k in range(P) if kinds[k] == "bad"]
    for mode, nsub in (("ctrl", 1), ("ctrl", 3), ("action", None)):
        U = _controls(m, P, T, mode, seed=20 + (nsub or 0))
        poses = mode == "action"

        def run(e, s):
            return _roll(e, t, q[idx[s]], v[idx[s]], w[idx[s]], U[idx[s]], mode, nsub, poses)

        got = run(env, slice(0, n))
        what = f"{robot} {mode} nsub={nsub}"
        _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), what + ": vs 1-warp CTAs")
        _dups_equal(got, idx, what + ": same pool state")
        _bit_equal(got, _env_ref(backend, cfg, q[idx], v[idx], w[idx], U[idx], mode, nsub, got.keys()), what + ": vs env path")
        for k in bad:   # mj_checkAcc at step 0: bit 4, the reset state, and on from there
            assert got["status"][k, 0] & 4 and not got["status"][k, 1:].any(), (what, got["status"][k])
        assert np.isfinite(got["qpos"]).all() and np.isfinite(got["qvel"]).all(), what
        if mode == "ctrl" and nsub == 1:
            # test_cta_shapes' mj_step bounds.  Worst norm-relative qvel error, SMPL / SMPL-X: 5.2e-5 / 1.0e-4 on the emulator, 7.9e-5 /
            # 9.5e-5 on an H100
            tol = 1e-4 if robot == ROBOT else 2e-4
            ncmp, worst = _check_steps(backend, env, got, q[idx], v[idx], w[idx], U[idx], range(P), lambda i: om, kinds, tol, m)
            print(f"{what}: {ncmp}/{P * T} pool-state steps against the oracle, worst qvel {worst:.2e}")
            assert ncmp >= P * T - 3 * T, ncmp


# ------------------------------------------------------------------ 2. a long horizon with an auto-reset in the middle
@pytest.mark.parametrize("poses", [True, False])
def test_long_horizon_matches_env_path(backend, monkeypatch, poses):
    """T_LONG action steps under stable PD with stale inertia (every step boundary goes through the scratch rows and l_spd_prologue)
    from the pool states on the 8-warp production handle, a NaN action row at step T_LONG // 2 on every fifth row: every recorded step
    bit-identical with the env path; the NaN rows raise their bit, reset and run on for the rest of the horizon."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    n = N_LONG[backend.name]
    q, v, w, kinds = _pool(ROBOT)
    idx = np.arange(n) % len(q)
    q, v, w = q[idx], v[idx], w[idx]
    u = _controls(m, n, T_LONG, "action", seed=31)
    tn = T_LONG // 2
    nan_rows = np.arange(1, n, 5)
    u[nan_rows, tn] = np.nan
    env = _production(backend, monkeypatch, cfg, N_DYN[backend.name][0], 8, ragged=False)
    got = _roll(env, backend.t, q, v, w, u, "action", None, poses)
    _bit_equal(got, _env_ref(backend, cfg, q, v, w, u, "action", None, got.keys()), f"{T_LONG} steps, poses={poses}: vs env path")
    st = got["status"]
    assert (st[nan_rows, tn] & 7).all(), st[nan_rows, tn]
    assert np.isfinite(got["qpos"]).all()
    # after the reset the row moves again: its later steps are not the reset state
    assert not np.array_equal(got["qpos"][nan_rows[0], -1], got["qpos"][nan_rows[0], tn])


# ------------------------------------------------------------------ 3. configuration branches against the env path
BRANCHES = {   # case: (handle overrides, mode, nsub, action scale)
    "spd_fresh": (dict(control_mode="uhc_pd", spd_inertia="fresh"), "action", None, None),
    "no_clip": (dict(control_mode="uhc_pd", clip_actions=False), "action", None, 3.0),
    "ctrl_uhc_pd": (dict(control_mode="uhc_pd"), "ctrl", 2, None),
    "ctrl_pd": (dict(control_mode="pd"), "ctrl", 2, None),
    "ctrl_simple_pid": (dict(control_mode="simple_pid"), "ctrl", 2, None),
}


@pytest.mark.parametrize("case", list(BRANCHES))
def test_config_branches_match_env_path(backend, monkeypatch, case):
    """Stable PD with fresh inertia (l_substeps' spd && !stale branch; the rollout writes no forward-state rows), unclipped actions up
    to 3 in magnitude, and ctrl mode (nsub = 2: the overflowing state's reset hands the caller's ctrl back to the second substep) on
    uhc_pd, pd and simple_pid handles, on the 8-warp production handle: bit-identical with the env path."""
    ov, mode, nsub, scale = BRANCHES[case]
    cfg, om = make_models(**ov)
    m = om.model
    n = N_BRANCH[backend.name]
    q, v, w, kinds = _pool(ROBOT)
    idx = np.arange(n) % len(q)
    assert "bad" in [kinds[i] for i in idx]
    q, v, w = q[idx], v[idx], w[idx]
    u = _controls(m, n, 3, mode, seed=41, scale=scale)
    env = _production(backend, monkeypatch, cfg, N_DYN[backend.name][0], 8, ragged=False)
    got = _roll(env, backend.t, q, v, w, u, mode, nsub, True)
    _bit_equal(got, _env_ref(backend, cfg, q, v, w, u, mode, nsub, got.keys()), f"{case}: vs env path")
    if case == "no_clip":   # the actions past 1 are taken: the clipped handle gives another trajectory
        clip = _roll(backend.batch(make_models(control_mode="uhc_pd")[0], n), backend.t, q, v, w, u, mode, nsub)
        assert not np.array_equal(clip["qvel"], got["qvel"])


# ------------------------------------------------------------------ 4. handle state and output selection
def test_wrench_handle_and_status_off(backend):
    """A handle whose xfrc_applied is set (and pushed through a step) with contact_wrench=True rolls out bit for bit what a plain handle
    does, in action and ctrl mode, poses included: xfrc_applied is not taken.  status=False (NULL status) leaves qpos, qvel and the
    poses bit-identical."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    n = 8
    q, v, w, _ = _pool(ROBOT)
    q, v, w = q[:n], v[:n], w[:n]
    t = backend.t
    plain = backend.batch(cfg, n)
    wrench = backend.batch(cfg, n, contact_wrench=True)
    assert _wpb(plain) == 1 and _wpb(wrench) == 1
    wrench.xfrc_applied = t(_wrenches(m, n, np.random.default_rng(51)))
    wrench.step(t(np.zeros((n, m.nu))))
    assert np.abs(wrench.contact_wrench.cpu().numpy()).max() > 0
    for mode, nsub in (("action", None), ("ctrl", 2)):
        u = _controls(m, n, 2, mode, seed=52)
        a = _roll(plain, t, q, v, w, u, mode, nsub, True)
        _bit_equal(_roll(wrench, t, q, v, w, u, mode, nsub, True), a, f"{mode}: wrench handle vs plain handle")
        off = _roll(plain, t, q, v, w, u, mode, nsub, True, status=False)
        assert "status" not in off
        _bit_equal(off, {k: a[k] for k in ("qpos", "qvel", "xpos", "xquat")}, f"{mode}: status=False")


# ------------------------------------------------------------------ 5. per-env parameter records and body shapes at production size
# Worst norm-relative qvel error under these rules (bound 2e-4): records 1.0e-4 on the emulator, 1.8e-4 on an H100; body shapes 4.7e-5
# on the emulator, 6.4e-5 on an H100.  The steps after the first start the oracle's solve from zeros and the kernel's from its own
# warm start, as in test_rollout's test_steps_match_oracle.
def _check_norms(e, r, i, tol, m, kind):
    """One step of a row with a parameter record or a body shape of its own against that row's oracle e, by the feature tests' rules
    for one mj_step (test_env_params' check_mj_step, test_gpu_parity's test_per_env_body_shapes_match_oracle): contact mask exact, qvel
    to 2 tol and qpos to tol norm-relative, no per-element bound; a contact in the guard band is not compared."""
    con = e.contacts()
    if e.ncon and (np.abs(con["dist"] - m.margin) < 1e-5).any():
        return False
    assert not r["status"][i] & (1 | 2 | 4 | 8 | 16), (i, kind, r["status"][i])
    assert int(r["contact_mask"][i]) == e.contact_mask, (i, kind, bin(int(r["contact_mask"][i])), bin(e.contact_mask))
    assert relerr(r["qvel"][i], e.qvel) < 2 * tol and relerr(r["qpos"][i], e.qpos) < tol, (i, relerr(r["qvel"][i], e.qvel))
    return True


def test_rollout_with_parameter_records(backend, monkeypatch):
    """An SMPL handle with draw() records on every env, n == num_envs, at the 8-warp production shape (k_roll5<WithPrm>): ctrl-mode
    steps of each pool state against the oracle of its env's variant model (test_env_params' bounds), bit-identical with 1-warp CTAs
    and across rows of the same pool state and record.  The overflowing state raises bit 4 and is not compared."""
    cfg, _ = make_models(control_mode="uhc_pd")
    m = model_from_cfg(cfg)
    n = N_SMPL[backend.name]
    q, v, w, kinds, _, idx = _tiled(ROBOT, n, seed=8)
    P, T = len(q), T_PROD[backend.name]
    prm = draw(m, P, 83)
    U = _controls(m, P, T, "ctrl", seed=84)
    t = backend.t

    def run(e, s):
        e.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        return _roll(e, t, q[idx[s]], v[idx[s]], w[idx[s]], U[idx[s]], "ctrl", 1)

    env = _production(backend, monkeypatch, cfg, n, 8)
    got = run(env, slice(0, n))
    _bit_equal(got, _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run), "records: 8-warp vs 1-warp CTAs")
    _dups_equal(got, idx, "records: same pool state")
    oms = {}
    bad = [k for k in range(P) if kinds[k] == "bad"]
    assert all(got["status"][k, 0] & 4 for k in bad), got["status"][bad]
    first = [k for k in range(P) if kinds[k] != "bad"]
    ncmp, worst = _check_steps(backend, env, got, q[idx], v[idx], w[idx], U[idx], first,
                               lambda i: oms.setdefault(i, oracle_for(cfg, m, prm, i)), kinds, 1e-4, m, check=_check_norms)
    print(f"records: {ncmp}/{len(first) * T} pool-state steps against the variant oracles, worst qvel {worst:.2e}")
    assert ncmp >= len(first) * T - 2 * T, ncmp


def test_rollout_per_env_shapes(backend, monkeypatch, tmp_path):
    """Three body shapes interleaved in ragged groups (every shape's last CTA has empty slots) at the 8-warp production shape: ctrl-mode
    steps of each row against its own shape's oracle (test_per_env_body_shapes_match_oracle's bounds), bit-identical with 1-warp CTAs
    and across rows of the same shape and state."""
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]

    def mk(k):
        return make_models(control_mode="uhc_pd", **({"robot.xml_path": paths[k]} if paths[k] else {}))
    n = N_SHAPES[backend.name]
    env_model = np.array([(i * 7 + i // 5) % 3 for i in range(n)], dtype=np.int32)
    assert (np.bincount(env_model) % (8 * EPW) != 0).all()
    made = [mk(k) for k in range(3)]
    oms = [x[1] for x in made]
    cfg0 = made[0][0]
    models = [model_from_cfg(x[0]) for x in made]
    m = models[0]
    pools = [rollout_states(oms[k], 12, seed=30 + k, every=9) for k in range(3)]
    pidx = np.zeros(n, dtype=np.int64)
    seen = [0, 0, 0]
    for i, k in enumerate(env_model):
        pidx[i] = seen[k] % 12
        seen[k] += 1
    q, v, w = (np.float32([pools[k][j][pidx[i]] for i, k in enumerate(env_model)]) for j in range(3))
    T = T_PROD[backend.name]
    U = _controls(m, 12, T, "ctrl", seed=61)[pidx]
    t = backend.t

    def run(e, s):
        return _roll(e, t, q[s], v[s], w[s], U[s], "ctrl", 1)

    env = _production(backend, monkeypatch, cfg0, n, 8, models=models, env_model=env_model)
    got = run(env, slice(0, n))
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg0, s.stop - s.start, models=models, env_model=env_model[s]), run,
                           chunk=CHUNK - 12)
    _bit_equal(got, ref, "per-env shapes: 8-warp vs 1-warp CTAs")
    key = env_model * 12 + pidx
    _dups_equal(got, np.unique(key, return_inverse=True)[1], "same shape and state")
    first = [int(np.flatnonzero(key == kk)[0]) for kk in np.unique(key)]
    kinds = ["rollout"] * n
    ncmp, worst = _check_steps(backend, env, got, q, v, w, U, first, lambda i: oms[env_model[i]], kinds, 1e-4, m, check=_check_norms)
    print(f"per-env shapes: {ncmp}/{len(first) * T} steps against the oracle, worst qvel {worst:.2e}")
    assert ncmp >= len(first) * T - 2 * T, ncmp


# ------------------------------------------------------------------ 6. inverse_fd: forward differences
def oracle_dfrc_forward(om, q, v, a, eps, cols):
    """One-sided fp64 FD of ref_inverse at the fp32 state on columns cols; per column whether the oracle's row set switched."""
    m = om.model
    nv = m.nv
    o = _oracle_env(om, q.astype(np.float64), v.astype(np.float64), np.zeros(m.nu))
    o.forward()
    f0, s0 = ref_inverse(o, a.astype(np.float64))[0], _row_set(o, a.astype(np.float64))
    D = np.zeros((nv, 3 * nv)); switched = np.zeros(3 * nv, bool)
    for j in cols:
        e = eps[j // nv]
        qq, vv, aa = _perturb3(m, q, v, a, j, e)
        o = _oracle_env(om, qq, vv, np.zeros(m.nu))
        o.forward()
        D[:, j] = (ref_inverse(o, aa)[0] - f0) / e
        switched[j] = _row_set(o, aa) != s0
    return D, switched


def _shifted(t, col, nv, e):
    """The (qpos, qvel, qacc) tensors t with column col (not a root-rotation one) moved by e; (tensor index, entry)."""
    k, j = (0, col + 1 if col >= 6 else col) if col < nv else (1, col - nv) if col < 2 * nv else (2, col - 2 * nv)
    tp = [x.clone() for x in t]
    tp[k][:, j] += e
    return tp, k, j


# (a) dfrc with centered=False against the one-sided oracle FD at the same eps (no truncation error between them), per column and per
# block as test_dfrc_matches_oracle: fp32 rounding of qfrc_inverse over eps instead of 2 eps.  Worst seen (column, block, root-rotation
# columns): 5.7e-4, 5.1e-4, 5.7e-4 on the emulator; 3.0e-4, 4.2e-4, 2.3e-4 on an H100.
FWD_COL_TOL, FWD_BLOCK_TOL = COL_TOL, BLOCK_TOL
NONROT_COLS = (0, 2, 6, 40, 74, 75, 78, 95, 149, 150, 155, 183, 224)   # SMPL: root translation, hinges, qvel, qacc


def test_inverse_fd_forward_differences(backend):
    """centered=False: dfrc against a one-sided fp64 oracle FD at the same eps on rows and columns the oracle does not switch (the
    root-rotation columns on their own); non-rotation columns bit for bit (inverse(x+) - inverse(x)) / (x+ - x), the minuend being
    each row's own nominal pass; qfrc_inverse bit-identical with the centered call and with inverse(); no KINK flags."""
    cfg, om, q, v, a, _ = _inv_states(ROBOT, 4, seed=11)
    nv = om.model.nv
    env = backend.batch(cfg, 64)
    assert _wpb(env) == 1
    tt = [backend.t(x) for x in (q, v, a)]
    f = env.inverse_fd(*tt, centered=False)
    c = env.inverse_fd(*tt)
    nom = env.inverse(*tt)
    assert torch.equal(f["qfrc_inverse"], c["qfrc_inverse"]) and torch.equal(f["qfrc_inverse"], nom)
    F = f["flags"].cpu().numpy()
    assert not (F & KINK).any()
    for col in NONROT_COLS:
        tp, k, j = _shifted(tt, col, nv, EPS[col // nv])
        want = (env.inverse(*tp) - nom) / (tp[k][:, j] - tt[k][:, j])[:, None]
        assert torch.equal(f["dfrc"][:, :, col], want), col
    K = f["dfrc"].cpu().numpy().astype(np.float64)
    worst = [0.0, 0.0, 0.0]
    nrot = 0
    for i in range(len(q)):
        O, sw = oracle_dfrc_forward(om, q[i], v[i], a[i], EPS, range(3 * nv))
        keep = (F[i] == 0) & ~sw
        assert keep.mean() >= 0.95, (i, keep.mean())
        col, blk = dfrc_errors(nv, K[i], O, keep)
        rk = np.flatnonzero(keep[3:6]) + 3
        rot = np.abs(K[i][:, rk] - O[:, rk]).max() / max(1.0, np.abs(O[:, :nv]).max()) if len(rk) else 0.0
        nrot += len(rk)
        worst = [max(worst[0], col), max(worst[1], blk), max(worst[2], rot)]
    print(f"centered=False: worst column {worst[0]:.2e}, block {worst[1]:.2e}, rotation columns {worst[2]:.2e} ({nrot} compared)")
    assert nrot >= 9
    assert worst[0] <= FWD_COL_TOL and worst[1] <= FWD_BLOCK_TOL and worst[2] <= FWD_COL_TOL, worst


# ------------------------------------------------------------------ 7. inverse_fd: column launches split over launch boundaries
# (num_envs, rows, warps per CTA, rows whose columns straddle a launch boundary); launches are of num_envs slots each
INVFD_LAUNCH = {"gpu": {"smpl_humanoid": (4096, 41, 8, [18, 36]),       # 9 225 slots: 4 096 + 4 096 + 1 033 (ragged)
                        "smplx_humanoid": (2049, 9, 4, [4, 8])},        # 4 293 slots: 2 049 + 2 049 + 195
                "emu": {"smpl_humanoid": (40, 2, 8, [0, 1]),            # 450 slots in 12 launches of 40 (the last 10)
                        "smplx_humanoid": (17, 2, 4, [0, 1])}}          # 954 slots in 57 launches of 17 (the last 2)


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_inverse_fd_launch_shapes(backend, monkeypatch, robot):
    """inverse_fd on a production handle, whose launches of num_envs slots split rows, against a 1-warp handle whose launches split
    them elsewhere and against a handle with a slot per column, which runs them all in one launch: qfrc_inverse, dfrc and flags
    bit-identical, compared as bit patterns (the pool's overflowing state has NaN columns)."""
    nenv, n, wpb, split = INVFD_LAUNCH[backend.name][robot]
    cfg, om = make_models(robot=robot, control_mode="torque")
    ncol = 3 * om.model.nv
    bounds = range(nenv, n * ncol, nenv)
    assert all(s % ncol for s in bounds)                           # every launch boundary falls inside a row
    assert sorted({s // ncol for s in bounds}) == split
    q, v, _, _, _, _ = _tiled(robot, 30, seed=12)
    idx = np.arange(n) % len(q)
    a = np.float32(np.random.default_rng(13).normal(size=(len(q), om.model.nv)) * 5.0)
    q, v, a = (x[idx] for x in (q, v, a))
    t = backend.t
    big = _production(backend, monkeypatch, cfg, nenv, wpb, ragged=nenv % (wpb * EPW) != 0)
    small = backend.batch(cfg, ONE_WARP_ENVS[backend.name])
    assert _wpb(small) == 1
    one = backend.batch(cfg, n * ncol)
    outs = [_np(e.inverse_fd(t(q), t(v), t(a))) for e in (big, small, one)]
    _bit_equal(_bits(outs[0]), _bits(outs[1]), f"{wpb}-warp launches of {nenv} slots vs 1-warp launches")
    _bit_equal(_bits(outs[0]), _bits(outs[2]), f"{wpb}-warp launches of {nenv} slots vs one launch")
    assert (outs[0]["flags"] == 0).mean() > 0.5


# ------------------------------------------------------------------ 8. inverse_fd on SMPL-X
def test_inverse_fd_smplx_edges(backend):
    """SMPL-X: root-translation, hinge, qvel and qacc columns bit for bit (inverse(x+) - inverse(x-)) / (x+ - x-); the qacc block equal to
    M + J^T diag(D [r < 0]) J of the oracle on unflagged columns."""
    cfg, om, q, v, a, _ = _inv_states("smplx_humanoid", 2, seed=23)
    m = om.model
    nv = m.nv
    env = backend.batch(cfg, 64)
    assert _wpb(env) == 1
    tt = [backend.t(x) for x in (q, v, a)]
    fd = env.inverse_fd(*tt)
    assert torch.equal(fd["qfrc_inverse"], env.inverse(*tt))
    for col in (1, 6, 70, nv - 1, nv, nv + 4, nv + 100, 2 * nv - 1, 2 * nv, 2 * nv + 9, 2 * nv + 120, 3 * nv - 1):
        e = EPS[col // nv]
        tp, k, j = _shifted(tt, col, nv, e)
        tm, _, _ = _shifted(tt, col, nv, -e)
        want = (env.inverse(*tp) - env.inverse(*tm)) / (tp[k][:, j] - tm[k][:, j])[:, None]
        assert torch.equal(fd["dfrc"][:, :, col], want), col
    K, F = fd["dfrc"].cpu().numpy().astype(np.float64)[:, :, 2 * nv:], fd["flags"].cpu().numpy()[:, 2 * nv:]
    worst, rows = 0.0, 0
    for i in range(len(q)):
        e = _forward(om, q[i], v[i])
        efc = e.efc()
        _, _, r = ref_inverse(e, a[i].astype(np.float64))
        H = e.M + efc["J"].T @ ((efc["D"] * (r < 0))[:, None] * efc["J"])
        keep = F[i] == 0
        assert keep.mean() >= 0.95, i
        err = np.linalg.norm(K[i][:, keep] - H[:, keep]) / np.linalg.norm(H[:, keep])
        worst = max(worst, err)
        rows += e.nefc > 0
    print(f"SMPL-X qacc block: worst {worst:.2e}")
    assert rows >= 1
    # test_qacc_block_structure's bound.  Worst seen: 4.5e-5 on the emulator, 4.6e-5 on an H100
    assert worst <= 1e-4, worst


# ------------------------------------------------------------------ 9. inverse_fd: bad rows among good ones
def test_inverse_fd_bad_rows(backend, monkeypatch):
    """On the 8-warp production handle: good rows (the lying state, whose contact entries overflow to global scratch, and rollout
    states) interleaved with the pool's overflowing state (qvel 8e9), an inf qvel, a NaN qacc, a qpos entry of 2e10 (finite, beyond
    mjMAXVAL) and a row past the joint-limit row cap.  Every column of a bad row has SOLVER; every good row is bit-identical with a
    call without the bad rows."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    nenv = N_DYN[backend.name][0]
    env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
    qp, vp, _, kinds = _pool(ROBOT)
    gi = [kinds.index("lying"), 1, 2]
    assert _forward(om, qp[gi[0]], vp[gi[0]]).ncon > NCS[ROBOT]
    good_q, good_v = np.float32(qp[gi]), np.float32(vp[gi])
    good_a = np.float32([_forward(om, good_q[i], good_v[i]).qacc.copy() for i in range(3)])
    bq, bv, ba = [], [], []

    def add(qq, vv, aa):
        bq.append(np.float32(qq)); bv.append(np.float32(vv)); ba.append(np.float32(aa))
    z = np.zeros(m.nv)
    add(qp[kinds.index("bad")], vp[kinds.index("bad")], z)
    x = good_v[1].copy(); x[0] = np.inf
    add(good_q[1], x, good_a[1])
    x = good_a[2].copy(); x[10] = np.nan
    add(good_q[2], good_v[2], x)
    x = good_q[1].copy(); x[9] = 2e10
    add(x, good_v[1], good_a[1])
    qc, vc = _past_cap(m, 5)
    assert _over_cap(_forward(om, qc, vc))
    add(qc, vc, z)
    # good, bad, bad, good, bad, bad, good, bad: bad and good rows share CTAs and launches
    order = [("g", 0), ("b", 0), ("b", 1), ("g", 1), ("b", 2), ("b", 3), ("g", 2), ("b", 4)]
    Q = np.float32([good_q[j] if s == "g" else bq[j] for s, j in order])
    V = np.float32([good_v[j] if s == "g" else bv[j] for s, j in order])
    A = np.float32([good_a[j] if s == "g" else ba[j] for s, j in order])
    good = np.array([i for i, (s, _) in enumerate(order) if s == "g"])
    badr = np.array([i for i, (s, _) in enumerate(order) if s == "b"])
    t = backend.t
    got = _np(env.inverse_fd(t(Q), t(V), t(A)))
    ref = _np(env.inverse_fd(t(Q[good]), t(V[good]), t(A[good])))
    _bit_equal(_bits({k: x[good] for k, x in got.items()}), _bits(ref), "inverse_fd: good rows next to bad rows")
    for r in badr:
        assert (got["flags"][r] & SOLVER).all(), (r, np.flatnonzero(~(got["flags"][r] & SOLVER).astype(bool))[:8])
    assert not (ref["flags"] & SOLVER).any()


# ------------------------------------------------------------------ 10. inverse_fd: one output at a time through the C ABI
def test_inverse_fd_output_selection(backend):
    """smplsim_inverse_fd with dfrc only (flags NULL) and with flags only (dfrc NULL), centered and not: the output written is bit for
    bit that of the call with both, and so is qfrc_inverse."""
    cfg, om, q, v, a, _ = _inv_states(ROBOT, 3, seed=29)
    nv = om.model.nv
    env = backend.batch(cfg, 32)
    assert _wpb(env) == 1
    L, h, s = env._L(), env._h, env._stream()
    t = backend.t
    tq, tv, ta = t(q), t(v), t(a)
    p = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None  # noqa: E731

    def call(centered, dfrc, flags):
        qf = t(np.full((3, nv), np.nan))
        D = t(np.full((3, nv, 3 * nv), np.nan)) if dfrc else None
        F = torch.full((3, 3 * nv), 0xAB, dtype=torch.uint8, device=tq.device) if flags else None
        cfgc = SmplsimInverseFdCfgC(*EPS, centered, 0)
        assert L.smplsim_inverse_fd(h, C.byref(cfgc), p(tq), p(tv), p(ta), 3, p(qf), p(D), p(F), s) == 0
        return {k: x.cpu().numpy() for k, x in (("qfrc_inverse", qf), ("dfrc", D), ("flags", F)) if x is not None}

    for centered in (1, 0):
        both = call(centered, True, True)
        assert np.isfinite(both["dfrc"]).all() and (both["flags"] != 0xAB).all()
        for dfrc, flags in ((True, False), (False, True)):
            one = call(centered, dfrc, flags)
            _bit_equal(_bits(one), _bits({k: both[k] for k in one}), f"centered={centered} dfrc={dfrc} flags={flags}")


# ------------------------------------------------------------------ 11. inverse_fd at non-default eps
EPS_ODD = (3e-3, 5e-2, 0.25)
# root-rotation columns at eps_qpos 0.3 and 1.0 against the centered oracle FD at the same eps (the same q (x) exp(+-eps e_k), so no
# truncation error between them): max|k - o| / max(1, max|o| of the dq block), on columns neither side flags or switches.  Worst seen:
# 1.4e-6 on the emulator, 1.1e-6 on an H100.
ROT_EPS_TOL = 1e-4


def test_inverse_fd_eps(backend):
    """At eps (3e-3, 5e-2, 0.25): root-translation, hinge, qvel and qacc columns bit for bit (inverse(x+) - inverse(x-)) / (x+ - x-).
    At eps_qpos 0.3 and 1.0: the root-rotation columns against the centered oracle FD at the same eps."""
    cfg, om, q, v, a, _ = _inv_states(ROBOT, 4, seed=37, nair=2)
    nv = om.model.nv
    env = backend.batch(cfg, 64)
    assert _wpb(env) == 1
    tt = [backend.t(x) for x in (q, v, a)]
    fd = env.inverse_fd(*tt, *EPS_ODD)
    for col in NONROT_COLS:
        e = EPS_ODD[col // nv]
        tp, k, j = _shifted(tt, col, nv, e)
        tm, _, _ = _shifted(tt, col, nv, -e)
        want = (env.inverse(*tp) - env.inverse(*tm)) / (tp[k][:, j] - tm[k][:, j])[:, None]
        assert torch.equal(fd["dfrc"][:, :, col], want), col
    worst, ncmp = 0.0, 0
    for eq in (0.3, 1.0):
        fd = env.inverse_fd(*tt, eps_qpos=eq)
        K, F = fd["dfrc"].cpu().numpy().astype(np.float64), fd["flags"].cpu().numpy()
        for i in range(len(q)):
            O, sw = oracle_dfrc(om, q[i], v[i], a[i], (eq, EPS[1], EPS[2]))
            keep = np.flatnonzero((F[i, 3:6] == 0) & ~sw[3:6]) + 3
            if len(keep):
                err = np.abs(K[i][:, keep] - O[:, keep]).max() / max(1.0, np.abs(O[:, :nv]).max())
                worst = max(worst, err)
                ncmp += len(keep)
    print(f"root-rotation columns at eps_qpos 0.3 / 1.0: {ncmp} compared, worst {worst:.2e}")
    assert ncmp >= 12       # the airborne rows at both eps at least
    assert worst <= ROT_EPS_TOL, worst
