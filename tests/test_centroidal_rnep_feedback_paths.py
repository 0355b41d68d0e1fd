"""Centroidal momentum (smplsim_centroidal, k_cent5), body accelerations / joint wrenches / IMU readings (smplsim_rne_post, k_rnep5) and
closed-loop rollouts (smplsim_rollout_feedback, k_rollfb5) on every kernel instance and launch path, against the fp64 references, against
1-warp CTAs and against each other.

test_centroidal, test_rne_post and test_rollout_feedback hold the three calls to their fp64 references on a few well-behaved rows in
1-warp CTAs; their production-shape tests only pin the 8-warp outputs to the 1-warp ones.  Here the references look at the rows and
instances those tests leave alone:

- the _pool states at the production CTA shapes (8-warp SMPL with num_envs rows plus a ragged second launch, 4-warp SMPL-X with a ragged
  last CTA): the lying state whose contact entries overflow to global scratch, states past their joint limits, the overflowing state;
- every template instance: k_cent5 on both classes, with and without self-collision (its overflow contact entries, where k_cent5 sums,
  lie elsewhere in each class's scratch) and parameter records; k_rnep5 and k_rollfb5 with records on SMPL-X; per-env body shapes;
- host paths no feature test reads: xfrc_applied and shared feedback references on a second launch, 64 IMU sites, control_applied ==
  NULL (the kernel's own u scratch), bad rows next to good ones, and the handle scratch that rollout, rollout(gains=...), rne_post and
  centroidal share (rne_post sums its joint wrenches in the rollout's step-boundary rows).

Every bound is the feature tests' own.  As in test_cta_shapes, the GPU reaches the production CTA shapes by env count alone and the
emulator forces them with SMPLSIM_WPB at a few dozen envs; every test asserts the CTA shape it ran.  The oracle runs once per pool state
and _dups_equal carries its verdict to every other row of that state."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
from smplsim_b200.abi import model_from_cfg  # noqa: E402
from test_centroidal import TOL_NE, _newton_euler, _np  # noqa: E402
from test_centroidal import _assert_within as cent_within  # noqa: E402
from test_centroidal import _errors as cent_errors  # noqa: E402
from test_cta_shapes import (CHUNK, EPW, N_DYN, N_SELF, N_SHAPES, N_SMPL, N_SMPLX, NCS, _bit_equal, _dups_equal,  # noqa: E402
                             _one_warp_chunks, _pool, _production, _shape_variant, _tiled)
from test_env_params import draw, oracle_for, variant  # noqa: E402
from test_forward_fd_paths import _bits, _past_cap  # noqa: E402
from test_inverse import _forward as _inv_forward  # noqa: E402
from test_inverse import _over_cap  # noqa: E402
from test_rne_post import TOL_ID, _check_identities, _f64, random_sites, ref_row  # noqa: E402
from test_rne_post import _assert_within as rnep_within  # noqa: E402
from test_rne_post import _errors as rnep_errors  # noqa: E402
from test_dynamics import _qmat  # noqa: E402
from test_rollout_feedback import _np_diff, _pre_states  # noqa: E402
from test_rollout_invfd_paths import T_PROD, _check_norms, _check_steps, _controls, _roll  # noqa: E402
from util_states import make_models, rollout_states  # noqa: E402

ROBOT = "smpl_humanoid"
ROBOTS = ["smpl_humanoid", "smplx_humanoid"]
ROLLOUT_ACTION, ROLLOUT_CTRL = 0, 1    # smplsim.h's rollout modes


def _prod(backend, monkeypatch, robot, cfg):
    """(handle, rows) at the production CTA shape: SMPL on an 8-warp handle of N_DYN envs, with num_envs rows plus a ragged 8-warp second
    launch; SMPL-X on a 4-warp handle of N_SMPLX envs (a ragged last CTA), one row per env."""
    if robot == ROBOT:
        nenv, extra = N_DYN[backend.name]
        env = _production(backend, monkeypatch, cfg, nenv, 8, ragged=False)
        assert extra % (8 * EPW) != 0
        return env, nenv + extra
    n = N_SMPLX[backend.name]
    return _production(backend, monkeypatch, cfg, n, 4), n


def _rows_of(d, rows):
    return {k: x[rows] for k, x in d.items()}


def _shapes(tmp_path, mode):
    """The three SMPL body shapes of test_cta_shapes' per-env test: (cfg, oracle model) per shape for control mode `mode`, and the
    stable-PD oracle models the start states come from."""
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a"), _shape_variant(tmp_path / "b", leg=0.85, arm=1.1, trunk=0.93, girth=0.9, density=0.9)]
    made = [make_models(control_mode=mode, **({"robot.xml_path": p} if p else {})) for p in paths]
    pd = [make_models(control_mode="uhc_pd", **({"robot.xml_path": p} if p else {}))[1] for p in paths]
    return made, pd


def _shape_rows(backend, made, pd):
    """N_SHAPES rows, the shapes interleaved in ragged groups (every shape's last 8-warp CTA has empty slots), 12 rollout states per
    shape: (n, env_model, pool index, q, v, w, (shape, state) index of each row, first row of each (shape, state))."""
    n = N_SHAPES[backend.name]
    env_model = np.array([(i * 7 + i // 5) % 3 for i in range(n)], dtype=np.int32)
    assert (np.bincount(env_model) % (8 * EPW) != 0).all()
    pools = [rollout_states(pd[k], 12, seed=30 + k, every=9) for k in range(3)]
    pidx = np.zeros(n, dtype=np.int64)
    seen = [0, 0, 0]
    for i, k in enumerate(env_model):
        pidx[i] = seen[k] % 12
        seen[k] += 1
    q, v, w = (np.float32([pools[k][j][pidx[i]] for i, k in enumerate(env_model)]) for j in range(3))
    key = env_model * 12 + pidx
    first = [int(np.flatnonzero(key == kk)[0]) for kk in np.unique(key)]
    return n, env_model, pidx, q, v, w, np.unique(key, return_inverse=True)[1], first


# ================================================================== 1. centroidal (k_cent5)
def _cent(e, t, q, v, jb):
    return _np(e.centroidal(t(q), t(v), jac_com_bodies=jb))


@pytest.mark.parametrize("robot", ROBOTS)
def test_centroidal_at_production_shape(backend, monkeypatch, robot):
    """The _pool states tiled over the rows at the production CTA shape: every state but the overflowing one against ref_subtree /
    ref_cmm (test_centroidal's TOL_COM / TOL), every state the forward pass does not flag against Newton-Euler with forward(contact_wrench
    =True)'s contact wrenches (TOL_NE: the lying state's overflowing contacts and the past-limit states' limit forces enter there);
    bit-identical with 1-warp CTAs and across rows of the same pool state."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    env, n = _prod(backend, monkeypatch, robot, cfg)
    q, v, _, kinds, ctrl, idx = _tiled(robot, n)
    P = len(q)
    t = backend.t
    jb = list(range(m.nbody))

    def run(e, s):
        return _cent(e, t, q[idx[s]], v[idx[s]], jb)

    got = run(env, slice(0, n))
    _bit_equal(_bits(got), _bits(_one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), run)), f"{robot}: vs 1-warp CTAs")
    _dups_equal(_bits(got), idx, f"{robot}: same pool state")
    keep = [k for k in range(P) if kinds[k] != "bad"]
    worst = cent_errors(m, q[keep], v[keep], {**_rows_of(got, keep), "_jb": np.array(jb)}, om)
    grav = np.broadcast_to(np.asarray(m.gravity, dtype=np.float64), (P, 3))
    masses = np.broadcast_to(np.asarray(m.body_mass, dtype=np.float64), (P, m.nbody))
    ne, checked = _newton_euler(env, backend, m, q, v, ctrl, grav, masses)
    print(f"{robot}: {len(keep)} pool states against the references", {k: f"{x:.1e}" for k, x in worst.items()},
          f"Newton-Euler {ne:.1e} on {checked}")
    cent_within(worst, robot)
    assert checked >= P - 1, checked      # only the overflowing state is flagged
    assert ne <= TOL_NE, ne


# (robot, self-collision, parameter records): the eight k_cent5 instances
CENT_INSTANCES = [(r, s, p) for r in ROBOTS for s in (False, True) for p in (False, True)]


@pytest.mark.parametrize("robot,selfcol,records", CENT_INSTANCES)
def test_centroidal_every_instance(backend, monkeypatch, robot, selfcol, records):
    """Each k_cent5 instance at its class's production CTA size (self-collision SMPL at N_SELF, SMPL-X at N_SMPLX), one row per env,
    draw() records per pool state where asked: each pool state against the references of its env's variant model; bit-identical with
    1-warp CTAs of a plain handle with the same records on the same rows (for self-collision handles: the overflow entries k_cent5 sums
    into lie elsewhere in that class's scratch) and across rows of the same pool state and record."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    cfg_h = make_models(env="getup", robot=robot, control_mode="torque", self_collision=True)[0] if selfcol else cfg
    m = om.model
    if robot == ROBOT:
        n, wpb = (N_SELF if selfcol else N_SMPL)[backend.name], 8
    else:
        n, wpb = N_SMPLX[backend.name], 4
    q, v, _, kinds, _, idx = _tiled(robot, n)
    P = len(q)
    prm = draw(m, P, 91) if records else None
    jb = [0, 3, m.nbody - 1]
    t = backend.t

    def run(e, s):
        if prm is not None:
            e.set_env_params(**{k: t(x[idx[s]]) for k, x in prm.items()})
        return _cent(e, t, q[idx[s]], v[idx[s]], jb)

    env = _production(backend, monkeypatch, cfg_h, n, wpb)
    got = run(env, slice(0, n))
    what = f"{robot} self-collision={selfcol} records={records}"
    _bit_equal(_bits(got), _bits(_one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run)),
               what + ": vs a plain handle's 1-warp CTAs")
    _dups_equal(_bits(got), idx, what + ": same pool state")
    worst = None
    keep = [k for k in range(P) if kinds[k] != "bad"]
    for k in keep:
        row = {**_rows_of(got, slice(k, k + 1)), "_jb": np.array(jb)}
        mk, ok = (variant(m, prm, k), oracle_for(cfg, m, prm, k)) if records else (m, om)
        w = cent_errors(mk, q[k:k + 1], v[k:k + 1], row, ok)
        worst = w if worst is None else {x: max(worst[x], w[x]) for x in w}
    print(f"{what}: {len(keep)} pool states against the references", {k: f"{x:.1e}" for k, x in worst.items()})
    cent_within(worst, what)


def test_centroidal_per_env_shapes(backend, monkeypatch, tmp_path):
    """Three body shapes interleaved in ragged groups at the 8-warp production shape: each (shape, state) against its own shape's
    references, bit-identical with 1-warp CTAs and across rows of the same shape and state."""
    made, pd = _shapes(tmp_path, "torque")
    n, env_model, pidx, q, v, _, key, first = _shape_rows(backend, made, pd)
    models = [model_from_cfg(c) for c, _ in made]
    cfg0 = made[0][0]
    jb = [0, 5, 23]
    t = backend.t

    def run(e, s):
        return _cent(e, t, q[s], v[s], jb)

    env = _production(backend, monkeypatch, cfg0, n, 8, models=models, env_model=env_model)
    got = run(env, slice(0, n))
    ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg0, s.stop - s.start, models=models, env_model=env_model[s]), run,
                           chunk=CHUNK - 12)
    _bit_equal(_bits(got), _bits(ref), "per-env shapes: 8-warp vs 1-warp CTAs")
    _dups_equal(_bits(got), key, "same shape and state")
    worst = None
    for i in first:
        om = made[env_model[i]][1]
        w = cent_errors(om.model, q[i:i + 1], v[i:i + 1], {**_rows_of(got, slice(i, i + 1)), "_jb": np.array(jb)}, om)
        worst = w if worst is None else {x: max(worst[x], w[x]) for x in w}
    print(f"per-env shapes: {len(first)} (shape, state) rows against the references", {k: f"{x:.1e}" for k, x in worst.items()})
    cent_within(worst, "per-env shapes")


def _good_bad_rows(q, v, kinds, n, bad_of):
    """n rows: the pool's good states tiled, every seventh row (from row 3) and the last but one (in the second launch of the SMPL
    production handle) one of the bad rows bad_of(j, q, v) in turn.  Returns (Q, V, indices of the good rows, indices of the bad rows)."""
    good = [k for k in range(len(q)) if kinds[k] != "bad"]
    Q, V, g, b = [], [], [], []
    for i in range(n):
        if i % 7 == 3 or i == n - 2:
            qq, vv = bad_of(len(b), q, v)
            b.append(i)
        else:
            k = good[len(g) % len(good)]
            qq, vv = q[k], v[k]
            g.append(i)
        Q.append(qq); V.append(vv)
    return np.float32(Q), np.float32(V), np.array(g), np.array(b)


def test_centroidal_bad_rows_stay_local(backend, monkeypatch):
    """Rows with a NaN qvel, an inf qpos and a qpos entry of 2e10 between good rows of every CTA and of both launches of the 8-warp
    production handle: every good row bit-identical with a call without the bad rows."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env, n = _prod(backend, monkeypatch, ROBOT, cfg)
    q, v, _, kinds = _pool(ROBOT)

    def bad_of(j, q, v):
        qq, vv = q[1].copy(), v[1].copy()
        if j % 3 == 0:
            vv[7] = np.nan
        elif j % 3 == 1:
            qq[0] = np.inf
        else:
            qq[9] = 2e10
        return qq, vv

    Q, V, g, b = _good_bad_rows(q, v, kinds, n, bad_of)
    assert b.max() >= env.num_envs and len(b) >= 3
    t = backend.t
    jb = [0, 4, m.nbody - 1]
    got = _cent(env, t, Q, V, jb)
    ref = _cent(env, t, Q[g], V[g], jb)
    _bit_equal(_bits(_rows_of(got, g)), _bits(ref), "good rows next to bad rows")
    assert not np.isfinite(got["subtree_linvel"][b[0]]).all() and not np.isfinite(got["subtree_com"][b[1]]).all()
    print(f"{len(g)} good rows bit-identical next to {len(b)} bad rows")


def test_centroidal_root_quaternion_sign_and_scale(backend, monkeypatch):
    """The root quaternion times -1 and times 1.7 on the 8-warp production handle: every output against the references at the
    normalised state, to test_centroidal's TOL_COM / TOL."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env, n = _prod(backend, monkeypatch, ROBOT, cfg)
    q, v, _, kinds = _pool(ROBOT)
    keep = [k for k in range(len(q)) if kinds[k] != "bad"]
    q, v = q[keep].copy(), v[keep]
    q[:, 3:7] /= np.linalg.norm(q[:, 3:7], axis=1, keepdims=True)
    idx = np.arange(n) % len(q)
    jb = list(range(m.nbody))
    t = backend.t
    for s in (-1.0, 1.7):
        qs = q.copy()
        qs[:, 3:7] *= s
        got = _cent(env, t, qs[idx], v[idx], jb)
        _dups_equal(_bits(got), idx, f"root quaternion x {s}: same state")
        worst = cent_errors(m, q, v, {**_rows_of(got, slice(0, len(q))), "_jb": np.array(jb)}, om)
        print(f"root quaternion x {s}: {len(q)} states against the normalised references", {k: f"{x:.1e}" for k, x in worst.items()})
        cent_within(worst, f"root quaternion x {s}")


# ================================================================== 2. rne_post (k_rnep5)
def _body_sites(m):
    """rne_post's imu_sites="bodies", written out for ref_row."""
    return [(b, np.zeros(3, np.float32), np.float32([1, 0, 0, 0])) for b in range(m.nbody)]


def _rnep_check(om_of, q, v, a, got, xf, sites, rows, kinds):
    """rows of got against ref_row of om_of(row) by test_rne_post's _errors (its skip rule); returns (worst, kinds of the rows compared)."""
    worst, seen = None, []
    for k in rows:
        worst, c = rnep_errors(om_of(k), q[k:k + 1], v[k:k + 1], a[k:k + 1], _rows_of(got, slice(k, k + 1)), sites,
                               None if xf is None else _f64(xf[k:k + 1]), worst)
        if c:
            seen.append(kinds[k])
    return worst, seen


@pytest.mark.parametrize("robot", ROBOTS)
def test_rne_post_at_production_shape(backend, monkeypatch, robot):
    """The _pool states with random qacc and nonzero xfrc_applied on every row at the production CTA shape, 64 random sites on SMPL (the
    site limit) and "bodies" (52 sites) on SMPL-X: bit-identical with 1-warp CTAs (whose launches of 8 rows move xfrc_applied at every
    launch) and across rows of the same pool state; each pool state but the overflowing one against ref_row under test_rne_post's skip
    rule, the lying state (contact entries past NCS) among them."""
    cfg, om = make_models(robot=robot, control_mode="torque")
    m = om.model
    env, n = _prod(backend, monkeypatch, robot, cfg)
    q, v, _, kinds, _, idx = _tiled(robot, n)
    P = len(q)
    rng = np.random.default_rng(101)
    a = np.float32(rng.normal(size=(P, m.nv)) * 5.0)
    xf = np.float32(rng.normal(size=(P, m.nbody, 6)) * 20.0)
    arg = random_sites(m, 64, seed=102) if robot == ROBOT else "bodies"
    sites = arg if robot == ROBOT else _body_sites(m)
    assert len(sites) == (64 if robot == ROBOT else 52)
    t = backend.t

    def run(e, s):
        r = idx[s]
        return _np(e.rne_post(t(q[r]), t(v[r]), t(a[r]), imu_sites=arg, xfrc_applied=t(xf[r])))

    got = run(env, slice(0, n))
    _bit_equal(_bits(got), _bits(_one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), run)), f"{robot}: vs 1-warp CTAs")
    _dups_equal(_bits(got), idx, f"{robot}: same pool state")
    assert _inv_forward(om, q[kinds.index("lying")], v[kinds.index("lying")]).ncon > NCS[robot]
    worst, seen = _rnep_check(lambda k: om, q, v, a, got, xf, sites, [k for k in range(P) if kinds[k] != "bad"], kinds)
    print(f"{robot}: {len(seen)} pool states against ref_row", {k: f"{x:.1e}" for k, x in worst.items()})
    assert "lying" in seen and "limit" in seen and len(seen) >= P - 6, seen
    rnep_within(worst, robot)


def _ne_per_body(m, jw, acc, ex, cw):
    """test_rne_post.test_identities' per-body Newton-Euler: F_b - sum_children F_c + contact_b = m_b (a_com - g) and the matching torque
    about xipos, with the kernel's joint wrenches jw, accelerations acc and contact wrenches cw and the oracle's poses and velocities.
    Worst error relative to max(m |g|, max |jw|)."""
    xpos, xquat = ex["xpos"], ex["xquat"]
    g = np.asarray(m.gravity, dtype=np.float64)
    sc = max(float(np.sum(m.body_mass)) * float(np.linalg.norm(g)), float(np.abs(jw).max()))
    worst = 0.0
    for b in range(m.nbody):
        R = _qmat(xquat[b])
        r = R @ np.asarray(m.body_ipos[b], dtype=np.float64)
        xx, yy, zz, xy, xz, yz = np.asarray(m.body_inertia[b], dtype=np.float64)
        Ic = R @ np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]]) @ R.T
        w, wd = ex["vel"][b, 3:], acc[b, 3:]
        acom = acc[b, :3] + np.cross(wd, r) + np.cross(w, np.cross(w, r))
        F, T = jw[b, :3].copy(), jw[b, 3:] - np.cross(r, jw[b, :3])
        for c in range(b + 1, m.nbody):
            if int(m.body_parent[c]) == b:
                F -= jw[c, :3]
                T -= jw[c, 3:] + np.cross(xpos[c] - xpos[b] - r, jw[c, :3])
        F += cw[b, :3]; T += cw[b, 3:]
        e = max(np.abs(F - float(m.body_mass[b]) * (acom - g)).max(), np.abs(T - (Ic @ wd + np.cross(w, Ic @ w))).max())
        worst = max(worst, e / sc)
    return worst


def test_rne_post_rows_past_the_oracle(backend, monkeypatch):
    """Rows ref_row cannot judge: three airborne states past the joint-limit row cap (_past_cap: the kernel drops the rows past it) and
    the lying state, tiled over the 8-warp production handle's two launches.  Bit-identical with 1-warp CTAs; each held to test_identities'
    per-body Newton-Euler against the kernel's own inverse(contact_wrench=True) (limit forces are internal to joint_wrench), to TOL_ID;
    the lying state also to the root and hinge projections of _check_identities."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env, n = _prod(backend, monkeypatch, ROBOT, cfg)
    qp, vp, _, kinds = _pool(ROBOT)
    li = kinds.index("lying")
    caps = [_past_cap(m, s) for s in (5, 6, 7)]
    q = np.float32([qp[li]] + [c[0] for c in caps])
    v = np.float32([vp[li]] + [c[1] for c in caps])
    assert _inv_forward(om, q[0], v[0]).ncon > NCS[ROBOT]
    assert all(_over_cap(_inv_forward(om, q[j], v[j])) for j in (1, 2, 3))
    a = np.float32(np.random.default_rng(111).normal(size=v.shape) * 5.0)
    idx = np.arange(n) % len(q)
    t = backend.t

    def run(e, s):
        r = idx[s]
        return _np(e.rne_post(t(q[r]), t(v[r]), t(a[r])))

    got = run(env, slice(0, n))
    _bit_equal(_bits(got), _bits(_one_warp_chunks(backend, n, lambda s: backend.batch(cfg, 8), run)), "vs 1-warp CTAs")
    _dups_equal(_bits(got), idx, "same state")
    qfrc, cw = (x.cpu().numpy().astype(np.float64) for x in env.inverse(t(q), t(v), t(a), contact_wrench=True))
    arm = np.asarray(m.dof_armature, dtype=np.float64)
    ne, proj = 0.0, None
    for j in range(len(q)):
        _, ex = ref_row(om, q[j], v[j], a[j])
        jw = got["joint_wrench"][j].astype(np.float64)
        ne = max(ne, _ne_per_body(m, jw, got["body_acc"][j].astype(np.float64), ex, cw[j]))
        if j == 0 and not ex["skip"]:
            proj = _check_identities(m, jw, ex, qfrc[j], _f64(a[j]), arm, TOL_ID, "lying")
    print(f"{len(q)} states (lying + 3 past the cap): Newton-Euler {ne:.1e}, lying projections {proj}")
    assert ne <= TOL_ID, ne


@pytest.mark.parametrize("case", ["records-smpl", "records-smplx", "shapes"])
def test_rne_post_records_and_shapes(backend, monkeypatch, tmp_path, case):
    """k_rnep5<WithPrm> at the production CTA size, one row per env: draw() records per pool state on 8-warp SMPL and 4-warp SMPL-X, each
    pool state against ref_row of its env's variant oracle; three SMPL body shapes in ragged groups, each (shape, state) against its own
    shape's oracle.  Random sites and xfrc_applied; bit-identical with 1-warp CTAs and across rows of the same state."""
    t = backend.t
    if case == "shapes":
        made, pd = _shapes(tmp_path, "torque")
        n, env_model, pidx, q, v, _, key, rows = _shape_rows(backend, made, pd)
        models = [model_from_cfg(c) for c, _ in made]
        m = models[0]
        cfg0 = made[0][0]
        # ref_row's central difference in time is off by about (H_FD |qvel|)^2 / 6 of body_acc: the second shape's rollout states reach
        # 300 rad/s (4e-4 there), so every row is scaled to |qvel| <= 30 (3e-6 at most)
        v = np.float32(v * np.minimum(1.0, 30.0 / np.abs(v).max(1, keepdims=True)))
        a = np.float32(np.random.default_rng(121).normal(size=(12, m.nv)) * 5.0)[pidx]
        xf = np.float32(np.random.default_rng(122).normal(size=(12, m.nbody, 6)) * 20.0)[pidx]
        sites = random_sites(m, 9, seed=123)

        def run(e, s):
            return _np(e.rne_post(t(q[s]), t(v[s]), t(a[s]), imu_sites=sites, xfrc_applied=t(xf[s])))
        env = _production(backend, monkeypatch, cfg0, n, 8, models=models, env_model=env_model)
        got = run(env, slice(0, n))
        ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg0, s.stop - s.start, models=models, env_model=env_model[s]), run,
                               chunk=CHUNK - 12)
        kinds = ["rollout"] * n
        om_of = lambda i: made[env_model[i]][1]  # noqa: E731
    else:
        robot = ROBOT if case == "records-smpl" else "smplx_humanoid"
        cfg, om = make_models(robot=robot, control_mode="torque")
        m = om.model
        n, wpb = (N_SMPL[backend.name], 8) if robot == ROBOT else (N_SMPLX[backend.name], 4)
        qp, vp, _, kp, _, key = _tiled(robot, n)
        P = len(qp)
        prm = draw(m, P, 124)
        rng = np.random.default_rng(125)
        ap, xfp = np.float32(rng.normal(size=(P, m.nv)) * 5.0), np.float32(rng.normal(size=(P, m.nbody, 6)) * 20.0)
        q, v, a, xf = qp[key], vp[key], ap[key], xfp[key]
        sites = random_sites(m, 9, seed=126)

        def run(e, s):
            e.set_env_params(**{k: t(x[key[s]]) for k, x in prm.items()})
            return _np(e.rne_post(t(q[s]), t(v[s]), t(a[s]), imu_sites=sites, xfrc_applied=t(xf[s])))
        env = _production(backend, monkeypatch, cfg, n, wpb)
        got = run(env, slice(0, n))
        ref = _one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run)
        kinds = [kp[k] for k in key]
        rows = [k for k in range(P) if kp[k] != "bad"]
        oms = {}
        om_of = lambda i: oms.setdefault(i, oracle_for(cfg, m, prm, i))  # noqa: E731
    _bit_equal(_bits(got), _bits(ref), f"{case}: vs 1-warp CTAs")
    _dups_equal(_bits(got), key, f"{case}: same state")
    worst, seen = _rnep_check(om_of, q, v, a, got, xf, sites, rows, kinds)
    print(f"{case}: {len(seen)}/{len(rows)} states against ref_row", {k: f"{x:.1e}" for k, x in worst.items()})
    assert len(seen) >= len(rows) - 6, (len(seen), len(rows))
    rnep_within(worst, case)


def test_rne_post_bad_rows_stay_local(backend, monkeypatch):
    """The rows of test_rollout_invfd_paths' test_inverse_fd_bad_rows on the 8-warp production handle: good rows (the lying state and
    rollout states at the oracle's qacc) interleaved with the overflowing state (qvel 8e9), an inf qvel, a NaN qacc, a qpos entry of 2e10
    and a row past the joint-limit row cap, with sites and xfrc_applied: every good row bit-identical with a call without the bad rows."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = _production(backend, monkeypatch, cfg, N_DYN[backend.name][0], 8, ragged=False)
    qp, vp, _, kinds = _pool(ROBOT)
    gi = [kinds.index("lying"), 1, 2]
    good_q, good_v = np.float32(qp[gi]), np.float32(vp[gi])
    good_a = np.float32([_inv_forward(om, good_q[i], good_v[i]).qacc.copy() for i in range(3)])
    z = np.zeros(m.nv)
    bq, bv, ba = [qp[kinds.index("bad")]], [vp[kinds.index("bad")]], [z]
    x = good_v[1].copy(); x[0] = np.inf
    bq.append(good_q[1]); bv.append(x); ba.append(good_a[1])
    x = good_a[2].copy(); x[10] = np.nan
    bq.append(good_q[2]); bv.append(good_v[2]); ba.append(x)
    x = good_q[1].copy(); x[9] = 2e10
    bq.append(x); bv.append(good_v[1]); ba.append(good_a[1])
    qc, vc = _past_cap(m, 5)
    bq.append(qc); bv.append(vc); ba.append(z)
    order = [("g", 0), ("b", 0), ("b", 1), ("g", 1), ("b", 2), ("b", 3), ("g", 2), ("b", 4)]
    Q = np.float32([good_q[j] if s == "g" else bq[j] for s, j in order])
    V = np.float32([good_v[j] if s == "g" else bv[j] for s, j in order])
    A = np.float32([good_a[j] if s == "g" else ba[j] for s, j in order])
    good = np.array([i for i, (s, _) in enumerate(order) if s == "g"])
    xf = np.float32(np.random.default_rng(131).normal(size=(len(order), m.nbody, 6)) * 20.0)
    sites = random_sites(m, 9, seed=132)
    t = backend.t
    got = _np(env.rne_post(t(Q), t(V), t(A), imu_sites=sites, xfrc_applied=t(xf)))
    ref = _np(env.rne_post(t(Q[good]), t(V[good]), t(A[good]), imu_sites=sites, xfrc_applied=t(xf[good])))
    _bit_equal(_bits(_rows_of(got, good)), _bits(ref), "rne_post: good rows next to bad rows")
    assert all(np.isfinite(x).all() for x in ref.values())
    print(f"{len(good)} good rows bit-identical next to {len(order) - len(good)} bad rows")


# ================================================================== 3. closed-loop rollouts (k_rollfb5)
def _law_worst(got, q0, v0, U, K, qr, vr, kidx, clip):
    """test_law_in_fp64's check on every row: each control[i, t] recomputed in fp64 from the recorded x_t, with gains / references
    K[kidx[i]], qr[kidx[i]], vr[kidx[i]] (fp32 inputs); worst |u - ref| / (sum |K dx| + |ubar|)."""
    xq, xv = (x.numpy().astype(np.float64) for x in _pre_states(torch.as_tensor(q0), torch.as_tensor(v0),
                                                                 {k: torch.as_tensor(got[k]) for k in ("qpos", "qvel")}))
    ug = got["control"].astype(np.float64)
    qr, vr, K = qr.astype(np.float64), vr.astype(np.float64), K.astype(np.float64)
    worst = 0.0
    for i in range(len(ug)):
        k = kidx[i]
        for s in range(U.shape[1]):
            dx = np.concatenate([_np_diff(qr[k, s], xq[i, s]), xv[i, s] - vr[k, s]])
            Kdx = K[k, s] * dx[None]
            ref = U[i, s].astype(np.float64) + Kdx.sum(1)
            scale = np.abs(Kdx).sum(1) + np.abs(U[i, s])
            if clip:
                ref = np.clip(ref, -1, 1)
            worst = max(worst, float(np.max(np.abs(ug[i, s] - ref) / scale)))
    return worst


# One oracle mj_step per recorded step of a feedback rollout.  The step is k_roll5's (a feedback run replays bit for bit through the
# open-loop path), but its start states and controls are the feedback's: there test_rollout_at_production_shape's 1e-4 and
# test_rollout_with_parameter_records' 2e-4 (qvel, norm-relative) held no margin.  Worst qvel seen, emulator / H100: production shapes
# 9.5e-5 / 1.3e-4 (FB_STEP_TOL, _check_row's qvel bound); records and shapes 1.7e-4 / 3.7e-4 (2 FB_NORM_TOL, _check_norms' qvel bound).
FB_STEP_TOL = 3e-3
FB_NORM_TOL = 4e-3


def _fb_problem(m, P, T, mode, seed, ctrl_gain=1.0):
    """Per pool state: controls (_controls), gains N(0, 1) x 0.05 (action) or x ctrl_gain (ctrl), and the generator for the references."""
    rng = np.random.default_rng(seed)
    K = np.float32(rng.normal(size=(P, T, m.nu, 2 * m.nv)) * (0.05 if mode == "action" else ctrl_gain))
    return _controls(m, P, T, mode, seed=seed + 1), K, rng


@pytest.mark.parametrize("robot", ROBOTS)
@pytest.mark.parametrize("shared", [False, True])
def test_feedback_law_at_production_shape(backend, monkeypatch, robot, shared):
    """The _pool start states tiled over the rows at the production CTA shape (SMPL: two launches), references one per row
    (ref_rows == n) or one schedule for every row (ref_rows == 1: the second launch reads the same rows), action mode under stable PD
    and ctrl mode with nsub 1 and 2: every control[i, t] against the law in fp64 (test_law_in_fp64's bound, 1e-5); bit-identical with
    1-warp CTAs and across rows of the same pool state; in ctrl mode with nsub = 1 every recorded step of each pool state against one
    oracle mj_step from the kernel's own state (test_rollout_at_production_shape's bounds), the overflowing state resetting at step 0
    and following the law from the reset state on."""
    cfg, om = make_models(robot=robot, control_mode="uhc_pd")
    m = om.model
    env, n = _prod(backend, monkeypatch, robot, cfg)
    q, v, w, kinds, _, idx = _tiled(robot, n)
    P, T = len(q), T_PROD[backend.name]
    bad = [k for k in range(P) if kinds[k] == "bad"]
    t = backend.t
    dev = torch.device(backend.device)
    for mode, nsub in (("action", None), ("ctrl", 1), ("ctrl", 2)):
        # ctrl gains x 0.2: with one shared schedule dx is the distance to pool state 0, and K dx then adds up to ~20 N m to the
        # U(-80, 80) torques, the range test_rollout_at_production_shape's step bounds were measured on
        U, K, rng = _fb_problem(m, P, T, mode, seed=140 + (nsub or 0) + 10 * shared, ctrl_gain=0.2)
        qr = np.float32(q[:, None] + rng.normal(size=(P, T, m.nq)) * 0.01)
        # the overflowing state's references hold qvel ~ 0, the reset state's: after its reset at step 0 the law runs on ordinary dx
        vr = np.float32(np.where(np.isin(np.arange(P), bad)[:, None], 0.0, v)[:, None] + rng.normal(size=(P, T, m.nv)) * 0.1)
        Kt, qrt, vrt = t(K), t(qr), t(vr)
        kidx = np.zeros(n, dtype=np.int64) if shared else idx

        def run(e, s):
            r = idx[s]
            if shared:
                fb = dict(gains=Kt[:1], qpos_ref=qrt[:1], qvel_ref=vrt[:1])
            else:
                ri = torch.as_tensor(r, device=dev)
                fb = dict(gains=Kt[ri], qpos_ref=qrt[ri], qvel_ref=vrt[ri])
            return _roll(e, t, q[r], v[r], w[r], U[r], mode, nsub, mode == "action", **fb)

        got = run(env, slice(0, n))
        what = f"{robot} {mode} nsub={nsub} ref_rows={'1' if shared else 'n'}"
        _bit_equal(_bits(got), _bits(_one_warp_chunks(backend, n, lambda s: backend.batch(cfg, s.stop - s.start), run)),
                   what + ": vs 1-warp CTAs")
        _dups_equal(_bits(got), idx, what + ": same pool state")
        for k in bad:   # mj_checkAcc at step 0: bit 4 and the reset state, from which the law runs on (checked below)
            assert got["status"][k, 0] & 4, (what, got["status"][k])
        law = _law_worst(got, q[idx], v[idx], U[idx], K, qr, vr, kidx, mode == "action" and cfg.env.clip_actions)
        msg = f"{what}: law on {n} x {T} rows, worst {law:.1e}"
        assert law < 1e-5, (what, law)
        if mode == "ctrl" and nsub == 1:
            ncmp, worst = _check_steps(backend, env, got, q[idx], v[idx], w[idx], got["control"], range(P), lambda i: om, kinds, FB_STEP_TOL,
                                       m)
            msg += f"; {ncmp}/{P * T} pool-state steps against the oracle, worst qvel {worst:.2e}"
            assert ncmp >= P * T - 3 * T, ncmp
        print(msg)


@pytest.mark.parametrize("case", ["records-smpl", "records-smplx", "shapes"])
def test_feedback_records_and_shapes(backend, monkeypatch, tmp_path, case):
    """k_rollfb5<WithPrm> at the production CTA size, one row per env, ctrl mode with nsub = 1: draw() records per pool state on 8-warp
    SMPL and 4-warp SMPL-X (the SMPL-X instance no feature test runs), and three SMPL body shapes in ragged groups.  Replaying the applied
    controls open loop on the same handle gives the same bits; every recorded step of each state against one mj_step of its env's variant
    or shape oracle (_check_norms, test_rollout_with_parameter_records' bounds); bit-identical across rows of the same state."""
    t = backend.t
    T = T_PROD[backend.name]
    if case == "shapes":
        made, pd = _shapes(tmp_path, "uhc_pd")
        n, env_model, pidx, q, v, w, key, first = _shape_rows(backend, made, pd)
        models = [model_from_cfg(c) for c, _ in made]
        m = models[0]
        U, K, rng = _fb_problem(m, 12, T, "ctrl", seed=151)
        U, K = U[pidx], K[pidx]
        env = _production(backend, monkeypatch, made[0][0], n, 8, models=models, env_model=env_model)
        kinds = ["rollout"] * n
        oracle_of = lambda i: made[env_model[i]][1]  # noqa: E731
    else:
        robot = ROBOT if case == "records-smpl" else "smplx_humanoid"
        cfg, _ = make_models(robot=robot, control_mode="uhc_pd")
        m = model_from_cfg(cfg)
        n, wpb = (N_SMPL[backend.name], 8) if robot == ROBOT else (N_SMPLX[backend.name], 4)
        qp, vp, wp, kp, _, key = _tiled(robot, n, seed=8)
        P = len(qp)
        prm = draw(m, P, 152)
        U, K, rng = _fb_problem(m, P, T, "ctrl", seed=153)
        q, v, w, U, K = qp[key], vp[key], wp[key], U[key], K[key]
        env = _production(backend, monkeypatch, cfg, n, wpb)
        env.set_env_params(**{k: t(x[key]) for k, x in prm.items()})
        kinds = [kp[k] for k in key]
        first = [k for k in range(P) if kp[k] != "bad"]
        oms = {}
        oracle_of = lambda i: oms.setdefault(i, oracle_for(cfg, m, prm, i))  # noqa: E731
    qr = np.float32(q[:, None] + rng.normal(size=(n, T, m.nq)) * 0.01)
    vr = np.float32(v[:, None] + rng.normal(size=(n, T, m.nv)) * 0.1)
    got = _roll(env, t, q, v, w, U, "ctrl", 1, gains=t(K), qpos_ref=t(qr), qvel_ref=t(vr))
    rep = _roll(env, t, q, v, w, got["control"], "ctrl", 1)
    _bit_equal(_bits(got), _bits(rep), f"{case}: feedback run vs replay of its controls")
    ncmp, worst = _check_steps(backend, env, got, q, v, w, got["control"], first, oracle_of, kinds, FB_NORM_TOL, m, check=_check_norms)
    print(f"{case}: {ncmp}/{len(first) * T} steps against the variant / shape oracles, worst qvel {worst:.2e}")
    assert ncmp >= len(first) * T - 2 * T, ncmp


def test_feedback_without_control_output(backend, monkeypatch):
    """smplsim_rollout_feedback with control_applied == NULL (u goes to the handle's own scratch row) over the two launches of the
    8-warp production handle, ref_rows 1 and n, action and ctrl mode: qpos, qvel, status and the poses bit-identical with the call that
    passes control_applied."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    env, n = _prod(backend, monkeypatch, ROBOT, cfg)
    assert n > env.num_envs
    q, v, w, _, _, idx = _tiled(ROBOT, n)
    q, v, w = q[idx], v[idx], w[idx]
    T = T_PROD[backend.name]
    L, h, s = env._L(), env._h, env._stream()
    t = backend.t
    p = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None  # noqa: E731
    tq, tv, tw = t(q), t(v), t(w)
    dev = tq.device
    nb = m.nbody
    checked = 0
    for mode, nsub, name in ((ROLLOUT_ACTION, 0, "action"), (ROLLOUT_CTRL, 2, "ctrl")):
        for R in (1, n):
            U, K, rng = _fb_problem(m, R, T, name, seed=161 + R % 7)
            tu = t(_controls(m, n, T, name, seed=162))
            tK = t(K)
            tqr = t(q[:R, None] + rng.normal(size=(R, T, m.nq)) * 0.01)
            tvr = t(v[:R, None] + rng.normal(size=(R, T, m.nv)) * 0.1)

            def call(with_u):
                out = {"qpos": t(np.full((n, T, m.nq), np.nan)), "qvel": t(np.full((n, T, m.nv), np.nan)),
                       "status": torch.full((n, T), 0xAB, dtype=torch.uint8, device=dev),
                       "xpos": t(np.full((n, T, nb, 3), np.nan)), "xquat": t(np.full((n, T, nb, 4), np.nan))}
                uo = t(np.full((n, T, m.nu), np.nan)) if with_u else None
                assert L.smplsim_rollout_feedback(h, mode, nsub, p(tq), p(tv), p(tw), None, None, p(tu), n, T, p(out["qpos"]),
                                                  p(out["qvel"]), p(out["status"]), p(out["xpos"]), p(out["xquat"]), p(tK), p(tqr),
                                                  p(tvr), R, 1, p(uo), s) == 0
                return {k: x.cpu().numpy() for k, x in out.items()}

            a, b = call(True), call(False)
            assert np.isfinite(a["qpos"]).all() and (a["status"] != 0xAB).all()
            _bit_equal(_bits(b), _bits(a), f"{name} ref_rows={R}: control_applied NULL vs given")
            checked += 1
    print(f"{checked} calls on {n} rows: control_applied NULL bit-identical with the call that passes it")


# ================================================================== 4. the handle scratch the calls share
def test_calls_share_handle_scratch(backend, monkeypatch):
    """rollout, rne_post, rollout(gains=...), centroidal and rollout again, in that order, on one 8-warp production handle and stream,
    with more rows than num_envs (rne_post sums its joint wrenches in the rows where rollout keeps its step-boundary state): each result
    bit-identical with the same call on a fresh handle."""
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    env, n = _prod(backend, monkeypatch, ROBOT, cfg)
    nenv = env.num_envs
    assert n > nenv
    q, v, w, _, _, idx = _tiled(ROBOT, n)
    q, v, w = q[idx], v[idx], w[idx]
    T = T_PROD[backend.name]
    t = backend.t
    rng = np.random.default_rng(171)
    a = np.float32(rng.normal(size=(n, m.nv)) * 5.0)
    xf = np.float32(rng.normal(size=(n, m.nbody, 6)) * 20.0)
    sites = random_sites(m, 9, seed=172)
    ua = _controls(m, n, T, "action", seed=173)
    uc = _controls(m, n, T, "ctrl", seed=174)
    K = t(rng.normal(size=(n, T, m.nu, 2 * m.nv)))
    qr, vr = t(q[:, None] + rng.normal(size=(n, T, m.nq)) * 0.01), t(v[:, None] + rng.normal(size=(n, T, m.nv)) * 0.1)
    calls = [("rollout", lambda e: _roll(e, t, q, v, w, ua, "action", None, True)),
             ("rne_post", lambda e: _np(e.rne_post(t(q), t(v), t(a), imu_sites=sites, xfrc_applied=t(xf)))),
             ("rollout(gains=...)", lambda e: _roll(e, t, q, v, w, uc, "ctrl", 2, True, gains=K, qpos_ref=qr, qvel_ref=vr)),
             ("centroidal", lambda e: _cent(e, t, q, v, [0, 7, m.nbody - 1])),
             ("rollout again", lambda e: _roll(e, t, q, v, w, ua, "action", None, True))]
    for name, f in calls:
        got = f(env)
        fresh = f(_production(backend, monkeypatch, cfg, nenv, 8, ragged=False))
        _bit_equal(_bits(got), _bits(fresh), f"{name}: shared handle vs fresh handle")
    print(f"{len(calls)} calls on {n} rows of one handle bit-identical with fresh handles")
