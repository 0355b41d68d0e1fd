"""Ray casting and camera images (smplsim_ray / smplsim_render, HumanoidBatchB200.ray / render, the B1 render(), MotionLibB200.render_clip).

The geometric reference is test-side numpy in fp64, written from the closed-form definitions in include/smplsim.h: spheres, capsules
(cylinder + end hemispheres), boxes (slab method) and the one-sided floor plane, smallest non-negative root.  It takes body poses from the
oracle's forward kinematics and geom data from the ModelDesc; the kernel gets the same poses rounded to fp32.

Guard band: a ray whose nearest geom changes when every geom (and the floor) is grown or shrunk by GUARD = 1e-4 m passes within 1e-4 m
of a silhouette; a ray whose two nearest hits lie within 1e-4 m of each other is a near tie.  Both are left out of the exact comparisons,
and their share is held below GUARD_CAP.  For RGB the band also takes pixels whose shadow ray changes under the same test, whose floor
point lies within 1e-4 m of a checker edge, or whose box hit lies within 1e-4 m of a box edge.

Worst error outside the guard band: the distance along the ray in metres (|dx| |vec|), relative beyond 1 m, and for floor hits also
times |cos| of the ray's angle to the floor normal (the plane intersection's condition number: far, grazing floor rays).  Emulator:
rays 1.05e-6, images 1.24e-6; H100: rays 1.05e-6, images 1.16e-6.  TOL_DIST = 2e-5 keeps a margin of over 15x.  Guard-band share:
at most 0.26 % of the rays and 0.04 % of the pixels on both, against GUARD_CAP = 3 %.  RGB: within 1 LSB of the numpy shading."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc
from smplsim_b200 import _lib
from smplsim_b200 import camera as cam
from smplsim_b200.cfg import make_cfg
from util_states import airborne_states, make_models, rollout_states

GUARD = 1e-4
GUARD_CAP = 0.03
TOL_DIST = 2e-5
SPHERE, CAPSULE, BOX = 2, 3, 6
EDGE = 200.0 / 120.0


# ------------------------------------------------------------------ test-side fp64 reference
def _qmat(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class Scene:
    """World pose of every robot geom of one row (fp64)."""

    def __init__(self, m, xpos, xquat):
        self.m = m
        xpos, xquat = np.asarray(xpos, np.float64), np.asarray(xquat, np.float64)
        self.Rb = np.array([_qmat(q) for q in xquat])
        self.xb = xpos
        b = np.asarray(m.geom_body)
        self.c = np.array([xpos[b[g]] + self.Rb[b[g]] @ m.geom_pos[g] for g in range(m.ngeom)])
        self.R = np.array([self.Rb[b[g]] @ np.asarray(m.geom_mat[g]).reshape(3, 3) for g in range(m.ngeom)])
        self.s = np.asarray(m.geom_size, np.float64)
        self.type = np.asarray(m.geom_type)
        self.body = b
        self.p0 = np.asarray(m.plane_pos, np.float64)
        self.pn = np.asarray(m.plane_normal, np.float64) / np.linalg.norm(m.plane_normal)

    def com(self):
        m = np.asarray(self.m.body_mass, np.float64)
        c = self.xb + np.einsum("bij,bj->bi", self.Rb, np.asarray(self.m.body_ipos, np.float64))
        return (m[:, None] * c).sum(0) / m.sum()


def _quad(a, b, c):
    det = b * b - a * c
    ok = det >= 0
    sd = np.sqrt(np.where(ok, det, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(ok, (-b - sd) / a, np.nan), np.where(ok, (-b + sd) / a, np.nan)


def _take(best, x, cond):
    return np.fmin(best, np.where(cond & (x >= 0), x, np.nan))


def hit_geom(S, g, P, V, infl=0.0):
    """[R] smallest x >= 0 with P + x V on geom g grown by `infl` (nan: none)."""
    p, v = (P - S.c[g]) @ S.R[g], V @ S.R[g]
    best = np.full(len(P), np.nan)
    t = S.type[g]
    if t == SPHERE:
        r = S.s[g, 0] + infl
        for x in _quad((v * v).sum(1), (p * v).sum(1), (p * p).sum(1) - r * r):
            best = _take(best, x, True)
    elif t == CAPSULE:
        r, h = S.s[g, 0] + infl, S.s[g, 1]
        a = v[:, 0] ** 2 + v[:, 1] ** 2
        for x in _quad(a, p[:, 0] * v[:, 0] + p[:, 1] * v[:, 1], p[:, 0] ** 2 + p[:, 1] ** 2 - r * r):
            best = _take(best, x, (a > 0) & (np.abs(p[:, 2] + x * v[:, 2]) <= h))
        for sg in (1.0, -1.0):
            q = p - np.array([0, 0, sg * h])
            for x in _quad((v * v).sum(1), (q * v).sum(1), (q * q).sum(1) - r * r):
                best = _take(best, x, sg * (p[:, 2] + x * v[:, 2]) >= h)
    else:
        s = S.s[g] + infl
        with np.errstate(divide="ignore", invalid="ignore"):
            ta, tb = (-s - p) / v, (s - p) / v
        t0 = np.nanmax(np.minimum(ta, tb), axis=1)
        t1 = np.nanmin(np.maximum(ta, tb), axis=1)
        out = (v == 0) & (np.abs(p) > s)
        hit = (t1 >= t0) & (t1 >= 0) & ~out.any(1)
        best = np.where(hit, np.where(t0 >= 0, t0, t1), np.nan)
    return best


def hit_plane(S, P, V, infl=0.0):
    dn, h = V @ S.pn, (P - S.p0) @ S.pn - infl
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where((dn < 0) & (h >= 0), -h / dn, np.nan)


def cast(S, P, V, flg_static=True, exclude=-1, infl=0.0):
    """[R, ngeom + 1] hit distance per MuJoCo geom id (nan: none)."""
    X = np.full((len(P), S.m.ngeom + 1), np.nan)
    if flg_static:
        X[:, 0] = hit_plane(S, P, V, infl)
    for g in range(S.m.ngeom):
        if S.body[g] != exclude:
            X[:, g + 1] = hit_geom(S, g, P, V, infl)
    return X


def _nearest(X):
    allnan = np.all(np.isnan(X), axis=1)
    ids = np.where(allnan, -1, np.nanargmin(np.where(allnan[:, None], 0.0, X), axis=1))
    d = np.where(allnan, -1.0, np.nanmin(np.where(allnan[:, None], np.inf, X), axis=1))
    return ids, d


def ref_rays(S, P, V, flg_static=True, exclude=-1):
    """Reference (dist, geomid) and the guard-band mask (True: excluded)."""
    X = cast(S, P, V, flg_static, exclude)
    ids, d = _nearest(X)
    guard = np.zeros(len(P), bool)
    for e in (GUARD, -GUARD):
        guard |= _nearest(cast(S, P, V, flg_static, exclude, e))[0] != ids
    srt = np.sort(np.where(np.isnan(X), np.inf, X), axis=1)
    vn = np.linalg.norm(V, axis=1)
    with np.errstate(invalid="ignore"):
        guard |= np.isfinite(srt[:, 1]) & ((srt[:, 1] - srt[:, 0]) * vn < GUARD)
    return d, ids, guard


def _scale(dist_m, ids, cosf):
    """Error scale of a hit dist_m metres along the ray: 1 m below 1 m, relative beyond; floor hits also by 1 / cos of the angle
    between ray and floor normal (the intersection's condition number: grazing floor rays far out)."""
    return np.maximum(1.0, dist_m) / np.where(ids == 0, np.maximum(cosf, 1e-6), 1.0)


def cam_pose(S, c):
    """Camera position and world axes (columns) of a smplsim_b200.camera.Camera."""
    mat = np.asarray(c.mat, np.float64).reshape(3, 3)
    pos = np.asarray(c.pos, np.float64)
    if c.mode == cam.TRACKCOM:
        pos = S.com() + pos
    elif c.mode == cam.BODY:
        pos, mat = S.xb[c.body] + S.Rb[c.body] @ pos, S.Rb[c.body] @ mat
    return pos, mat


def pixel_rays(c, W, H, pos, mat):
    ty = np.tan(np.deg2rad(c.fovy) / 2)
    tx = ty * W / H
    cc, rr = np.meshgrid(np.arange(W), np.arange(H))
    u = (2 * (cc + 0.5) / W - 1) * tx
    v = (1 - 2 * (rr + 0.5) / H) * ty
    D = u.reshape(-1, 1) * mat[:, 0] + v.reshape(-1, 1) * mat[:, 1] - mat[:, 2]
    return np.broadcast_to(pos, D.shape).copy(), D


def _normal(S, g, X):
    q = (X - S.c[g]) @ S.R[g]
    t = S.type[g]
    if t == SPHERE:
        n = q
    elif t == CAPSULE:
        n = q - np.stack([0 * q[:, 0], 0 * q[:, 0], np.clip(q[:, 2], -S.s[g, 1], S.s[g, 1])], 1)
    else:
        d = np.abs(q) - S.s[g]
        k = np.argmax(d, axis=1)
        n = np.zeros_like(q)
        n[np.arange(len(q)), k] = np.sign(q[np.arange(len(q)), k])
    n = n @ S.R[g].T
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def ref_render(S, c, W, H, geom_rgb=None):
    """(depth, seg, rgb, guard, rgb_guard, |ray direction|, |cos| of the ray's angle to the floor normal) images [H, W] / [H, W, 3]."""
    pos, mat = cam_pose(S, c)
    P, D = pixel_rays(c, W, H, pos, mat)
    d, ids, guard = ref_rays(S, P, D, True, c.exclude_body)
    depth = np.where(ids >= 0, d, c.zfar)
    alb_tab = np.tile([0.8, 0.6, 0.4], (S.m.ngeom, 1)) if geom_rgb is None else np.asarray(geom_rgb, np.float64)
    col = np.zeros((len(P), 3))
    rguard = guard.copy()
    bg = ids < 0
    t = (D[:, 2] / np.linalg.norm(D, axis=1) + 1) / 2
    col[bg] = t[bg, None] * np.array([0.4, 0.5, 0.6])
    X = P + d[:, None] * D
    n = np.zeros_like(P)
    alb = np.zeros_like(P)
    fl = ids == 0
    n[fl] = S.pn
    ax = np.array([1.0, 0, 0]) - S.pn[0] * S.pn
    ax /= np.linalg.norm(ax)
    uv = np.stack([(X - S.p0) @ ax, (X - S.p0) @ np.cross(S.pn, ax)], 1) / EDGE
    k = np.floor(uv).sum(1).astype(np.int64)
    alb[fl] = np.where(k[fl] & 1, 0.8, 0.0)[:, None]
    rguard |= fl & (np.abs(uv - np.round(uv)).min(1) * EDGE < GUARD)
    for g in range(S.m.ngeom):
        sel = ids == g + 1
        if not sel.any():
            continue
        n[sel] = _normal(S, g, X[sel])
        alb[sel] = alb_tab[g]
        if S.type[g] == BOX:
            q = (X[sel] - S.c[g]) @ S.R[g]
            rguard[np.nonzero(sel)[0][(np.abs(q) > S.s[g] - GUARD).sum(1) >= 2]] = True
    hit = ids >= 0
    flip = (n * D).sum(1) > 0
    n[flip] *= -1
    lit = 0.1 + 0.4 * np.maximum(0.0, -(n @ -mat[:, 2]))
    up = np.array([0.0, 0.0, 1.0])
    sh_cast = hit & (n[:, 2] > 0)
    if sh_cast.any():
        Ps = X[sh_cast] + 1e-4 * n[sh_cast]
        Vs = np.broadcast_to(up, Ps.shape).copy()
        shs = []
        for e in (0.0, GUARD, -GUARD):
            Xs = np.full((len(Ps), S.m.ngeom), np.nan)
            for g in range(S.m.ngeom):
                Xs[:, g] = hit_geom(S, g, Ps, Vs, e)
            shs.append(~np.all(np.isnan(Xs), axis=1))
        s = np.ones(len(P))
        s[sh_cast] = np.where(shs[0], 0.0, 1.0)
        rguard[np.nonzero(sh_cast)[0][(shs[1] != shs[0]) | (shs[2] != shs[0])]] = True
        lit = lit + np.maximum(0.0, n[:, 2]) * s
    col[hit] = np.clip(alb[hit] * lit[hit, None], 0, 1)
    rgb = np.floor(255 * col + 0.5)
    return (depth.reshape(H, W), ids.reshape(H, W), rgb.reshape(H, W, 3), guard.reshape(H, W), rguard.reshape(H, W),
            np.linalg.norm(D, axis=1).reshape(H, W), (np.abs(D @ S.pn) / np.linalg.norm(D, axis=1)).reshape(H, W))


# ------------------------------------------------------------------ states
def _poses(om, q):
    """Oracle forward kinematics of each qpos row, rounded to fp32: xpos [n, nb, 3], xquat [n, nb, 4]."""
    xp, xq = [], []
    for qi in q:
        e = orc.OracleEnv(om)
        e.qpos[:] = qi
        e.qvel[:] = 0
        e.forward()
        xp.append(e.xpos.copy()); xq.append(e.xquat.copy())
    return np.float32(xp), np.float32(xq)


def _states(om, n, seed):
    """Airborne states followed by rollout states (standing, stumbling, fallen)."""
    na = max(1, n // 3)
    qa, _ = airborne_states(om.model, na, seed=seed)
    qc, _, _ = rollout_states(om, n - na, seed=seed + 1, every=17)
    return np.concatenate([qa, qc])


def _random_rays(rng, xpos, R):
    """Rays around the robot: origins in a box about the root, aimed at a random body (+ noise), lengths 0.5-2 (vec not unit)."""
    n = len(xpos)
    root = xpos[:, 0]
    P = root[:, None, :] + rng.uniform([-1.5, -1.5, -1.0], [1.5, 1.5, 1.5], (n, R, 3))
    P[..., 2] = np.maximum(P[..., 2], 0.02)
    tgt = xpos[np.arange(n)[:, None], rng.integers(0, xpos.shape[1], (n, R))] + rng.normal(size=(n, R, 3)) * 0.1
    V = tgt - P
    V *= (rng.uniform(0.5, 2.0, (n, R)) / np.linalg.norm(V, axis=2))[..., None]
    k = R // 8        # some rays in random directions (sky, floor, from inside geoms)
    V[:, :k] = rng.normal(size=(n, k, 3))
    P[:, k:2 * k] = tgt[:, k:2 * k]
    return P, V


# ------------------------------------------------------------------ 1. known answers
def _upright(m, n=1, z=3.0):
    q = np.zeros((n, m.nq))
    q[:, 2] = z
    q[:, 3:7] = [0.5, 0.5, 0.5, 0.5]
    return q


def test_known_answers(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 1)
    xp, xq = _poses(om, _upright(m, 1, 0.94))
    tx, tq = backend.t(xp), backend.t(xq)
    # vertical rays away from the robot: down from h hits the floor at h / 2; from below the floor going up: nothing
    h = np.array([0.5, 1.0, 3.0, 7.0])
    P = np.stack([[4.0, -3.0, 0.0], [-5.0, 2.0, 0.0], [3.0, 3.0, 0.0], [-4.0, -4.0, 0.0]])
    P[:, 2] = h
    V = np.tile([0.0, 0.0, -2.0], (4, 1))
    r = env.ray(backend.t(P[None]), backend.t(V[None]), xpos=tx, xquat=tq)
    assert np.array_equal(r["geomid"].cpu().numpy()[0], [0, 0, 0, 0])
    assert np.allclose(r["dist"].cpu().numpy()[0], h / 2, rtol=1e-6, atol=0)
    Pb = P.copy(); Pb[:, 2] = -h
    r = env.ray(backend.t(Pb[None]), backend.t(-V[None]), xpos=tx, xquat=tq)
    assert np.array_equal(r["geomid"].cpu().numpy()[0], [-1] * 4) and np.all(r["dist"].cpu().numpy() == -1)
    r = env.ray(backend.t(P[None]), backend.t(V[None]), xpos=tx, xquat=tq, flg_static=False)
    assert np.array_equal(r["geomid"].cpu().numpy()[0], [-1] * 4)
    # down onto the head from above: the Head geom, or with bodyexclude=Head whatever lies below it (never a Head geom)
    S = Scene(m, xp[0], xq[0])
    head = m.body_names.index("Head")
    Ph = np.array([[xp[0, head, 0], xp[0, head, 1], 3.0]])
    r = env.ray(backend.t(Ph[None]), backend.t(V[None, :1]), xpos=tx, xquat=tq)
    assert m.geom_body[r["geomid"].item() - 1] == head
    r = env.ray(backend.t(Ph[None]), backend.t(V[None, :1]), xpos=tx, xquat=tq, bodyexclude=head)
    gid = r["geomid"].item()
    assert gid == 0 or m.geom_body[gid - 1] != head
    d, ids, _ = ref_rays(S, Ph, V[:1], exclude=head)
    assert gid == ids[0]


def test_closed_form_distances(backend):
    """A capsule hit perpendicular to its axis (|p - axis| - r), a box face, a sphere from outside and from its centre (exit)."""
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 1)
    xp, xq = _poses(om, _upright(m))
    S = Scene(m, np.float64(xp[0]), np.float64(xq[0]))
    P, V, want, gids = [], [], [], []
    g = m.geom_names.index("L_Knee")                       # capsule: from 7 cm off the axis at its middle, towards the axis
    perp = np.cross(S.R[g][:, 2], [0.0, 0.0, 1.0]); perp /= np.linalg.norm(perp)
    p = S.c[g] + 0.07 * perp
    P.append(p); V.append(-0.5 * perp); want.append((0.07 - S.s[g, 0]) / 0.5); gids.append(g + 1)
    g = m.geom_names.index("Pelvis")                        # box: 5 cm in front of the +z face, along -z of the box
    ez = S.R[g][:, 2]
    P.append(S.c[g] + (S.s[g, 2] + 0.05) * ez); V.append(-ez); want.append(0.05); gids.append(g + 1)
    P, V = np.array(P), np.array(V)
    r = env.ray(backend.t(P[None]), backend.t(V[None]), xpos=backend.t(xp), xquat=backend.t(xq), flg_static=False)
    assert np.array_equal(r["geomid"].cpu().numpy()[0], gids)
    assert np.abs(r["dist"].cpu().numpy()[0] - want).max() < 2e-6
    # a sphere: the same model with the Head box replaced by a sphere of radius 0.1
    from smplsim_b200.abi import model_from_cfg
    ms = model_from_cfg(cfg)
    g = ms.geom_names.index("Head")
    ms.geom_type = ms.geom_type.copy(); ms.geom_size = ms.geom_size.copy()
    ms.geom_type[g], ms.geom_size[g] = SPHERE, [0.1, 0.0, 0.0]
    env_s = backend.batch(cfg, 1, model=ms)
    c = S.c[g]
    P = np.array([c + [0.0, 0.3, 0.0], c, c + [0.0, 0.0, 0.02]])
    V = np.array([[0.0, -2.0, 0.0], [0.0, 0.0, 4.0], [1.0, 0.0, 0.0]])
    r = env_s.ray(backend.t(P[None]), backend.t(V[None]), xpos=backend.t(xp), xquat=backend.t(xq), flg_static=False)
    assert np.array_equal(r["geomid"].cpu().numpy()[0], [g + 1] * 3)
    want = [0.2 / 2.0, 0.1 / 4.0, np.sqrt(0.1 ** 2 - 0.02 ** 2)]
    assert np.abs(r["dist"].cpu().numpy()[0] - want).max() < 2e-6


# ------------------------------------------------------------------ 2. ray against the reference
def _check_rays(m_of_row, xp, xq, P, V, out, **kw):
    worst, nguard, ntot = 0.0, 0, 0
    dk, gk = out["dist"].cpu().numpy(), out["geomid"].cpu().numpy()
    for i in range(len(xp)):
        S = Scene(m_of_row(i), xp[i], xq[i])
        d, ids, guard = ref_rays(S, P[i], V[i], **kw)
        ok = ~guard
        assert np.array_equal(gk[i][ok], ids[ok]), (i, np.nonzero(gk[i][ok] != ids[ok]))
        hit = ok & (ids >= 0)
        if hit.any():
            vn = np.linalg.norm(V[i], axis=1)
            sc = _scale(d * vn, ids, np.abs(V[i] @ S.pn) / vn)
            worst = max(worst, float((np.abs(dk[i][hit] - d[hit]) * vn[hit] / sc[hit]).max()))
        assert np.all(dk[i][ok & (ids < 0)] == -1)
        nguard += int(guard.sum()); ntot += len(guard)
    assert worst < TOL_DIST, worst
    assert nguard <= GUARD_CAP * ntot, (nguard, ntot)
    return worst, nguard / ntot


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_ray_matches_reference(backend, robot):
    cfg, om = make_models(robot=robot, control_mode="uhc_pd")
    n = 6 if robot == "smpl_humanoid" else 3
    xp, xq = _poses(om, _states(om, n, seed=21))
    rng = np.random.default_rng(2)
    P, V = _random_rays(rng, np.float64(xp), 256)
    env = backend.batch(cfg, 4)
    tP, tV = backend.t(P), backend.t(V)
    out = env.ray(tP, tV, xpos=backend.t(xp), xquat=backend.t(xq))
    w, share = _check_rays(lambda i: om.model, np.float64(xp), np.float64(xq), P, V, out)
    print(f"{robot}: worst |dx| |vec| {w:.2e} m, guard share {share:.4f}")
    b = om.model.body_names.index("L_Knee")
    out = env.ray(tP, tV, xpos=backend.t(xp), xquat=backend.t(xq), flg_static=False, bodyexclude=b)
    ids = out["geomid"].cpu().numpy()
    assert not np.isin(ids, [g + 1 for g in range(om.model.ngeom) if om.model.geom_body[g] == b]).any() and not (ids == 0).any()
    _check_rays(lambda i: om.model, np.float64(xp), np.float64(xq), P, V, out, flg_static=False, exclude=b)


def _three_shapes(tmp_path):
    from test_gpu_parity import _shape_variant
    (tmp_path / "a").mkdir(); (tmp_path / "b").mkdir()
    paths = [None, _shape_variant(tmp_path / "a", leg=1.18, arm=0.88, trunk=1.07, girth=1.15, density=1.2),
             _shape_variant(tmp_path / "b", leg=0.9, arm=1.1, trunk=0.95, girth=0.9, density=0.9)]
    return [make_models(control_mode="torque", **({"robot.xml_path": p} if p else {})) for p in paths]


def test_ray_per_env_shapes(backend, tmp_path):
    from smplsim_b200.abi import model_from_cfg
    mk = _three_shapes(tmp_path)
    n = 6
    em = np.array([i % 3 for i in range(n)], dtype=np.int32)
    q = _states(mk[0][1], n, seed=7)
    poses = [_poses(mk[em[i]][1], q[i:i + 1]) for i in range(n)]
    xp, xq = np.concatenate([p[0] for p in poses]), np.concatenate([p[1] for p in poses])
    env = backend.batch(mk[0][0], n, models=[model_from_cfg(c) for c, _ in mk], env_model=em)
    P, V = _random_rays(np.random.default_rng(4), np.float64(xp), 128)
    out = env.ray(backend.t(P), backend.t(V), xpos=backend.t(xp), xquat=backend.t(xq))
    _check_rays(lambda i: mk[em[i]][1].model, np.float64(xp), np.float64(xq), P, V, out)
    with pytest.raises(_lib.SmplsimError, match="num_envs"):
        env.ray(backend.t(P[:2]), backend.t(V[:2]), xpos=backend.t(xp[:2]), xquat=backend.t(xq[:2]))
    r = env.render("side", 32, 24, depth=True, xpos=backend.t(xp), xquat=backend.t(xq))
    assert r["depth"].shape == (n, 24, 32)


# ------------------------------------------------------------------ 3. camera conventions
def test_fixed_camera_conventions(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 3)
    q = _upright(m, 3, 0.94)
    q[1, 0] += 2.0
    q[2, 0] += 2.0; q[2, 1] += 2.0
    q[:, 0:2] -= _poses(om, q[:1])[0][0, 0, :2]          # root over the origin in row 0
    xp, xq = _poses(om, q)
    down = cam.Camera(cam.FIXED, np.array([0.0, 0.0, 10.0]), np.eye(3), fovy=30.0, zfar=77.0)
    W, H = 64, 48
    out = env.render(down, W, H, depth=True, segmentation=True, rgb=False, xpos=backend.t(xp), xquat=backend.t(xq))
    seg, dep = out["segmentation"].cpu().numpy(), out["depth"].cpu().numpy()
    rows, cols = np.nonzero(seg[1] > 0)
    assert len(cols) > 5 and cols.min() >= W // 2                  # +2 m in x: right half
    rows, cols = np.nonzero(seg[2] > 0)
    assert len(rows) > 5 and rows.max() < H // 2 and cols.min() >= W // 2   # +2 m in y as well: top half
    fl = seg == 0
    assert fl.sum() > 0.8 * seg.size and np.abs(dep[fl] - 10.0).max() < 1e-5    # z-depth, not ray length
    side = cam.fixed([-6.0, 0.0, 1.0], lookat=[0.0, 0.0, 1.0], zfar=77.0)
    out = env.render(side, W, H, depth=True, segmentation=True, rgb=False, xpos=backend.t(xp), xquat=backend.t(xq))
    seg, dep = out["segmentation"].cpu().numpy(), out["depth"].cpu().numpy()
    assert np.all(seg[:, : H // 2 - 1][seg[:, : H // 2 - 1] <= 0] == -1)     # above the horizon: sky ...
    assert np.all(dep[seg == -1] == 77.0) and (seg == -1).sum() > 0.3 * seg.size   # ... reads zfar


def test_camera_helpers():
    m = make_models(control_mode="torque")[1].model
    M = cam.xyaxes_mat([0, -1, 0, 1, 0, 2])
    assert np.allclose(M.T @ M, np.eye(3)) and np.allclose(M[:, 0], [0, -1, 0]) and np.allclose(np.cross(M[:, 0], M[:, 1]), M[:, 2])
    assert np.allclose(M[:, 1], np.array([1, 0, 2]) / np.sqrt(5))
    c = cam.named(m, "side")
    assert c.mode == cam.TRACKCOM and np.allclose(c.pos, np.array([-3.0, 0, 2.4]) - cam.robot_com(m, m.qpos0))
    c1 = cam.named(m, 1)
    assert c1.mode == c.mode and np.array_equal(c1.pos, c.pos) and np.array_equal(c1.mat, c.mat)
    assert cam.named(m, 0).name == "back" and cam.named(m, 2).name == "front_side"
    e = cam.named(m, "egocentric")
    assert e.mode == cam.BODY and e.body == e.exclude_body == m.body_names.index("Head") and e.fovy == 80.0
    for bad in (-1, 3, "top", "free"):
        with pytest.raises(ValueError, match="supported"):
            cam.named(m, bad)
    from smplsim_b200.abi import SmplsimCameraC
    assert C.sizeof(SmplsimCameraC) == 72


# ------------------------------------------------------------------ 4. render against the reference
def _check_images(S_of_row, c, W, H, out, geom_rgb=None):
    worst, nguard, ntot, nrgb = 0.0, 0, 0, 0
    dk, sk, rk = (out[k].cpu().numpy() if k in out else None for k in ("depth", "segmentation", "rgb"))
    for i in range(dk.shape[0]):
        depth, seg, rgb, guard, rguard, dn, cosf = ref_render(S_of_row(i), c, W, H, geom_rgb)
        ok = ~guard
        assert np.array_equal(sk[i][ok], seg[ok]), (i, int((sk[i][ok] != seg[ok]).sum()))
        hit = ok & (seg >= 0)
        if hit.any():
            err = np.abs(dk[i] - depth) * dn / _scale(depth * dn, seg, cosf)
            worst = max(worst, float(err[hit].max()))
        assert np.all(dk[i][ok & (seg < 0)] == c.zfar)
        if rk is not None:
            okr = ~rguard
            diff = np.abs(rk[i].astype(np.int64) - rgb.astype(np.int64))[okr]
            assert diff.max() <= 1, (i, diff.max(), int((diff > 1).sum()))
            nrgb += int(okr.sum())
        nguard += int(guard.sum()); ntot += guard.size
    assert worst < TOL_DIST, worst
    assert nguard <= GUARD_CAP * ntot, (nguard, ntot)
    return worst, nguard / ntot


@pytest.mark.parametrize("name", ["back", "side", "front_side", "egocentric"])
def test_render_matches_reference(backend, name):
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q = _states(om, 6, seed=9)
    q[0, :3] = [0.3, -0.2, 1.1]                         # one row standing-height, for the egocentric camera to see the body below
    xp, xq = _poses(om, q)
    env = backend.batch(cfg, 4)
    c = cam.named(m, name)
    W, H = 64, 48
    out = env.render(c, W, H, depth=True, segmentation=True, rgb=True, xpos=backend.t(xp), xquat=backend.t(xq))
    assert out["rgb"].shape == (6, H, W, 3) and out["rgb"].dtype == torch.uint8
    w, share = _check_images(lambda i: Scene(m, np.float64(xp[i]), np.float64(xq[i])), c, W, H, out)
    print(f"{name}: worst depth error {w:.2e} m, guard share {share:.4f}")
    if name != "egocentric":
        assert (out["segmentation"] > 0).sum().item() > 100          # the robot is in view
    # a per-geom colour table
    tab = np.random.default_rng(0).uniform(0, 1, (m.ngeom, 3))
    out = env.render(c, W, H, depth=True, segmentation=True, rgb=True, xpos=backend.t(xp[:2]), xquat=backend.t(xq[:2]), geom_rgb=tab)
    _check_images(lambda i: Scene(m, np.float64(xp[i]), np.float64(xq[i])), c, W, H, out, geom_rgb=np.float32(tab))


# ------------------------------------------------------------------ 5. tracking and body cameras
def test_trackcom_and_egocentric(backend):
    cfg, om = make_models(control_mode="uhc_pd")
    m = om.model
    q = _states(om, 4, seed=13)
    xp, xq = _poses(om, q)
    xp2 = xp + np.float32([1.75, -2.5, 0.0])               # the root translated horizontally
    env = backend.batch(cfg, 4)
    c = cam.named(m, "side")
    W, H = 64, 48
    a = env.render(c, W, H, segmentation=True, rgb=False, xpos=backend.t(xp), xquat=backend.t(xq))["segmentation"].cpu().numpy()
    b = env.render(c, W, H, segmentation=True, rgb=False, xpos=backend.t(xp2), xquat=backend.t(xq))["segmentation"].cpu().numpy()
    for i in range(len(q)):
        g1 = ref_render(Scene(m, np.float64(xp[i]), np.float64(xq[i])), c, W, H)[3]
        g2 = ref_render(Scene(m, np.float64(xp2[i]), np.float64(xq[i])), c, W, H)[3]
        ok = ~(g1 | g2)
        assert np.array_equal(np.maximum(a[i], 0)[ok], np.maximum(b[i], 0)[ok]), i     # robot pixels unchanged (floor / sky aside)
    ego = cam.named(m, "egocentric")
    head_ids = [g + 1 for g in range(m.ngeom) if m.geom_body[g] == ego.body]
    s = env.render(ego, W, H, segmentation=True, rgb=False, xpos=backend.t(xp), xquat=backend.t(xq))["segmentation"].cpu().numpy()
    assert not np.isin(s, head_ids).any()
    c2 = cam.body(m, "Head", exclude=False, xyaxes=(-1, 0, 0, 0, 1, 0))
    s2 = env.render(c2, W, H, segmentation=True, rgb=False, xpos=backend.t(xp), xquat=backend.t(xq))["segmentation"].cpu().numpy()
    assert np.all(s2 == s2[:, :1, :1]) and np.all(s2 > 0)     # without the exclusion the camera sits inside a geom and sees only it


# ------------------------------------------------------------------ 6. B1 and the motion library
def _b1_env(backend, **top):
    from smplsim_b200.envs import HumanoidSpeed
    ov = {"env.render_mode": "rgb_array"}
    ov.update(top)
    cfg = make_cfg(env="speed", seed=4, overrides=ov)

    class Env(HumanoidSpeed):
        def _make_batch(self, c, device):
            return backend.batch(c, 1, seed=4)

    return Env(cfg, device=backend.device)


def test_b1_render(backend):
    env = _b1_env(backend, headless=False)
    env.reset()
    rng = np.random.default_rng(3)
    env.step(np.clip(rng.normal(size=env.get_action_size()) * 0.3, -1, 1).astype(np.float32))
    f = env.render()
    assert isinstance(f, np.ndarray) and f.shape == (240, 320, 3) and f.dtype == np.uint8
    want = env._b.render("side", 320, 240)["rgb"][0].cpu().numpy()
    assert np.array_equal(f, want) and f.std() > 0
    env.cfg.env["camera"] = 2
    assert np.array_equal(env.render(), env._b.render("front_side", 320, 240)["rgb"][0].cpu().numpy())
    for bad in ("nope", -1):
        env.cfg.env["camera"] = bad
        with pytest.raises(ValueError, match="supported"):
            env.render()
    assert _b1_env(backend, headless=True).render() is None
    assert _b1_env(backend, **{"env.render_mode": "human", "headless": False}).render() is None


def test_motion_lib_render_clip(backend):
    from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables
    cfg, _ = make_models(control_mode="uhc_pd")
    env = backend.batch(cfg, 2)
    lib = MotionLibB200(env, synthetic_tables(env, num_clips=3, frames=5))
    v = lib.render_clip(1, camera="back", width=40, height=30)
    assert v.shape == (5, 30, 40, 3) and v.dtype == torch.uint8
    nb = env.model.nbody
    xp, xq = lib.tables["xpos"][5:10].view(5, nb, 3), lib.tables["xquat"][5:10].view(5, nb, 4)
    assert torch.equal(v, env.render("back", 40, 30, xpos=xp.contiguous(), xquat=xq.contiguous())["rgb"])
    with pytest.raises(ValueError):
        lib.render_clip(3)


# ------------------------------------------------------------------ 7. side effects, determinism, errors
def test_render_leaves_the_stepper_alone(backend):
    """step -> ray + render -> step and step -> step: every output and state row bit-identical."""
    cfg, om = make_models(env="speed", seed=5)
    m = om.model
    n = 8
    res = []
    for with_r in (False, True):
        env = backend.batch(cfg, n, seed=5, contact_wrench=True)
        env.reset()
        rng = np.random.default_rng(1)
        rows = []
        for t in range(2):
            act = backend.t(np.clip(rng.normal(size=(n, m.nu)) * 0.2, -1, 1))
            rows += [x.cpu().numpy().copy() for x in env.step(act)]
            if with_r and t == 0:
                env.render("side", 40, 30, depth=True, segmentation=True)
                env.render("egocentric", 16, 8)
                P = env.xpos[:, :1].repeat(1, 16, 1).contiguous()
                env.ray(P, torch.ones_like(P))
        rows += [x.cpu().numpy().copy() for x in (env.qpos, env.qvel, env.qacc_warm, env.qpos_fwd, env.qvel_fwd, env.ctrl, env.qacc,
                                                  env.contact_mask, env.solver_iter, env.status, env.contact_wrench, env.body_linvel,
                                                  env.xpos, env.xquat, env.obs_buf)]
        res.append(rows)
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def _determinism(backend, n, W, H):
    cfg, om = make_models(control_mode="uhc_pd")
    env = backend.batch(cfg, n)
    env.reset()
    for _ in range(2):
        env.step(backend.t(np.clip(np.random.default_rng(0).normal(size=(n, om.model.nu)) * 0.3, -1, 1)))
    a = env.render("side", W, H, depth=True, segmentation=True)
    b = env.render("side", W, H, depth=True, segmentation=True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    P = env.xpos[:, :4].contiguous()
    V = (torch.roll(env.xpos, 3, 1)[:, :4] - P).contiguous()
    r1, r2 = env.ray(P, V), env.ray(P, V)
    assert torch.equal(r1["dist"], r2["dist"]) and torch.equal(r1["geomid"], r2["geomid"])


def test_determinism(backend):
    _determinism(backend, 3, 48, 40)


@pytest.mark.gpu_only
def test_determinism_4096(backend):
    _determinism(backend, 4096, 64, 64)


def test_arguments(backend):
    cfg, om = make_models(control_mode="torque")
    m = om.model
    env = backend.batch(cfg, 2)
    env.reset()
    xp, xq = env.xpos, env.xquat
    P = backend.t(np.zeros((2, 3, 3))); V = backend.t(np.ones((2, 3, 3)))
    with pytest.raises(ValueError, match="shape"):
        env.ray(P[:, :, :2].contiguous(), V)
    with pytest.raises(ValueError, match="shape"):
        env.ray(P, V[:1])
    with pytest.raises(ValueError, match="float32"):
        env.ray(P.double(), V)
    with pytest.raises(ValueError, match="live on"):
        env.ray(P, V.to("meta"))
    with pytest.raises(ValueError, match="contiguous"):
        env.ray(P, V, xpos=xp.transpose(0, 1).contiguous().transpose(0, 1), xquat=xq)
    with pytest.raises(ValueError, match="both"):
        env.render(xpos=xp)
    with pytest.raises(ValueError, match="geom_rgb"):
        env.render(geom_rgb=np.zeros((3, 3)))
    with pytest.raises(ValueError):
        env.render(rgb=False)
    L, p = env._L(), lambda t: C.c_void_p(t.data_ptr())
    s = env._stream()
    d, g = backend.t(np.zeros((2, 3))), backend.t(np.zeros((2, 3)), torch.int32)
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 3, p(P), p(V), 1, -1, p(d), p(g), s) == 0
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 3, p(P), p(V), 1, -1, None, p(g), s) == 0
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 3, p(P), p(V), 1, m.nbody, p(d), p(g), s) == -1      # body index
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 3, p(P), p(V), 1, -2, p(d), p(g), s) == -1
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 0, p(P), p(V), 1, -1, p(d), p(g), s) == -1          # nray <= 0
    assert L.smplsim_ray(env._h, p(xp), p(xq), 2, 3, p(P), p(V), 1, -1, None, None, s) == -1          # no output
    assert L.smplsim_ray(env._h, p(xp), p(xq), -1, 3, p(P), p(V), 1, -1, p(d), p(g), s) == -1
    assert L.smplsim_ray(env._h, None, None, 0, 0, None, None, 1, -1, None, None, s) == 0              # n = 0: nothing read
    img = backend.t(np.zeros((2, 4, 4)))
    ok = cam.Camera(cam.BODY, np.zeros(3), np.eye(3), body=3, exclude_body=3).c_struct()

    def rc(c, w=4, h=4, dep=img, n=2):
        return L.smplsim_render(env._h, p(xp), p(xq), n, C.byref(c), w, h, None, None if dep is None else p(dep), None, None, s)

    assert rc(ok) == 0
    assert rc(ok, dep=None) == -1                                                                  # no output
    assert rc(ok, w=0) == -1 and rc(ok, h=-1) == -1                                                # size
    for field, val in (("body", m.nbody), ("body", -1), ("exclude_body", m.nbody), ("exclude_body", -2), ("fovy", 0.0),
                       ("fovy", 180.0), ("fovy", float("nan")), ("mode", 3)):
        bad = cam.Camera(cam.BODY, np.zeros(3), np.eye(3), body=3, exclude_body=3).c_struct()
        setattr(bad, field, val)
        assert rc(bad) == -1, (field, val)
    assert rc(ok, w=0, dep=None, n=0) == 0
    assert L.smplsim_render(env._h, p(xp), p(xq), 2, None, 4, 4, None, p(img), None, None, s) == -1
