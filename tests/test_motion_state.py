"""Blended motion-library states (smplsim_motion_blend, MotionLibB200.get_motion_state / blend_into) and the options built on them:
interpolated and future imitation targets, blended AMP demonstration and MoCap-reset frames.  The kernel is held to a fixture made by
the reference's own get_motion_state (tests/golden/make_golden_motion_state.py); the tasks to the fp64 restatements of
test_imitation.py and test_amp.py fed the blended states.  Every kernel test runs on the GPU and on the host emulator."""
import ctypes
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200 import _lib  # noqa: E402
from smplsim_b200.abi import BLEND_LERP, BLEND_POS, BLEND_QPOS, BLEND_ROW0, BLEND_SLERP  # noqa: E402
from smplsim_b200.amp import HumanoidAmpB200  # noqa: E402
from test_amp import TOL as AMP_TOL, amp_frame, near_threshold, qrot as quat_rotate  # noqa: E402
from test_imitation import GUARD, GUARD_CAP, fma32, heading_inv, make_env, qconj, qmul, qrot, spread, actions  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "motion_state.npz")


def within(got, want, tol=1e-6):
    """|got - want| <= tol max(1, |want|): 1e-6 absolute / relative."""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64)) / np.maximum(1.0, np.abs(want))
    assert err.max() <= tol, err.max()


def blend_call(env, tables, kinds, ids, times, offset=None, n=None):
    """smplsim_motion_blend over caller tables [F, w] (numpy) with the clip rows of the golden fixture: outs, f0, f1, blend."""
    g = np.load(GOLDEN)
    dv = env.device
    t = lambda a, d=torch.float32: torch.as_tensor(np.ascontiguousarray(a), dtype=d, device=dv)  # noqa: E731
    tabs = [t(x.reshape(x.shape[0], -1)) for x in tables]
    n = len(ids) if n is None else n
    ids_t, tm = t(ids, torch.int32), t(times)
    meta = [t(g["motion_len"]), t(g["num_frames"], torch.int32), t(g["motion_dt"]), t(g["length_starts"], torch.int32)]
    outs = [torch.full((n, x.shape[1]), np.nan, dtype=torch.float32, device=dv) for x in tabs]
    f0, f1 = torch.zeros(n, dtype=torch.int32, device=dv), torch.zeros(n, dtype=torch.int32, device=dv)
    bl = torch.zeros(n, dtype=torch.float32, device=dv)
    off = None if offset is None else t(offset)
    k = len(tabs)
    L = env._L()
    rc = L.smplsim_motion_blend(env._h, ids_t.data_ptr(), tm.data_ptr(), n, *[m.data_ptr() for m in meta], k,
                                (ctypes.c_void_p * k)(*[x.data_ptr() for x in tabs]), (ctypes.c_int32 * k)(*[x.shape[1] for x in tabs]),
                                (ctypes.c_int32 * k)(*kinds), None if off is None else off.data_ptr(),
                                (ctypes.c_void_p * k)(*[o.data_ptr() for o in outs]), f0.data_ptr(), f1.data_ptr(), bl.data_ptr(), env._stream())
    return rc, [o.cpu().numpy() for o in outs], f0.cpu().numpy(), f1.cpu().numpy(), bl.cpu().numpy()


# ------------------------------------------------------------------ fp64 restatement of the reference's slerp
def slerp64(q0, q1, t):
    q0, q1 = np.asarray(q0, np.float64), np.asarray(q1, np.float64).copy()
    c = (q0 * q1).sum(-1)
    q1[c < 0] *= -1
    c = np.abs(c)[..., None]
    ht = np.arccos(np.minimum(c, 1.0))
    s = np.sqrt(np.maximum(1.0 - c * c, 0.0))
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.sin((1 - t) * ht) / s * q0 + np.sin(t * ht) / s * q1
    q = np.where(np.abs(s) < 0.001, 0.5 * q0 + 0.5 * q1, q)
    return np.where(c >= 1, q0, q)


def six(q):
    """six(q) with q * v evaluated as the kernels do (quat_rotate: v (2 w^2 - 1) + 2 w u x v + 2 u (u . v)): the slerped targets are not
    renormalised, and for those this is not q (0, v) q^-1."""
    return np.concatenate([quat_rotate(q, np.array([1.0, 0, 0])), quat_rotate(q, np.array([0, 0, 1.0]))])


def golden_tables(g):
    return [g["gts"], g["grs"], g["gvs"], g["gavs"], g["dof_pos"], g["dof_vel"], g["motion_aa"]]


KINDS = [BLEND_POS, BLEND_SLERP, BLEND_LERP, BLEND_LERP, BLEND_LERP, BLEND_LERP, BLEND_ROW0]
NAMES = ["rg_pos", "rb_rot", "body_vel", "body_ang_vel", "dof_pos", "dof_vel", "motion_aa"]


# ------------------------------------------------------------------ the kernel against the reference
@pytest.mark.parametrize("with_offset", [False, True])
def test_kernel_matches_reference_golden(backend, with_offset):
    g = np.load(GOLDEN)
    env = make_env(backend, 4)
    ids, times = g["ids"], g["times"]
    n = len(ids)
    rc, outs, f0, f1, bl = blend_call(env.batch, golden_tables(g), KINDS, ids, times, g["offset"] if with_offset else None)
    assert rc == 0
    starts = g["length_starts"][ids]
    assert np.array_equal(f0 - starts, g["frame_idx0"]) and np.array_equal(f1 - starts, g["frame_idx1"])
    within(bl, g["blend"])
    tag = "out_off_" if with_offset else "out_"
    for name, got in zip(NAMES, outs):
        want = g[tag + name].reshape(n, -1)
        within(got, want)
    # the planted slerp cases are all present: a negative dot product, the midpoint fallback, identical rotations
    q0, q1 = g["grs"][f0], g["grs"][f1]
    c = (q0.astype(np.float64) * q1).sum(-1)
    mid = (bl > 0) & (bl < 1)
    assert (c[mid] < 0).any() and (np.sqrt(np.maximum(1 - c[mid] ** 2, 0)) < 1e-3).any() and (np.abs(q0 - q1).max(-1)[mid] == 0).any()


def test_qpos_and_qvel_extension_against_restatement(backend):
    """QPOS: lerp with the root quaternion slerped and the offset on the root position; qvel rows: LERP."""
    g = np.load(GOLDEN)
    env = make_env(backend, 4)
    ids, times, off = g["ids"], g["times"], g["offset"]
    qpos = np.concatenate([g["gts"][:, 0], g["grs"][:, 0], g["dof_pos"]], axis=1)
    qvel = np.concatenate([g["gvs"][:, 0], g["gavs"][:, 0], g["dof_vel"]], axis=1)
    rc, (gq, gv), f0, f1, bl = blend_call(env.batch, [qpos, qvel], [BLEND_QPOS, BLEND_LERP], ids, times, off)
    assert rc == 0
    b = bl.astype(np.float64)[:, None]
    want_q = (1 - b) * qpos[f0] + b * qpos[f1]
    want_q[:, :3] += off
    want_q[:, 3:7] = slerp64(qpos[f0, 3:7], qpos[f1, 3:7], b)
    within(gq, want_q, 1e-5)
    within(gv, (1 - b) * qvel[f0] + b * qvel[f1], 1e-5)
    # and the reference's own pieces: root position with the offset, root rotation, joint angles
    within(gq, np.concatenate([g["out_off_root_pos"], g["out_off_root_rot"], g["out_off_dof_pos"]], axis=1))
    within(gv, np.concatenate([g["out_off_root_vel"], g["out_off_root_ang_vel"], g["out_off_dof_vel"]], axis=1))


# ------------------------------------------------------------------ known answers
def test_known_answers(backend):
    env = make_env(backend, 4, clips=5, frames=9)
    lib = env.lib
    dt = float(lib._motion_dt[0])
    # on a frame time the blend is the gather
    ids = backend.t(np.repeat(np.arange(5), 9), torch.int32)
    t = backend.t(np.tile(np.arange(9, dtype=np.float32) * np.float32(dt), 5))
    s, r = lib.get_motion_state(ids, t), lib.get_motion_state_intervaled(ids, t)
    for k in ("xpos", "body_vel", "body_ang_vel", "dof_pos", "dof_vel", "qvel"):
        within(s["rg_pos" if k == "xpos" else k].cpu().numpy().reshape(45, -1), r[k].cpu().numpy().reshape(45, -1))
    within(s["qpos"][:, [0, 1, 2] + list(range(7, lib.tables["qpos"].shape[1]))].cpu().numpy(),
           r["qpos"][:, [0, 1, 2] + list(range(7, lib.tables["qpos"].shape[1]))].cpu().numpy())
    # rotations: the reference's slerp at blend 0 returns q0 scaled by sin(acos c) / sqrt(1 - c^2) (not normalised: 1 to rounding of
    # c^2), and the midpoint of the pair when it is within 0.002 rad: the direction of the gathered rotation to 1e-6 in the dot product
    got = np.concatenate([s["rb_rot"].cpu().numpy().reshape(-1, 4), s["qpos"][:, 3:7].cpu().numpy()]).astype(np.float64)
    want = np.concatenate([r["xquat"].cpu().numpy().reshape(-1, 4), r["qpos"][:, 3:7].cpu().numpy()]).astype(np.float64)
    assert (np.abs((got / np.linalg.norm(got, axis=1, keepdims=True) * want).sum(1)) >= 1 - 1e-6).all()
    assert set(s) >= {"root_pos", "root_rot", "dof_pos", "root_vel", "root_ang_vel", "dof_vel", "motion_aa", "rg_pos", "rb_rot", "body_vel",
                      "body_ang_vel", "motion_bodies", "qpos", "qvel", "frame_idx0", "frame_idx1", "blend"}
    # an offset moves every body position and the qpos root, nothing else
    d = np.array([0.5, -1.0, 0.25], np.float32)
    so = lib.get_motion_state(ids, t, offset=backend.t(np.tile(d, (45, 1))))
    within(so["rg_pos"].cpu().numpy(), s["rg_pos"].cpu().numpy() + d)
    within(so["qpos"].cpu().numpy()[:, :3], s["qpos"].cpu().numpy()[:, :3] + d)
    assert torch.equal(so["rb_rot"], s["rb_rot"]) and torch.equal(so["qpos"][:, 3:], s["qpos"][:, 3:])
    # half way between identity and a turn by a about z: the turn by a / 2
    a = 1.1
    qz = lambda x: np.array([np.cos(x / 2), 0, 0, np.sin(x / 2)], np.float32)  # noqa: E731
    g = np.load(GOLDEN)
    rot = np.zeros((int(g["num_frames"].sum()), 4), np.float32)
    rot[:, 0] = 1
    s1 = g["length_starts"][1]
    rot[s1 + 1] = qz(a)
    rc, (q,), f0, f1, bl = blend_call(env.batch, [rot], [BLEND_SLERP], np.array([1]), np.array([0.5 * g["motion_dt"][1]], np.float32))
    assert rc == 0 and bl[0] == np.float32(0.5) and (f0[0], f1[0]) == (s1, s1 + 1)
    within(q[0], qz(a / 2))


# ------------------------------------------------------------------ imitation: blended and future targets
def restate_blended(env, T, fdt):
    """The observation tail, reward, mpjpe, max distance and flags with ref(t) = get_motion_state (nearest frames:
    get_motion_state_intervaled when the env does not interpolate), T targets fdt apart."""
    b, lib, e = env.batch, env.lib, env.cfg.env
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    xp, xq, lv, av = f64(b.xpos), f64(b.xquat), f64(b.body_linvel), f64(b.body_angvel)
    ids, t0 = env.motion_ids.cpu().numpy(), env.motion_start_times.cpu().numpy()
    prog = b.progress_buf.cpu().numpy()
    N, B, J = env.num_envs, env.tracked_bodies, len(env.tracked_bodies)
    upright = bool(env.cfg.robot.has_upright_start)
    mlen = lib._motion_lengths.cpu().numpy()

    def ref(times):
        tm = torch.as_tensor(np.asarray(times, np.float32), device=env.device)
        if env.interpolate:
            s = lib.get_motion_state(env.motion_ids, tm)
            return {k: f64(s[k]) for k in ("rg_pos", "rb_rot", "body_vel", "body_ang_vel")}, s["frame_idx0"].cpu().numpy()
        s = lib.get_motion_state_intervaled(env.motion_ids, tm)
        return dict(rg_pos=f64(s["xpos"]), rb_rot=f64(s["xquat"]), body_vel=f64(s["body_vel"]), body_ang_vel=f64(s["body_ang_vel"])), s["frame_idx"].cpu().numpy()

    t_now = [fma32(prog[i], env.dt, t0[i]) for i in range(N)]
    t_next = [fma32(prog[i] + 1, env.dt, t0[i]) for i in range(N)]
    now, f_now = ref(t_now)
    fut = [ref([fma32(k, fdt, x) for x in t_next]) for k in range(T)]
    k_, w_ = [e.im_k_pos, e.im_k_rot, e.im_k_vel, e.im_k_angvel], [e.im_w_pos, e.im_w_rot, e.im_w_vel, e.im_w_angvel]
    obs = np.zeros((N, T * 24 * J))
    rew, mp, md = np.zeros(N), np.zeros(N), np.zeros(N)
    term, trunc = np.zeros(N, bool), np.zeros(N, bool)
    for i in range(N):
        h = heading_inv(xq[i, 0], upright)
        for k, (nx, _) in enumerate(fut):
            o = obs[i, 24 * J * k:24 * J * (k + 1)]
            for j, bd in enumerate(B):
                o[3 * j:3 * j + 3] = qrot(h, nx["rg_pos"][i, bd] - xp[i, bd])
                o[3 * J + 6 * j:3 * J + 6 * j + 6] = six(qmul(qmul(qmul(h, nx["rb_rot"][i, bd]), qconj(xq[i, bd])), qconj(h)))
                o[9 * J + 3 * j:9 * J + 3 * j + 3] = qrot(h, nx["body_vel"][i, bd] - lv[i, bd])
                o[12 * J + 3 * j:12 * J + 3 * j + 3] = qrot(h, nx["body_ang_vel"][i, bd] - av[i, bd])
                o[15 * J + 3 * j:15 * J + 3 * j + 3] = qrot(h, nx["rg_pos"][i, bd] - xp[i, 0])
                o[18 * J + 6 * j:18 * J + 6 * j + 6] = six(qmul(h, nx["rb_rot"][i, bd]))
        s, dist = np.zeros(4), []
        for bd in B:
            dp = now["rg_pos"][i, bd] - xp[i, bd]
            dq = qmul(now["rb_rot"][i, bd], qconj(xq[i, bd]))
            th = 2 * np.arctan2(np.linalg.norm(dq[1:]), abs(dq[0]))
            dv, dw = now["body_vel"][i, bd] - lv[i, bd], now["body_ang_vel"][i, bd] - av[i, bd]
            s += [dp @ dp, th * th, dv @ dv, dw @ dw]
            dist.append(np.sqrt(dp @ dp))
        rew[i] = sum(w_[c] * np.exp(-k_[c] * s[c] / J) for c in range(4))
        mp[i], md[i] = np.mean(dist), np.max(dist)
        term[i] = (prog[i] > 1 and md[i] > np.float32(e.termination_distance)) or bool(b.status.cpu().numpy()[i] & 7)
        trunc[i] = t_next[i] > mlen[ids[i]] or prog[i] > e.episode_length
    return obs, rew, mp, md, term, trunc, f_now, fut[0][1]


def check_blended(env, T, fdt, full=True):
    obs, rew, mp, md, term, trunc, f_now, f_next = restate_blended(env, T, fdt)
    S = env.batch.num_obs
    got = env.obs_buf.cpu().numpy()
    assert got.shape[1] == S + T * 24 * len(env.tracked_bodies) == env.num_obs
    assert np.array_equal(got[:, :S], env.batch.obs_buf.cpu().numpy())
    assert (np.abs(got[:, S:] - obs) / np.maximum(1.0, np.abs(obs).max(axis=1, keepdims=True))).max() < 1e-5
    fr = env.ref_frames.cpu().numpy()
    assert np.array_equal(fr[:, 1], f_next)
    if not full:
        return
    assert np.array_equal(fr[:, 0], f_now)
    assert np.abs(env.rew_buf.cpu().numpy() - rew).max() < 1e-5
    assert np.abs(env.mpjpe.cpu().numpy() - mp).max() < 1e-6
    clear = np.abs(md - env.cfg.env.termination_distance) >= GUARD
    assert (~clear).sum() <= GUARD_CAP
    assert np.array_equal(env.terminate_buf.cpu().numpy().astype(bool)[clear], term[clear])
    assert np.array_equal(env.truncate_buf.cpu().numpy().astype(bool), trunc)


@pytest.mark.parametrize("interp,T", [(True, 3), (True, 1), (False, 3)])
def test_imitation_blended_future_targets_match_restatement(backend, interp, T):
    n = 16
    env = make_env(backend, n, im_interpolate=interp, num_traj_samples=T, traj_sample_timestep_inv=15)
    assert env.num_obs == env.batch.num_obs + 24 * env.model.nbody * T
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    check_blended(env, T, np.float32(1 / 15), full=False)
    rng = np.random.default_rng(5)
    for _ in range(3):
        env.step(actions(env, backend, rng))
        check_blended(env, T, np.float32(1 / 15))


def test_defaults_are_the_nearest_frame_task(backend):
    """interpolate = 0 and T = 1 (the cfg defaults, and num_future = 0 in the C struct) give the rows of the task without options."""
    n = 8
    a, b = make_env(backend, n), make_env(backend, n, im_interpolate=False, num_traj_samples=1)
    ids, t0 = spread(a, backend)
    for env in (a, b):
        env.reset(None, motion_ids=ids, motion_times=t0)
    assert torch.equal(a.obs_buf, b.obs_buf) and a._icfg.num_future == 1
    a._icfg.num_future = 0
    a._task(None, obs_only=True)
    assert torch.equal(a.obs_buf, b.obs_buf)


def test_interpolating_reset_lands_on_the_blended_qpos(backend):
    n = 8
    env = make_env(backend, n, im_interpolate=True)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    s = env.lib.get_motion_state(ids, t0)
    assert torch.equal(env.batch.qpos, s["qpos"]) and torch.equal(env.batch.qvel, s["qvel"])
    assert (s["blend"] > 0).any()                                  # the start times fall between frames
    check_blended(env, 1, np.float32(1 / 30), full=False)


# ------------------------------------------------------------------ AMP
def blended_frame(lib, ids, times, amp_cfg, upright):
    """test_amp.py's restated frame fed the blended states of get_motion_state."""
    s = lib.get_motion_state(torch.as_tensor(np.asarray(ids), dtype=torch.int32, device=lib.env.device),
                             torch.as_tensor(np.asarray(times), dtype=torch.float32, device=lib.env.device))
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    from smplsim_b200.amp import amp_c_cfg
    xp, xq = f64(s["rg_pos"]), f64(s["rb_rot"])
    keys = amp_c_cfg(lib.env.model, amp_cfg)[1]
    return amp_frame(xp[:, 0], xq[:, 0], f64(s["root_vel"]), f64(s["root_ang_vel"]), f64(s["dof_pos"]), f64(s["dof_vel"]), xp[:, keys],
                     upright, amp_cfg["local_root_obs"], amp_cfg["root_height_obs"]), near_threshold(f64(s["dof_pos"]))


def close(got, want, skip):
    err = (np.abs(got - want) / np.maximum(1.0, np.abs(want).max(axis=-1, keepdims=True)))[~skip]
    assert err.max() < AMP_TOL, err.max()


def test_amp_blended_demo_and_fill_ref_match_restatement(backend):
    n = 8
    env = make_env(backend, n, im_interpolate=True)
    amp = HumanoidAmpB200(env)
    assert amp.cfg["interpolate"] and amp._ccfg.interpolate == 1       # taken from the imitation env
    K, lib, dt = amp.num_amp_obs_steps, env.lib, env.dt
    up = bool(env.cfg.robot.has_upright_start)
    ids = backend.t(np.arange(n) % lib.num_motions(), torch.int32)
    t0 = backend.t(np.array([0.0, 0.05, 0.1, 0.2, 0.31, 0.4, 0.02, 0.43]))
    amp.reset(None, motion_ids=ids, motion_times=t0)
    got = amp.amp_obs_buf.cpu().numpy()
    idn, tn = ids.cpu().numpy(), t0.cpu().numpy()
    for k in range(1, K):
        close(got[:, k], *blended_frame(lib, idn, [fma32(-k, dt, x) for x in tn], amp.cfg, up))
    L = float(lib._motion_lengths[0])
    times = np.array([0.0, 0.01, L, L + 0.5, -0.2, L / 2, 0.3, 0.12], dtype=np.float32)
    demo = lib.amp_obs_demo(motion_ids=ids, motion_times=backend.t(times)).cpu().numpy()
    for k in range(K):
        close(demo[:, k], *blended_frame(lib, idn, [fma32(-k, dt, x) for x in times], amp.cfg, up))
    # the caller's key wins; nearest-frame demo rows differ from the blended ones
    plain = HumanoidAmpB200(env, amp_cfg={"interpolate": False})
    nd = lib.amp_obs_demo(motion_ids=ids, motion_times=backend.t(times)).cpu().numpy()
    assert plain.cfg["interpolate"] is False and plain._ccfg.interpolate == 0 and not np.array_equal(nd, demo)


# ------------------------------------------------------------------ arguments, determinism
def test_bad_arguments_are_refused(backend):
    g = np.load(GOLDEN)
    env = make_env(backend, 4)
    b, L = env.batch, env.batch._L()
    ids, times = g["ids"][:4], g["times"][:4]
    for tabs, kinds in (([g["gvs"]], [7]), ([g["gvs"]], [-1]), ([g["gts"]], [BLEND_SLERP]), ([g["dof_pos"][:, :5]], [BLEND_POS]),
                        ([g["dof_pos"][:, :5]], [BLEND_QPOS])):
        rc = blend_call(b, tabs, kinds, ids, times)[0]
        assert rc == -1 and b"smplsim_motion_blend" in L.smplsim_last_error()
    assert blend_call(b, [g["gvs"]], [BLEND_LERP], ids, times)[0] == 0

    def variant(struct, **kw):
        c = type(struct)()
        ctypes.memmove(ctypes.byref(c), ctypes.byref(struct), ctypes.sizeof(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    from smplsim_b200.batched import _ptr
    def call(icfg):
        return L.smplsim_imitation(b._h, ctypes.byref(icfg), ctypes.byref(env._tab), _ptr(env.motion_ids), _ptr(env.motion_start_times),
                                   _ptr(b.progress_buf), ctypes.byref(b._aux), _ptr(b.obs_buf), None, 1, _ptr(env.obs_buf), None, None, None,
                                   None, None, b._stream())
    assert call(env._icfg) == 0
    for kw in (dict(num_future=-1), dict(future_dt=-0.1), dict(future_dt=float("nan")), dict(interpolate=2)):
        assert call(variant(env._icfg, **kw)) == -1 and b"smplsim_imitation" in L.smplsim_last_error()
    with pytest.raises(ValueError, match="num_traj_samples"):
        make_env(backend, 4, num_traj_samples=0)
    amp = HumanoidAmpB200(env)
    F = L.smplsim_amp_obs_dim(b._h, ctypes.byref(variant(amp._ccfg, interpolate=3)))
    assert F == -1 and b"interpolate" in L.smplsim_last_error()


def test_abi_structs_and_version():
    import subprocess
    import tempfile
    from smplsim_b200.abi import SmplsimAmpCfgC, SmplsimImitationCfgC
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "smplsim.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", '
           'sizeof(SmplsimImitationCfg), offsetof(SmplsimImitationCfg, interpolate), offsetof(SmplsimImitationCfg, num_future), '
           'offsetof(SmplsimImitationCfg, future_dt), sizeof(SmplsimAmpCfg), offsetof(SmplsimAmpCfg, interpolate)); return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(d, "s")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    assert sizes == [ctypes.sizeof(SmplsimImitationCfgC), SmplsimImitationCfgC.interpolate.offset, SmplsimImitationCfgC.num_future.offset,
                     SmplsimImitationCfgC.future_dt.offset, ctypes.sizeof(SmplsimAmpCfgC), SmplsimAmpCfgC.interpolate.offset]
    L = ctypes.CDLL(_lib.build())
    L.smplsim_version.restype = ctypes.c_int
    assert L.smplsim_version() >= 290


def run_fixed(backend, n, steps):
    env = make_env(backend, n, clips=8, frames=12, seed=4, im_interpolate=True, num_traj_samples=3)
    env.lib._gen.manual_seed(11)
    amp = HumanoidAmpB200(env)
    rng = np.random.default_rng(4)
    amp.reset()
    out = []
    for _ in range(steps):
        amp.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
        out += [env.obs_buf.clone(), env.rew_buf.clone(), amp.amp_obs_buf.clone()]
        amp.reset_done()
        out += [env.obs_buf.clone(), amp.amp_obs_buf.clone()]
    return out, env.clip_episodes.clone()


def test_two_runs_are_bit_identical(backend):
    (a, ea), (b, eb) = run_fixed(backend, 8, 12), run_fixed(backend, 8, 12)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(ea, eb)


@pytest.mark.gpu_only
def test_two_runs_are_bit_identical_4096(backend):
    (a, ea), (b, eb) = run_fixed(backend, 4096, 20), run_fixed(backend, 4096, 20)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and torch.equal(ea, eb) and ea.sum() > 0
