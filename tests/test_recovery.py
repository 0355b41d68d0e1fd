"""Fail-state recovery for the imitation task (smplsim_imitation_recovery, HumanoidImB200's reset policy, HumanoidAmpB200's history
fill): zero-out-far observation and reward, point goal and power against an fp64 restatement of include/smplsim.h; the recovery
window; the plain task when every field is zero; recovery, fall and MoCap episodes of ``reset``; evaluation unchanged; argument
checks.  Every kernel test runs on the GPU and on the host emulator."""
import ctypes

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200.abi import SmplsimImitationRecoveryC  # noqa: E402
from smplsim_b200.amp import HumanoidAmpB200  # noqa: E402
from smplsim_b200.batched import _ptr  # noqa: E402
from smplsim_b200.imitation import RESET_FALL, RESET_MOCAP, RESET_NONE, RESET_RECOVERY  # noqa: E402
from test_imitation import GUARD, SUBSET, fma32, heading_inv, make_env, qconj, qmul, qrot, spread  # noqa: E402
from test_motion_state import six  # noqa: E402  (the rotation rule of the header, also for the unnormalised slerp)

REC = dict(zero_out_far=True, far_distance=3.0, power_coefficient=0.00005)
OFFSETS = [0.1, 0.5, 5.0]        # metres off the clip: below termination_distance, between it and far_distance, beyond far_distance


# ------------------------------------------------------------------ fp64 restatement
def refs(env, times):
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    tm = torch.as_tensor(np.asarray(times, np.float32), device=env.device)
    if env.interpolate:
        s = env.lib.get_motion_state(env.motion_ids, tm)
        return dict(p=f64(s["rg_pos"]), q=f64(s["rb_rot"]), v=f64(s["body_vel"]), w=f64(s["body_ang_vel"]))
    s = env.lib.get_motion_state_intervaled(env.motion_ids, tm)
    return dict(p=f64(s["xpos"]), q=f64(s["xquat"]), v=f64(s["body_vel"]), w=f64(s["body_ang_vel"]))


def zof(R, i, root, td, far):
    """The zeroed-out pose of env i: per-body targets (p, q, v, w or None for 'zero difference')."""
    P, q0 = R["p"][i, 0].copy(), R["q"][i, 0]
    d = np.linalg.norm(P - root)
    if d > far:
        P = root + (P - root) * far / d
    nb = R["p"].shape[1]
    if d > td:
        return [(P, q0, None, None) for _ in range(nb)]
    return [((P if b == 0 else R["p"][i, b]), R["q"][i, b], R["v"][i, b], R["w"][i, b]) for b in range(nb)]


def restate(env, goal_prev, full=True):
    """obs tail, reward, mpjpe, max distance, distance-terminated, goal distance, power of every env."""
    b, e = env.batch, env.cfg.env
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    xp, xq, lv, av = f64(b.xpos), f64(b.xquat), f64(b.body_linvel), f64(b.body_angvel)
    t0, prog = env.motion_start_times.cpu().numpy(), b.progress_buf.cpu().numpy()
    N, B, J, T = env.num_envs, env.tracked_bodies, len(env.tracked_bodies), env.num_future
    upright = bool(env.cfg.robot.has_upright_start)
    td, far, zon, pk = np.float32(e.termination_distance), np.float32(e.far_distance), bool(e.zero_out_far), float(e.power_coefficient)
    fdt = np.float32(1.0 / e.traj_sample_timestep_inv)
    t_next = [fma32(prog[i] + 1, env.dt, t0[i]) for i in range(N)]
    now = refs(env, [fma32(prog[i], env.dt, t0[i]) for i in range(N)])
    fut = [refs(env, [fma32(k, fdt, x) for x in t_next]) for k in range(T)]
    k_, w_ = [e.im_k_pos, e.im_k_rot, e.im_k_vel, e.im_k_angvel], [e.im_w_pos, e.im_w_rot, e.im_w_vel, e.im_w_angvel]
    ctrl, qvel = f64(b.ctrl), f64(b.qvel)
    obs, rew, mp, md, g, pw = (np.zeros((N, T * 24 * J)),) + tuple(np.zeros(N) for _ in range(5))
    zero = np.zeros(N, bool)
    for i in range(N):
        h, root = heading_inv(xq[i, 0], upright), xp[i, 0]
        for k, R in enumerate(fut):
            tg = zof(R, i, root, td, far) if zon else [(R["p"][i, bd], R["q"][i, bd], R["v"][i, bd], R["w"][i, bd])
                                                        for bd in range(R["p"].shape[1])]
            o = obs[i, 24 * J * k:24 * J * (k + 1)]
            for j, bd in enumerate(B):
                p_, q_, v_, w__ = tg[bd]
                o[3 * j:3 * j + 3] = qrot(h, p_ - xp[i, bd])
                o[3 * J + 6 * j:3 * J + 6 * j + 6] = six(qmul(qmul(qmul(h, q_), qconj(xq[i, bd])), qconj(h)))
                o[9 * J + 3 * j:9 * J + 3 * j + 3] = 0.0 if v_ is None else qrot(h, v_ - lv[i, bd])
                o[12 * J + 3 * j:12 * J + 3 * j + 3] = 0.0 if w__ is None else qrot(h, w__ - av[i, bd])
                o[15 * J + 3 * j:15 * J + 3 * j + 3] = qrot(h, p_ - root)
                o[18 * J + 6 * j:18 * J + 6 * j + 6] = six(qmul(h, q_))
        g[i] = np.linalg.norm((now["p"][i, 0] - root)[:2])
        tg = zof(now, i, root, td, far) if zon else None
        zero[i] = zon and np.linalg.norm(now["p"][i, 0] - root) > td
        s, dist = np.zeros(4), []
        for bd in B:
            dist.append(np.linalg.norm(now["p"][i, bd] - xp[i, bd]))
            p_, q_, v_, w__ = tg[bd] if zon else (now["p"][i, bd], now["q"][i, bd], now["v"][i, bd], now["w"][i, bd])
            dp, dq = p_ - xp[i, bd], qmul(q_, qconj(xq[i, bd]))
            dv = np.zeros(3) if v_ is None else v_ - lv[i, bd]
            dw = np.zeros(3) if w__ is None else w__ - av[i, bd]
            th = 2 * np.arctan2(np.linalg.norm(dq[1:]), abs(dq[0]))
            s += [dp @ dp, th * th, dv @ dv, dw @ dw]
        rew[i] = sum(w_[c] * np.exp(-k_[c] * s[c] / J) for c in range(4))
        if zero[i] and goal_prev is not None:
            rew[i] = np.clip((goal_prev[i] - np.float32(g[i])) / np.float32(env.dt), 0.0, 1.0)
        pw[i] = np.abs(ctrl[i] * qvel[i, 6:]).sum()
        if pk > 0 and prog[i] > 3:
            rew[i] -= pk * pw[i]
        mp[i], md[i] = np.mean(dist), np.max(dist)
    return obs, rew, mp, md, g, pw, zero


def check(env, goal_prev, full=True, obs_rows=True, rec_prev=None):
    obs, rew, mp, md, g, pw, zero = restate(env, goal_prev)
    S = env.batch.num_obs
    got = env.obs_buf.cpu().numpy()[:, S:]
    if obs_rows:
        assert (np.abs(got - obs) / np.maximum(1.0, np.abs(obs).max(axis=1, keepdims=True))).max() < 1e-5
    assert np.abs(env.goal_dist.cpu().numpy() - g).max() < 2e-6 * max(1.0, g.max())
    if not full:
        return zero
    # the point-goal reward divides a difference of float32 distances by dt: held to the kernel's own goal distance to 2e-6 of it / dt
    tol = np.where(zero, 2e-6 * np.maximum(1.0, g) / env.dt + 1e-5, 1e-5)
    assert (np.abs(env.rew_buf.cpu().numpy() - rew) <= tol + 1e-5 * np.abs(rew)).all()
    assert np.abs(env.mpjpe.cpu().numpy() - mp).max() < 1e-6 * max(1.0, mp.max())
    assert np.allclose(env.power.cpu().numpy(), pw, rtol=1e-5, atol=1e-5)
    prog = env.batch.progress_buf.cpu().numpy()
    clear = np.abs(md - env.cfg.env.termination_distance) >= GUARD
    want = (prog > 1) & (md > np.float32(env.cfg.env.termination_distance))
    if rec_prev is not None:                 # the recovery window: no distance termination, counted down
        want &= ~(rec_prev > 0)
        assert np.array_equal(env.recovery.cpu().numpy(), np.maximum(rec_prev - 1, 0))
    want |= (env.batch.status.cpu().numpy() & 7) != 0
    assert np.array_equal(env.terminate_buf.cpu().numpy().astype(bool)[clear], want[clear])
    return zero


def place_off_clip(env, backend, offsets):
    """A MoCap reset on spread clips, then every env moved horizontally off its clip by offsets[i % len(offsets)] metres."""
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    q = env._qpos0.clone()
    d = backend.t(np.array([offsets[i % len(offsets)] for i in range(env.num_envs)]))
    q[:, 0] += d * 0.6
    q[:, 1] += d * 0.8
    env.batch.reset(None, init_mode=2, qpos0=q, qvel0=env._qvel0)
    env._task(None, obs_only=True)


@pytest.mark.parametrize("robot,tracked,interp,T", [("smpl_humanoid", None, False, 1), ("smpl_humanoid", SUBSET, True, 3),
                                                    ("smplx_humanoid", SUBSET, False, 1), ("smplx_humanoid", None, True, 1)])
def test_zero_out_far_goal_and_power_match_restatement(backend, robot, tracked, interp, T):
    n = 12
    env = make_env(backend, n, robot=robot, tracked=tracked, im_interpolate=interp, num_traj_samples=T, traj_sample_timestep_inv=15, **REC)
    place_off_clip(env, backend, OFFSETS)
    check(env, None, full=False)
    rng = np.random.default_rng(7)
    seen = np.zeros(n, bool)
    for _ in range(5):        # p = 1..5: the power penalty starts at p = 4
        prev = env.goal_dist.cpu().numpy().copy()
        a = backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.3, -1, 1))
        env.step(a)
        seen |= check(env, prev)
    assert seen.any() and not seen.all()       # some envs scored by the point goal, the others by tracking
    assert (env.power.cpu().numpy() > 0).all()


def test_recovery_window_suppresses_distance_termination_only(backend):
    n, R = 6, 3
    env = make_env(backend, n, recovery_episode_prob=1.0, recovery_steps=R)
    place_off_clip(env, backend, [0.5])          # every env 0.5 m off: distance termination from p = 2 on
    env.recovery.fill_(R)
    zero_a = backend.t(np.zeros((n, env.num_actions)))
    for k in range(1, R + 3):
        env.step(zero_a)
        term = env.terminate_buf.cpu().numpy().astype(bool)
        assert (term == (k > R and k > 1)).all(), k
        assert (env.recovery.cpu().numpy() == max(R - k, 0)).all()
    # aux.status bits still terminate inside the window
    env.recovery.fill_(R)
    env.batch.status.copy_(backend.t(np.array([1, 0, 2, 0, 4, 0]), torch.uint8))
    env._task(None, obs_only=False)
    assert env.terminate_buf.cpu().numpy().tolist() == [1, 0, 1, 0, 1, 0]
    assert (env.recovery.cpu().numpy() == R - 1).all()


def test_all_fields_zero_is_the_plain_task(backend):
    """A zeroed SmplsimImitationRecovery gives bit for bit the outputs of smplsim_imitation, with one launch each."""
    n = 8
    env = make_env(backend, n)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    rng = np.random.default_rng(3)
    env.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
    outs = (env.obs_buf, env.rew_buf, env.terminate_buf, env.truncate_buf, env.mpjpe, env.ref_frames)
    want = [t.clone() for t in outs]
    for t in outs:
        t.zero_()
    env._rec = SmplsimImitationRecoveryC()
    g0 = env.gpu_launches
    env._task(None, obs_only=False)
    assert env.gpu_launches == g0 + 1
    for t, w in zip(outs, want):
        assert torch.equal(t, w)
    # a default `im` env and one with every recovery key spelled out at its off value issue the same launches
    a, b = make_env(backend, n), make_env(backend, n, fall_init_prob=0.0, recovery_episode_prob=0.0, zero_out_far=False, power_coefficient=0.0)
    assert a._rec is None and b._rec is None
    for x in (a, b):
        x.reset()
        x.step(backend.t(np.zeros((n, x.num_actions))))
        x.reset_done()
    assert a.gpu_launches == b.gpu_launches
    assert torch.equal(a.obs_buf, b.obs_buf)


def test_recovery_episodes_keep_the_state(backend):
    n, R = 8, 5
    env = make_env(backend, n, recovery_episode_prob=1.0, recovery_steps=R)
    env.reset()
    rng = np.random.default_rng(1)
    for _ in range(2):
        env.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
    term = backend.t([1, 1, 0, 0, 1, 0, 1, 0], torch.uint8)
    trunc = backend.t([0, 1, 1, 0, 0, 0, 0, 1], torch.uint8)
    env.terminate_buf.copy_(term); env.truncate_buf.copy_(trunc)
    torch.bitwise_or(term, trunc, out=env.reset_buf)
    b = env.batch
    qpos, qvel, obs, ids = b.qpos.clone(), b.qvel.clone(), env.obs_buf.clone(), env.motion_ids.clone()
    env.reset_done()
    kind = env.reset_kind.cpu().numpy()
    tm, tr = term.cpu().numpy().astype(bool), trunc.cpu().numpy().astype(bool)
    dev = lambda x: torch.as_tensor(x, device=env.device)  # noqa: E731
    assert (kind[tm] == RESET_RECOVERY).all() and (kind[tr & ~tm] == RESET_MOCAP).all() and (kind[~tm & ~tr] == RESET_NONE).all()
    assert torch.equal(b.qpos[dev(tm)], qpos[dev(tm)]) and torch.equal(b.qvel[dev(tm)], qvel[dev(tm)])
    assert (b.progress_buf.cpu().numpy()[tm | tr] == 0).all()
    assert (env.recovery.cpu().numpy()[tm] == R).all() and (env.recovery.cpu().numpy()[~tm] == 0).all()
    out = dev(~tm & ~tr)                          # untouched
    assert torch.equal(b.qpos[out], qpos[out]) and torch.equal(env.obs_buf[out], obs[out]) and torch.equal(env.motion_ids[out], ids[out])
    assert env.reset_counts.tolist() == [0, n + int((tr & ~tm).sum()), 0, int(tm.sum())]
    # an explicit reset is a MoCap reset and clears the window
    env.reset(None, motion_ids=env.motion_ids, motion_times=env.motion_start_times)
    assert (env.recovery.cpu().numpy() == 0).all() and (env.reset_kind.cpu().numpy() == RESET_MOCAP).all()


def test_fall_episodes_come_from_the_own_bank_column(backend):
    n = 6
    env = make_env(backend, n, fall_init_prob=1.0)
    bank = env.fall_qpos.cpu().numpy()
    assert bank.shape == (8, n, env.model.nq)
    assert not np.array_equal(bank[0], bank[1])          # the rounds differ
    env.reset()
    sel = np.array([1, 0, 1, 1, 0, 1], bool)
    env.terminate_buf.zero_()
    env.reset_buf.copy_(torch.as_tensor(sel, dtype=torch.uint8, device=env.device))
    qpos = env.batch.qpos.cpu().numpy().copy()
    env.reset_done()
    got = env.batch.qpos.cpu().numpy()
    kind = env.reset_kind.cpu().numpy()
    assert (kind[sel] == RESET_FALL).all() and (kind[~sel] == RESET_NONE).all()
    for i in np.flatnonzero(sel):
        assert any(np.array_equal(got[i], bank[r, i]) for r in range(8)), i
    assert np.array_equal(got[~sel], qpos[~sel])
    assert (env.recovery.cpu().numpy()[sel] == env.recovery_steps).all()


def run_seeded(backend, n, steps):
    env = make_env(backend, n, seed=4, fall_init_prob=0.3, recovery_episode_prob=0.5, **REC)
    env.reset()
    rng = np.random.default_rng(2)
    out = []
    for _ in range(steps):
        env.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
        env.reset_done()
        out.append([t.clone() for t in (env.obs_buf, env.rew_buf, env.recovery, env.goal_dist, env.power, env.reset_kind)])
    return out, env.reset_counts.tolist()


def test_two_seeded_runs_are_bit_identical(backend):
    a, ca = run_seeded(backend, 8, 6)
    b, cb = run_seeded(backend, 8, 6)
    assert ca == cb
    for x, y in zip(a, b):
        assert all(torch.equal(u, v) for u, v in zip(x, y))


def test_evaluate_is_unchanged_by_recovery(backend):
    def policy(obs):
        return torch.tanh(obs[:, :69] * 0.1)
    res = []
    for ov in ({}, dict(fall_init_prob=0.3, recovery_episode_prob=0.5, **REC)):
        env = make_env(backend, 2, clips=3, frames=10, **ov)
        env.reset()
        env.recovery.fill_(7)
        res.append(env.evaluate(policy, termination_distance=0.5))
        if ov:                                    # the evaluation's MoCap resets cleared the windows
            assert (env.recovery.cpu().numpy() == 0).all()
    assert torch.equal(res[0].sums, res[1].sums) and torch.equal(res[0].frames, res[1].frames)
    assert torch.equal(res[0].success, res[1].success)


def test_amp_history_follows_the_kinds(backend):
    n = 6
    env = make_env(backend, n, fall_init_prob=1.0, recovery_episode_prob=1.0)
    amp = HumanoidAmpB200(env)
    amp.reset()
    assert (env.reset_kind.cpu().numpy() == RESET_FALL).all()
    h = amp.amp_obs_buf.cpu().numpy()
    assert all(np.array_equal(h[i, k], h[i, 0]) for i in range(n) for k in range(h.shape[1]))     # FILL: the current frame everywhere
    rng = np.random.default_rng(0)
    for _ in range(3):
        amp.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
    term = backend.t([1, 0, 0, 1, 0, 0], torch.uint8)
    trunc = backend.t([0, 1, 0, 0, 0, 0], torch.uint8)
    env.terminate_buf.copy_(term); env.truncate_buf.copy_(trunc)
    torch.bitwise_or(term, trunc, out=env.reset_buf)
    before = amp.amp_obs_buf.clone()
    amp.reset_done()
    kind = env.reset_kind.cpu().numpy()
    assert kind.tolist()[:4] == [RESET_RECOVERY, RESET_FALL, RESET_NONE, RESET_RECOVERY]
    rec_or_none = (kind == RESET_RECOVERY) | (kind == RESET_NONE)
    assert torch.equal(amp.amp_obs_buf[torch.as_tensor(rec_or_none, device=env.device)],
                       before[torch.as_tensor(rec_or_none, device=env.device)])
    h = amp.amp_obs_buf.cpu().numpy()
    assert all(np.array_equal(h[1, k], h[1, 0]) for k in range(h.shape[1]))
    # MoCap kinds fill from the clip (the frames behind the reset time differ)
    env2 = make_env(backend, n, fall_init_prob=0.0, recovery_episode_prob=1.0)
    amp2 = HumanoidAmpB200(env2)
    amp2.reset()
    h2 = amp2.amp_obs_buf.cpu().numpy()
    assert (env2.reset_kind.cpu().numpy() == RESET_MOCAP).all()
    assert any(not all(np.array_equal(h2[i, k], h2[i, 0]) for k in range(h2.shape[1])) for i in range(n))


def test_bad_arguments_are_refused(backend):
    env = make_env(backend, 4, power_coefficient=0.00005, zero_out_far=True)
    b = env.batch
    L = b._L()

    def call(**kw):
        r = SmplsimImitationRecoveryC()
        ctypes.memmove(ctypes.byref(r), ctypes.byref(env._rec), ctypes.sizeof(r))
        for k, v in kw.items():
            setattr(r, k, v)
        return L.smplsim_imitation_recovery(b._h, ctypes.byref(env._icfg), ctypes.byref(r), ctypes.byref(env._tab), _ptr(env.motion_ids),
                                            _ptr(env.motion_start_times), _ptr(b.progress_buf), ctypes.byref(b._aux), _ptr(b.obs_buf),
                                            None, 0, _ptr(env.obs_buf), _ptr(env.rew_buf), _ptr(env.terminate_buf), _ptr(env.truncate_buf),
                                            _ptr(env.mpjpe), None, b._stream())
    assert call() == 0
    for kw in (dict(zero_out_far=2), dict(far_distance=0.0), dict(far_distance=-1.0), dict(far_distance=float("nan")), dict(goal_dist=None),
               dict(power_coefficient=-1.0), dict(power_coefficient=float("nan")), dict(qvel=None), dict(power_coefficient=0.0, qvel=None)):
        assert call(**kw) == -1 and b"smplsim_imitation" in L.smplsim_last_error(), kw
    assert call(zero_out_far=0, far_distance=0.0, goal_dist=None) == 0       # far_distance and goal_dist only matter with zero_out_far
    assert call(power_coefficient=0.0, power=None, qvel=None) == 0          # qvel only matters when the power is asked for
    assert L.smplsim_imitation_recovery(b._h, ctypes.byref(env._icfg), None, ctypes.byref(env._tab), _ptr(env.motion_ids),
                                        _ptr(env.motion_start_times), _ptr(b.progress_buf), ctypes.byref(b._aux), _ptr(b.obs_buf), None, 1,
                                        _ptr(env.obs_buf), None, None, None, None, None, b._stream()) == -1
    for kw in (dict(fall_init_prob=1.5), dict(recovery_episode_prob=-0.1), dict(recovery_steps=-1)):
        with pytest.raises(ValueError):
            make_env(backend, 2, **kw)


@pytest.mark.gpu_only
def test_kind_fractions_at_production_shape(backend):
    """4 096 SMPL envs (8-warp CTAs) at the im_recovery probabilities: the kinds within 5 sigma of their binomial means."""
    n = 4096
    env = make_env(backend, n, fall_init_prob=0.3, recovery_episode_prob=0.5, **REC)
    env.reset()
    g = torch.Generator(device=env.device); g.manual_seed(9)
    term = (torch.rand(n, generator=g, device=env.device) < 0.5).to(torch.uint8)
    env.terminate_buf.copy_(term); env.truncate_buf.copy_(1 - term)
    env.reset_buf.fill_(1)
    env.reset_done()
    kind, tm = env.reset_kind.cpu().numpy(), term.cpu().numpy().astype(bool)
    nt, nr = int(tm.sum()), int((kind == RESET_RECOVERY).sum())
    assert (kind[~tm] != RESET_RECOVERY).all()
    assert abs(nr - 0.5 * nt) < 5 * np.sqrt(nt * 0.25)
    rest = n - nr
    nf = int((kind == RESET_FALL).sum())
    assert abs(nf - 0.3 * rest) < 5 * np.sqrt(rest * 0.21)
    assert nf + nr + int((kind == RESET_MOCAP).sum()) == n
    rng = np.random.default_rng(0)
    for _ in range(3):
        prev, rec_prev = env.goal_dist.cpu().numpy().copy(), env.recovery.cpu().numpy().copy()
        env.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.3, -1, 1)))
        if _ == 2:
            # the observation rows are held to the restatement by the tests above: here envs lie on the floor, where the root's x axis
            # can point nearly straight up and the heading (atan2 of its horizontal part) is ill-conditioned in float32
            check(env, prev, obs_rows=False, rec_prev=rec_prev)
        env.reset_done()
