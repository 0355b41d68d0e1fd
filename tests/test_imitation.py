"""The motion-imitation task (smplsim_imitation, HumanoidImB200): tracking observation, reward, early termination, truncation and
mpjpe against an fp64 numpy restatement of the definitions in include/smplsim.h, written here body by body with quaternion helpers of
its own; the frame rule against the gather kernel; the masked reference-state reset; the env protocol; argument checks.  Every kernel
test runs on the GPU and on the host emulator."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200 import _lib  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GUARD = 1e-5        # flags are compared outside |max distance - termination_distance| < GUARD (float32 rounding of the distance)
GUARD_CAP = 2       # ... and at most this many envs of a check may fall inside the band
SUBSET = ["L_Wrist", "R_Wrist", "L_Ankle", "R_Ankle", "Head"]        # names both SMPL and SMPL-X have


# ------------------------------------------------------------------ fp64 restatement
def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def qconj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def qrot(q, v):
    """v rotated by the unit quaternion q: q (0, v) q^-1."""
    return qmul(qmul(q, np.array([0.0, *v])), qconj(q))[1:]


def six(q):
    return np.concatenate([qrot(q, [1.0, 0, 0]), qrot(q, [0, 0, 1.0])])


def heading_inv(root, upright):
    if not upright:
        root = qmul(root, np.array([0.5, -0.5, -0.5, -0.5]))
    d = qrot(root, [1.0, 0, 0])
    hd = np.arctan2(d[1], d[0])
    return np.array([np.cos(-hd / 2), 0.0, 0.0, np.sin(-hd / 2)])


def fma32(k, dt, t0):
    """t0 + k dt with one rounding to float32 (the product of two float32 is exact in fp64)."""
    return np.float32(np.float64(np.float32(k)) * np.float64(np.float32(dt)) + np.float64(np.float32(t0)))


def restate(env, p=None):
    """obs tail, reward, mpjpe, max distance, terminated, truncated of every env from the tensors the kernel read: the batch's body
    state, the env's clip / start time / step counter, and the two table rows ``env.ref_frames`` names (the frame rule itself is held
    to the gather kernel in test_frame_rule_is_the_gathers)."""
    b, lib, e = env.batch, env.lib, env.cfg.env
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    xp, xq, lv, av = f64(b.xpos), f64(b.xquat), f64(b.body_linvel), f64(b.body_angvel)
    nb = b.model.nbody
    T = {k: f64(lib.tables[k]) for k in ("xpos", "xquat", "body_vel", "body_ang_vel")}
    fr = env.ref_frames.cpu().numpy()
    ids, t0 = env.motion_ids.cpu().numpy(), env.motion_start_times.cpu().numpy()
    prog = b.progress_buf.cpu().numpy() if p is None else p
    status = b.status.cpu().numpy()
    mlen = lib._motion_lengths.cpu().numpy()
    B, J = env.tracked_bodies, len(env.tracked_bodies)
    upright = bool(env.cfg.robot.has_upright_start)
    k = [e.im_k_pos, e.im_k_rot, e.im_k_vel, e.im_k_angvel]
    w = [e.im_w_pos, e.im_w_rot, e.im_w_vel, e.im_w_angvel]
    N = env.num_envs
    obs, rew, mp, md = np.zeros((N, 24 * J)), np.zeros(N), np.zeros(N), np.zeros(N)
    term, trunc = np.zeros(N, bool), np.zeros(N, bool)
    for i in range(N):
        h = heading_inv(xq[i, 0], upright)
        nxt = {k_: T[k_][fr[i, 1]].reshape(nb, -1) for k_ in T}
        now = {k_: T[k_][fr[i, 0]].reshape(nb, -1) for k_ in T}
        o = obs[i]
        s = np.zeros(4)
        dist = []
        for j, bd in enumerate(B):
            o[3 * j:3 * j + 3] = qrot(h, nxt["xpos"][bd] - xp[i, bd])
            o[3 * J + 6 * j:3 * J + 6 * j + 6] = six(qmul(qmul(qmul(h, nxt["xquat"][bd]), qconj(xq[i, bd])), qconj(h)))
            o[9 * J + 3 * j:9 * J + 3 * j + 3] = qrot(h, nxt["body_vel"][bd] - lv[i, bd])
            o[12 * J + 3 * j:12 * J + 3 * j + 3] = qrot(h, nxt["body_ang_vel"][bd] - av[i, bd])
            o[15 * J + 3 * j:15 * J + 3 * j + 3] = qrot(h, nxt["xpos"][bd] - xp[i, 0])
            o[18 * J + 6 * j:18 * J + 6 * j + 6] = six(qmul(h, nxt["xquat"][bd]))
            dp = now["xpos"][bd] - xp[i, bd]
            dq = qmul(now["xquat"][bd], qconj(xq[i, bd]))
            th = 2 * np.arctan2(np.linalg.norm(dq[1:]), abs(dq[0]))
            dv, dw = now["body_vel"][bd] - lv[i, bd], now["body_ang_vel"][bd] - av[i, bd]
            s += [dp @ dp, th * th, dv @ dv, dw @ dw]
            dist.append(np.sqrt(dp @ dp))
        rew[i] = sum(w[c] * np.exp(-k[c] * s[c] / J) for c in range(4))
        mp[i], md[i] = np.mean(dist), np.max(dist)
        term[i] = (prog[i] > 1 and md[i] > np.float32(e.termination_distance)) or bool(status[i] & 7)
        trunc[i] = fma32(prog[i] + 1, env.dt, t0[i]) > mlen[ids[i]] or prog[i] > e.episode_length
    return obs, rew, mp, md, term, trunc


def make_env(backend, n, robot="smpl_humanoid", v=2, tracked=None, clips=6, frames=14, seed=0, tables=None, **ov):
    cfg = make_cfg(env="im", robot=robot, overrides={"env.self_obs_v": v, **{f"env.{k}": x for k, x in ov.items()}})
    motion = tables if tables is not None else (lambda b: synthetic_tables(b, num_clips=clips, frames=frames, seed=3))
    return HumanoidImB200(cfg, motion, num_envs=n, seed=seed, tracked_bodies=tracked, batch_factory=backend.batch)


def spread(env, backend, seed=1):
    """Different clips and start times per env (times on and between frames)."""
    rng = np.random.default_rng(seed)
    K = env.lib.num_motions()
    ids = backend.t(np.arange(env.num_envs) % K, torch.int32)
    t0 = backend.t(rng.uniform(0.0, 0.2, env.num_envs))
    return ids, t0


def actions(env, backend, rng, sigma=0.5):
    return backend.t(np.clip(rng.normal(size=(env.num_envs, env.num_actions)) * sigma, -1, 1))


def check_against_restatement(env, full=True):
    obs, rew, mp, md, term, trunc = restate(env)
    S = env.batch.num_obs
    got = env.obs_buf.cpu().numpy()
    assert got.shape[1] == S + 24 * len(env.tracked_bodies) == env.num_obs
    assert np.array_equal(got[:, :S], env.batch.obs_buf.cpu().numpy())          # the stepper's self observation, copied
    # 1e-5 absolute; rows holding velocity differences above 1 m/s or rad/s (random actions) are held to 1e-5 of their largest entry:
    # a float32 rotation of a vector of length L rounds at 1e-7 L
    assert (np.abs(got[:, S:] - obs) / np.maximum(1.0, np.abs(obs).max(axis=1, keepdims=True))).max() < 1e-5
    if not full:
        return
    assert np.abs(env.rew_buf.cpu().numpy() - rew).max() < 1e-5
    assert np.abs(env.mpjpe.cpu().numpy() - mp).max() < 1e-6
    clear = np.abs(md - env.cfg.env.termination_distance) >= GUARD
    assert (~clear).sum() <= GUARD_CAP
    assert np.array_equal(env.terminate_buf.cpu().numpy().astype(bool)[clear], term[clear])
    assert np.array_equal(env.truncate_buf.cpu().numpy().astype(bool), trunc)
    assert np.array_equal(env.reset_buf.cpu().numpy().astype(bool), env.terminate_buf.cpu().numpy().astype(bool) | trunc)


# ------------------------------------------------------------------ observation, reward, flags
@pytest.mark.parametrize("robot,v,tracked,n,steps", [("smpl_humanoid", 2, None, 64, 4), ("smpl_humanoid", 1, SUBSET, 16, 3),
                                                      ("smplx_humanoid", 2, None, 8, 2), ("smplx_humanoid", 1, SUBSET, 8, 2)])
def test_obs_reward_flags_match_fp64_restatement(backend, robot, v, tracked, n, steps):
    env = make_env(backend, n, robot=robot, v=v, tracked=tracked)
    nb = env.model.nbody
    assert env.num_obs == env.batch.num_obs + 24 * (len(tracked) if tracked else nb)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    assert (env.progress_buf == 0).all()
    check_against_restatement(env, full=False)
    rng = np.random.default_rng(5)
    for _ in range(steps):
        env.step(actions(env, backend, rng))
        check_against_restatement(env)
    assert torch.isfinite(env.obs_buf).all() and (env.rew_buf > 0).all() and (env.rew_buf <= 1.0 + 1e-6).all()


def test_known_answers(backend):
    """On a reference frame the position and rotation terms equal their weights; a shifted clip gives exp(-k_p |d|^2); a root turned
    about z gives the expected angle; the termination distance is a strict bound and p <= 1 never terminates."""
    n = 8
    env = make_env(backend, n, im_k_vel=0.0, im_k_angvel=0.0)     # velocity terms pinned to their weights: the rest is exact
    e, b, nb = env.cfg.env, env.batch, env.model.nbody
    ids, t0 = spread(env, backend)
    t0 = (torch.round(t0 * 30) + 0.5) / 30                         # mid-frame: the frame rule picks the frame below, clear of rounding
    env.reset(None, motion_ids=ids, motion_times=t0)
    # the kernel is a function of the tensors it reads: evaluate it at p = 0 on the freshly reset state (reference row now = frame of t0)
    env._task(None, obs_only=False)
    assert np.allclose(env.rew_buf.cpu().numpy(), 1.0, atol=2e-5)  # w_p + w_r + w_v + w_w with zero error (FK of qpos vs the xpos table: 1e-6 m)
    assert env.mpjpe.max() < 1e-5 and not env.terminate_buf.any()
    # shift every body by d: exp(-k_p |d|^2), mpjpe |d|, rotation term untouched
    d = np.array([0.03, -0.04, 0.12])
    base = b.xpos.clone()
    b.xpos.copy_(base + backend.t(d))
    env._task(None, obs_only=False)
    want = e.im_w_pos * np.exp(-e.im_k_pos * d @ d) + e.im_w_rot + e.im_w_vel + e.im_w_angvel
    assert np.allclose(env.rew_buf.cpu().numpy(), want, atol=2e-5) and np.allclose(env.mpjpe.cpu().numpy(), np.linalg.norm(d), atol=1e-5)
    b.xpos.copy_(base)
    # turn the simulated root by a about z: th_root = a, the other bodies 0
    a = 0.7
    rz = np.array([np.cos(a / 2), 0, 0, np.sin(a / 2)])
    q0 = b.xquat.clone()
    turned = np.stack([qmul(rz, q) for q in q0[:, 0].cpu().numpy().astype(np.float64)])
    b.xquat[:, 0] = backend.t(turned)
    env._task(None, obs_only=False)
    want = e.im_w_pos + e.im_w_rot * np.exp(-e.im_k_rot * a * a / nb) + e.im_w_vel + e.im_w_angvel
    assert np.allclose(env.rew_buf.cpu().numpy(), want, atol=2e-5)
    b.xquat.copy_(q0)
    # one body termination_distance +- 1e-3 away along z at step p; the start time moved back p periods keeps the reference row
    for p, off, flag in ((2, 1e-3, True), (2, -1e-3, False), (1, 1e-3, False), (0, 1e-3, False)):
        b.xpos.copy_(base)
        b.xpos[:, 7, 2] += e.termination_distance + off
        b.progress_buf.fill_(p)
        env.motion_start_times.copy_(t0 - p * env.dt)
        env._task(None, obs_only=False)
        assert np.allclose(restate(env)[3], e.termination_distance + off, atol=1e-5)
        assert env.terminate_buf.cpu().numpy().astype(bool).tolist() == [flag] * n, (p, off)


def test_frame_rule_is_the_gathers(backend):
    """The two table rows the task kernel uses are the rows get_motion_state_intervaled picks for the same clip and time, bit for bit:
    t < 0, t past the clip's end, the last frame, frame boundaries and times between frames."""
    n = 64
    env = make_env(backend, n, clips=5, frames=9)
    lib, rng = env.lib, np.random.default_rng(2)
    L = float(lib._motion_lengths[0])
    t = rng.uniform(-0.1, L + 0.2, n)
    t[:6] = [-0.5, 0.0, L, L + 1.0, L - 1e-7, 4.5 / 30]
    ids = backend.t(rng.integers(0, 5, n), torch.int32)
    t0 = backend.t(t)
    env.motion_ids.copy_(ids); env.motion_start_times.copy_(t0)
    env.batch.progress_buf.zero_()
    env._task(None, obs_only=True)
    fr = env.ref_frames.cpu().numpy()
    now = lib.get_motion_state_intervaled(ids, t0)
    t1 = backend.t(np.array([fma32(1, env.dt, x) for x in t0.cpu().numpy()]))
    nxt = lib.get_motion_state_intervaled(ids, t1)
    assert np.array_equal(fr[:, 0], now["frame_idx"].cpu().numpy()) and np.array_equal(fr[:, 1], nxt["frame_idx"].cpu().numpy())
    for k in ("xpos", "xquat", "body_vel", "body_ang_vel"):
        tab = lib.tables[k].cpu().numpy()
        assert np.array_equal(tab[fr[:, 0]], now[k].cpu().numpy().reshape(n, -1)) and np.array_equal(tab[fr[:, 1]], nxt[k].cpu().numpy().reshape(n, -1))
    starts = lib.length_starts.cpu().numpy()[ids.cpu().numpy()]
    assert fr[0, 0] == starts[0] and fr[1, 0] == starts[1] and fr[2, 0] == starts[2] + 8 and fr[3, 0] == starts[3] + 8 and fr[5, 0] == starts[5] + 4


# ------------------------------------------------------------------ reset path
def test_masked_reset_touches_only_masked_envs(backend):
    n = 16
    env = make_env(backend, n)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    rng = np.random.default_rng(0)
    env.step(actions(env, backend, rng))
    keep = {k: getattr(env, k).clone() for k in ("obs_buf", "motion_ids", "motion_start_times", "rew_buf", "terminate_buf", "truncate_buf", "mpjpe")}
    q, v = env.batch.qpos.clone(), env.batch.qvel.clone()
    mask = torch.zeros(n, dtype=torch.uint8, device=env.device)
    mask[[1, 5, 6]] = 1
    new_ids = (ids + 2) % env.lib.num_motions()
    new_t = (torch.round((t0 + 0.1) * 30) + 0.5) / 30          # mid-frame
    env.reset(mask, motion_ids=new_ids, motion_times=new_t)
    o = ~mask.bool()
    for k in ("obs_buf", "motion_ids", "motion_start_times"):
        assert torch.equal(getattr(env, k)[o], keep[k][o]), k
    for k in ("rew_buf", "terminate_buf", "truncate_buf", "mpjpe"):         # observation-only call: untouched everywhere
        assert torch.equal(getattr(env, k), keep[k]), k
    assert torch.equal(env.batch.qpos[o], q[o]) and torch.equal(env.batch.qvel[o], v[o])
    m = mask.bool()
    assert torch.equal(env.motion_ids[m], new_ids[m]) and torch.equal(env.motion_start_times[m], new_t[m]) and (env.progress_buf[m] == 0).all()
    assert (env.progress_buf[o] == 1).all()
    # the reset envs sit on the expected frame's qpos
    lib = env.lib
    row = (lib.length_starts.long()[new_ids.long()] + torch.floor(new_t * 30).long())[m]
    assert torch.equal(env.batch.qpos[m], lib.tables["qpos"][row])
    assert torch.allclose(env.batch.xpos[m].reshape(int(m.sum()), -1), lib.tables["xpos"][row], atol=1e-5)
    check_against_restatement(env, full=False)
    # index-tensor form, sampled clips: still only those envs
    before = env.motion_start_times.clone()
    env.reset(torch.tensor([2, 3], device=env.device))
    assert torch.equal(env.motion_start_times[4:], before[4:]) and (env.progress_buf[[2, 3]] == 0).all()


def test_truncation_at_the_clips_end_and_episode_length(backend):
    n = 4
    env = make_env(backend, n, frames=7, episode_length=3, termination_distance=100.0)    # 6 frame periods = 6 control steps long
    ids = backend.t(np.zeros(n), torch.int32)
    t0 = backend.t(np.array([0.0, 2 / 30, 3.5 / 30, 0.0]))
    env.reset(None, motion_ids=ids, motion_times=t0)
    L = float(env.lib._motion_lengths[0])
    zero = backend.t(np.zeros((n, env.num_actions)))
    for p in range(1, 5):
        env.step(zero)
        want = [bool(fma32(p + 1, env.dt, x) > np.float32(L)) or p > 3 for x in t0.cpu().numpy()]
        assert env.truncate_buf.cpu().numpy().astype(bool).tolist() == want, p
        assert not env.terminate_buf.any()
    assert want == [True, True, True, True]          # env 0 and 3: p = 4 > episode_length; env 1: clip end
    # env 2 (t0 = 3.5/30, clip 6/30 long): the next target passes the end on its 2nd step
    env.reset(None, motion_ids=ids, motion_times=t0)
    env.step(zero)
    assert env.truncate_buf.cpu().numpy().tolist() == [0, 0, 0, 0]
    env.step(zero)
    assert env.truncate_buf.cpu().numpy().tolist() == [0, 0, 1, 0]


def test_stepper_autoreset_reports_terminated(backend):
    """An env whose velocity passes mj_checkVel's bound is put back to qpos0 by the stepper (status bit 2): the task reports it
    terminated, whatever its distance to the clip; the others carry on."""
    n = 4
    env = make_env(backend, n, termination_distance=100.0)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    b = env.batch
    v = b.qvel.clone()
    v[2, 8] = 1e11
    b.set_state(b.qpos.clone(), v)
    env.step(backend.t(np.zeros((n, env.num_actions))))
    assert b.status.cpu().numpy()[2] & 2
    assert env.terminate_buf.cpu().numpy().tolist() == [0, 0, 1, 0] and env.reset_buf[2] == 1
    assert torch.isfinite(env.obs_buf).all() and torch.isfinite(env.rew_buf).all()
    assert env.clip_terminations.sum() == 1 and env.clip_terminations[int(env.motion_ids[2])] == 1


# ------------------------------------------------------------------ protocol
def test_gym_wrapper_sampler_and_termination_history(backend):
    from smplsim_b200.batched import GymVectEnvB200
    from smplsim_b200.learning import BatchedSampler
    n = 8
    env = make_env(backend, n, clips=4, frames=10)
    venv = GymVectEnvB200(env)
    obs, _ = venv.reset()
    assert obs.shape == (n, env.num_obs) and torch.isfinite(obs).all()
    rng = np.random.default_rng(0)
    obs, rew, term, trunc, info = venv.step(actions(env, backend, rng))
    assert obs.shape == (n, env.num_obs) and rew.shape == (n,) and term.dtype == torch.bool and info["final_observation"].shape == obs.shape
    assert torch.isfinite(obs).all() and torch.isfinite(rew).all()
    gen = torch.Generator(device=env.device); gen.manual_seed(0)
    sampler = BatchedSampler(env, lambda o: 0.3 * torch.randn(n, env.num_actions, generator=gen, device=env.device))
    env.clip_episodes.zero_()
    batch = sampler.sample(12)                       # longer than a clip: episodes end and envs are reset in stream
    assert batch["states"].shape == (12, n, env.num_obs) and batch["rewards"].shape == (12, n)
    assert all(torch.isfinite(x).all() for x in batch.values())
    assert (batch["not_done"] == 0).any() and env.clip_episodes.sum() == (batch["not_done"] == 0).sum()
    # a failed clip draws the sampling weight
    env.clip_terminations.zero_()
    env.motion_ids.fill_(2); env._ids64.fill_(2)
    env.batch.xpos[:, 3, 2] += 5.0
    env.batch.progress_buf.fill_(2)
    env._task(None, obs_only=False)
    assert env.terminate_buf.all()
    env.clip_terminations.index_add_(0, env._ids64, env.terminate_buf.double())
    hist = env.termination_history() + 1.0
    before = env.lib._sampling_batch_prob.clone()
    assert env.lib.update_sampling_prob(hist)
    after = env.lib._sampling_batch_prob
    assert after[2] > before[2] and (after[[0, 1, 3]] < before[[0, 1, 3]]).all() and abs(float(after.sum()) - 1) < 1e-12
    assert np.bincount(env.lib.sample_motions(400).cpu().numpy(), minlength=4).argmax() == 2


def test_task_kernel_leaves_the_stepper_alone(backend):
    """A task-none batch stepped with and without the imitation kernel interleaved: qpos, qvel and self observation bit-identical."""
    n = 8
    env = make_env(backend, n)
    plain = backend.batch(env.cfg, n, seed=0)
    ids, t0 = spread(env, backend)
    env.reset(None, motion_ids=ids, motion_times=t0)
    plain.reset(None, init_mode=2, qpos0=env._qpos0, qvel0=env._qvel0)
    rng = np.random.default_rng(3)
    for _ in range(3):
        a = actions(env, backend, rng)
        env.step(a); plain.step(a)
        assert torch.equal(env.batch.qpos, plain.qpos) and torch.equal(env.batch.qvel, plain.qvel)
        assert torch.equal(env.batch.obs_buf, plain.obs_buf) and torch.equal(env.obs_buf[:, :plain.num_obs], plain.obs_buf)


def run_fixed(backend, n, steps, seed):
    env = make_env(backend, n, clips=8, frames=12, seed=seed)
    env.lib._gen.manual_seed(11)
    rng = np.random.default_rng(seed)
    env.reset()
    obs, rew = [], []
    for _ in range(steps):
        a = backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1))
        env.step(a)
        obs.append(env.obs_buf.clone()); rew.append(env.rew_buf.clone())
        env.reset_done()
        obs.append(env.obs_buf.clone())
    return torch.stack(obs), torch.stack(rew), env.clip_episodes.clone()


def test_two_runs_are_bit_identical(backend):
    a, b = run_fixed(backend, 8, 20, 4), run_fixed(backend, 8, 20, 4)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and a[2].sum() > 0


@pytest.mark.gpu_only
def test_two_runs_are_bit_identical_4096(backend):
    a, b = run_fixed(backend, 4096, 20, 4), run_fixed(backend, 4096, 20, 4)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and a[2].sum() > 0


# ------------------------------------------------------------------ arguments / ABI
def test_bad_arguments_are_refused(backend):
    n = 4
    with pytest.raises(_lib.SmplsimError, match="out of range"):
        make_env(backend, n, tracked=[0, 24])
    with pytest.raises(_lib.SmplsimError, match="num_tracked"):
        make_env(backend, n, tracked=[])
    with pytest.raises(ValueError, match="unknown body"):
        make_env(backend, n, tracked=["Tail"])
    env = make_env(backend, n)
    with pytest.raises(ValueError, match="shape"):
        env.reset(None, motion_ids=torch.zeros(n + 1, dtype=torch.int32, device=env.device))
    with pytest.raises(ValueError, match="shape"):
        env.reset(None, motion_ids=torch.zeros(n, dtype=torch.int32, device=env.device), motion_times=torch.zeros(2, device=env.device))
    # SMPL tables on an SMPL-X handle
    with pytest.raises(ValueError, match="columns"):
        make_env(backend, n, robot="smplx_humanoid", tables=synthetic_tables(env.batch, num_clips=2, frames=4))
    b, L = env.batch, env.batch._L()

    def call(icfg, tab):
        from smplsim_b200.batched import _ptr
        return L.smplsim_imitation(b._h, ctypes.byref(icfg), ctypes.byref(tab), _ptr(env.motion_ids), _ptr(env.motion_start_times),
                                   _ptr(b.progress_buf), ctypes.byref(b._aux), _ptr(b.obs_buf), None, 0, _ptr(env.obs_buf), _ptr(env.rew_buf),
                                   _ptr(env.terminate_buf), _ptr(env.truncate_buf), _ptr(env.mpjpe), None, b._stream())

    def variant(struct, **kw):
        c = type(struct)()
        ctypes.memmove(ctypes.byref(c), ctypes.byref(struct), ctypes.sizeof(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    assert call(env._icfg, env._tab) == 0
    for icfg, tab in ((env._icfg, variant(env._tab, nbody=52)), (env._icfg, variant(env._tab, num_motions=0)), (env._icfg, variant(env._tab, xquat=None)),
                      (variant(env._icfg, num_tracked=0), env._tab), (variant(env._icfg, num_tracked=25), env._tab),
                      (variant(env._icfg, tracked_bodies=None, num_tracked=5), env._tab), (variant(env._icfg, self_obs_dim=3), env._tab)):
        assert call(icfg, tab) == -1 and b"smplsim_imitation" in L.smplsim_last_error()
    bad = np.array([0, -1, 3], dtype=np.int32)
    assert call(variant(env._icfg, tracked_bodies=bad.ctypes.data, num_tracked=3), env._tab) == -1
    assert L.smplsim_imitation_obs_dim(b._h, 24) == env.num_obs and L.smplsim_imitation_obs_dim(b._h, -1) == -1


def test_abi_structs_and_version():
    from smplsim_b200.abi import SmplsimImitationCfgC, SmplsimMotionTablesC
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "smplsim.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(SmplsimImitationCfg), '
           'sizeof(SmplsimMotionTables), offsetof(SmplsimImitationCfg, tracked_bodies), offsetof(SmplsimImitationCfg, episode_length), '
           'offsetof(SmplsimMotionTables, num_motions));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        sizes = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    assert sizes == [ctypes.sizeof(SmplsimImitationCfgC), ctypes.sizeof(SmplsimMotionTablesC), SmplsimImitationCfgC.tracked_bodies.offset,
                     SmplsimImitationCfgC.episode_length.offset, SmplsimMotionTablesC.num_motions.offset]
    L = ctypes.CDLL(_lib.build())
    L.smplsim_version.restype = ctypes.c_int
    assert L.smplsim_version() >= 270
    cfg = make_cfg(env="im")
    assert cfg.env.task == "HumanoidIm" and cfg.env.state_init == "MoCap" and cfg.env.self_obs_v == 2 and cfg.robot.create_vel_sensors
    assert (cfg.env.im_k_pos, cfg.env.im_k_rot, cfg.env.im_k_vel, cfg.env.im_k_angvel) == (100.0, 10.0, 0.1, 0.1)
    assert (cfg.env.im_w_pos, cfg.env.im_w_rot, cfg.env.im_w_vel, cfg.env.im_w_angvel) == (0.5, 0.3, 0.1, 0.1) and cfg.env.termination_distance == 0.25
