"""Tracking evaluation (smplsim_track_eval, HumanoidImB200.evaluate): the kernel's per-frame metrics and per-clip sums against a fixture
made by the reference's own smpl_eval functions (tests/golden/make_golden_eval.py); agreement with the imitation task's mpjpe; the
scoring window and success rule; evaluate end to end against an fp64 numpy restatement of the definitions in include/smplsim.h;
argument checks, ABI layout and reproducibility.  Every kernel test takes the suite's ``backend`` fixture: the GPU and the host
emulator."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200 import _lib  # noqa: E402
from smplsim_b200.abi import (TRACK_METRICS, SmplsimAuxC, SmplsimMotionTablesC, SmplsimTrackEvalCfgC,  # noqa: E402
                              SmplsimTrackEvalStateC)
from smplsim_b200.batched import _ptr  # noqa: E402
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import synthetic_tables  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "eval_metrics.npz")
# Tolerances against the fp64 reference on float32 inputs.  Positions are float32 values of up to ~2 m (ulp 2.4e-7 m = 2.4e-4 mm);
# a difference y - x, a norm and a 24- or 52-term mean each round at 1e-7 relative, so the distance metrics sit within a few 1e-4 mm.
# The Procrustes fit adds the float32 eigenvector of a 4x4 matrix (error ~1e-7 of its largest entry over the eigenvalue gap) times
# point distances of ~1 m: 1e-3 mm in all.  Rotation angles: a float32 quaternion product and atan2 give ~1e-7 rad, 1e-5 rad in all.
TOL_MM, TOL_RAD = 1e-3, 1e-5
TOL = np.array([TOL_MM] * 5 + [TOL_RAD])


# ------------------------------------------------------------------ fp64 restatement of include/smplsim.h (tracking evaluation)
def procrustes_err(y, x):
    """mean_j |s Q y0_j - x0_j| for the proper rotation Q and scale s of the best similarity fit of the points y onto x ([J, 3])."""
    x0, y0 = x - x.mean(0), y - y.mean(0)
    U, sv, Vt = np.linalg.svd(y0.T @ x0)           # maximise trace(Q y0^T x0): Q = V diag(1, 1, det) U^T
    dsign = np.sign(np.linalg.det(Vt.T @ U.T))
    D = np.diag([1.0, 1.0, dsign])
    Q = Vt.T @ D @ U.T
    lam = sv[0] + sv[1] + dsign * sv[2]
    s = lam / (y0 ** 2).sum()
    return np.linalg.norm(s * y0 @ Q.T - x0, axis=1).mean()


def qangle(qr, qs):
    """angle of qr (x) qs^-1 for wxyz [J, 4] arrays."""
    w1, v1 = qr[:, 0], qr[:, 1:]
    w2, v2 = qs[:, 0], -qs[:, 1:]
    w = w1 * w2 - (v1 * v2).sum(1)
    v = w1[:, None] * v2 + w2[:, None] * v1 + np.cross(v1, v2)
    return 2 * np.arctan2(np.linalg.norm(v, axis=1), np.abs(w))


def restate_clip(x, y, qr, qs):
    """Per-frame metrics [F, 6] (NaN where undefined) of one clip's scored frames: x, y [F, J, 3] reference / simulated positions,
    qr, qs [F, J, 4]; body 0 of the arrays is the root."""
    F = x.shape[0]
    out = np.full((F, 6), np.nan)
    d = y - x
    for f in range(F):
        xr, yr = x[f] - x[f, 0], y[f] - y[f, 0]
        out[f, 0] = np.linalg.norm(d[f], axis=1).mean() * 1000
        out[f, 1] = np.linalg.norm(yr - xr, axis=1).mean() * 1000
        out[f, 2] = procrustes_err(yr, xr) * 1000
        if f >= 1:
            out[f, 3] = np.linalg.norm(d[f] - d[f - 1], axis=1).mean() * 1000
        if f >= 2:
            out[f, 4] = np.linalg.norm(d[f] - 2 * d[f - 1] + d[f - 2], axis=1).mean() * 1000
        out[f, 5] = qangle(qr[f], qs[f]).mean()
    return out


# ------------------------------------------------------------------ direct kernel calls
class Eval:
    """The state arrays of smplsim_track_eval for n envs and J eval bodies on a backend, and the call."""

    def __init__(self, backend, b, J, bodies=None, interpolate=0, dt=0.0):
        dv, n = backend.device, b.num_envs
        self.b, self.backend = b, backend
        self.active = torch.ones(n, dtype=torch.uint8, device=dv)
        self.prev = torch.zeros(n, 2, J, 3, dtype=torch.float32, device=dv)
        self.frames = torch.zeros(n, dtype=torch.int32, device=dv)
        self.sums = torch.zeros(n, 6, dtype=torch.float64, device=dv)
        self.success = torch.zeros(n, dtype=torch.uint8, device=dv)
        self.fm = torch.zeros(n, 6, dtype=torch.float32, device=dv)
        self._bodies = None if bodies is None else np.ascontiguousarray(bodies, dtype=np.int32)
        self.cfg = SmplsimTrackEvalCfgC(num_bodies=J, bodies=None if bodies is None else self._bodies.ctypes.data, interpolate=interpolate, dt=dt)
        self.st = SmplsimTrackEvalStateC(active=_ptr(self.active), prev_diff=_ptr(self.prev), frames=_ptr(self.frames), sums=_ptr(self.sums),
                                         success=_ptr(self.success), frame_metrics=_ptr(self.fm))

    def __call__(self, tab, ids, t0, progress, aux, term, trunc, cfg=None, st=None):
        b = self.b
        return b._L().smplsim_track_eval(b._h, ctypes.byref(cfg or self.cfg), ctypes.byref(tab), _ptr(ids), _ptr(t0), _ptr(progress),
                                         ctypes.byref(aux), _ptr(term), _ptr(trunc), ctypes.byref(st or self.st), b._stream())


class FixtureClips:
    """The fixture group's reference clips as motion tables (row 0 of each clip a dummy pose 1 m off, rows 1..F the reference frames,
    so that step p's frame rule must land on row p) and its simulated frames as the poses aux points at."""

    def __init__(self, backend, tag):
        z = np.load(GOLDEN)
        self.z, self.tag = z, tag
        self.F = z[f"{tag}_nframes"].astype(np.int64)
        robot = "smpl_humanoid" if tag == "b24" else "smplx_humanoid"
        self.b = backend.batch(make_cfg(env="im", robot=robot), len(self.F), seed=0)
        nb = self.b.model.nbody
        gp, gr = z[f"{tag}_gt_pos"], z[f"{tag}_gt_rot"]
        assert gp.shape[1] == nb
        self.starts_fix = np.concatenate([[0], np.cumsum(self.F)[:-1]])
        rows_p, rows_q = [], []
        for c, F in enumerate(self.F):
            s = self.starts_fix[c]
            rows_p += [gp[s] + np.float32(1.0)] + list(gp[s:s + F])
            rows_q += [gr[s]] + list(gr[s:s + F])
        R = len(rows_p)
        self.dt = np.float32(1.0 / 30.0)
        t = backend.t
        self.tabs = dict(xpos=t(np.stack(rows_p).reshape(R, -1)), xquat=t(np.stack(rows_q).reshape(R, -1)), vel=t(np.zeros((R, 3 * nb))),
                         mlen=t((self.F * self.dt).astype(np.float32)), nf=t(self.F + 1, torch.int32), mdt=t(np.full(len(self.F), self.dt)),
                         starts=t(np.concatenate([[0], np.cumsum(self.F + 1)[:-1]]), torch.int32))
        T = self.tabs
        self.tab = SmplsimMotionTablesC(xpos=_ptr(T["xpos"]), xquat=_ptr(T["xquat"]), body_vel=_ptr(T["vel"]), body_ang_vel=_ptr(T["vel"]),
                                        motion_len=_ptr(T["mlen"]), num_frames=_ptr(T["nf"]), motion_dt=_ptr(T["mdt"]),
                                        length_starts=_ptr(T["starts"]), num_motions=len(self.F), nbody=nb)
        n = len(self.F)
        self.ids = t(np.arange(n), torch.int32)
        self.t0 = t(np.full(n, 0.5 * self.dt))         # mid-frame: t0 + p dt lands on row p
        self.xpos = torch.zeros(n, nb, 3, device=backend.device)
        self.xquat = torch.zeros(n, nb, 4, device=backend.device)
        self.xquat[..., 0] = 1
        self.aux = SmplsimAuxC(xpos=_ptr(self.xpos), xquat=_ptr(self.xquat))
        self.progress = torch.zeros(n, dtype=torch.int32, device=backend.device)
        self.term = torch.zeros(n, dtype=torch.uint8, device=backend.device)
        self.trunc = torch.zeros(n, dtype=torch.uint8, device=backend.device)
        self.backend, self.nb = backend, nb

    def run(self, ev, pos_key="pred", term_at=None, trunc_at=None, steps=None):
        """Steps p = 1 .. max F: clip c's frame p - 1 as the simulated pose; by default truncated at p = F.  Returns frame_metrics per step
        [P, n, 6] (NaN rows for envs that were not active) and the active mask before each step."""
        z, tag, n = self.z, self.tag, len(self.F)
        pp, pr = z[f"{tag}_{pos_key}_pos"], z[f"{tag}_{pos_key}_rot"]
        trunc_at = self.F if trunc_at is None else trunc_at
        term_at = np.full(n, 10 ** 6) if term_at is None else term_at
        fms, acts = [], []
        for p in range(1, int(self.F.max() if steps is None else steps) + 1):
            k = np.minimum(p - 1, self.F - 1) + self.starts_fix
            self.xpos.copy_(self.backend.t(pp[k]))
            self.xquat.copy_(self.backend.t(pr[k]))
            self.progress.fill_(p)
            self.trunc.copy_(self.backend.t(trunc_at == p, torch.uint8))
            self.term.copy_(self.backend.t(term_at == p, torch.uint8))
            ev.fm.fill_(float("nan"))
            acts.append(ev.active.cpu().numpy().astype(bool))
            assert ev(self.tab, self.ids, self.t0, self.progress, self.aux, self.term, self.trunc) == 0, _lib.lib().smplsim_last_error() if self.backend.name == "gpu" else ""
            fms.append(ev.fm.cpu().numpy().astype(np.float64))
        return np.stack(fms), np.stack(acts)


@pytest.mark.parametrize("tag", ["b24", "b52"])
def test_kernel_matches_reference_fixture(backend, tag):
    fx = FixtureClips(backend, tag)
    z, F, nb = fx.z, fx.F, fx.nb
    # the frame rule reads row p at step p: the reference frames themselves as the simulated poses give exact zeros for every
    # difference metric (row p - 1 or p + 1 would not: the dummy row is 1 m off, the frames move), and the fit and angles stay at
    # float32 rounding
    ev0 = Eval(backend, fx.b, nb, dt=float(fx.dt))
    fm0, _ = fx.run(ev0, pos_key="gt")
    assert np.nanmax(np.abs(fm0[..., [0, 1, 3, 4]])) == 0.0, "frame rule: step p did not read table row p"
    assert np.nanmax(fm0[..., 2]) < TOL_MM and np.nanmax(fm0[..., 5]) < TOL_RAD
    # the metrics against the reference's smpl_eval
    ev = Eval(backend, fx.b, nb, dt=float(fx.dt))
    fm, act = fx.run(ev)
    per = {k: z[f"{tag}_{k}"] for k in TRACK_METRICS}
    off = {k: 0 for k in TRACK_METRICS}
    sums = ev.sums.cpu().numpy()
    for c, Fc in enumerate(F):
        got = fm[:Fc, c]                                         # steps 1..F of clip c
        assert act[:Fc, c].all() and not act[Fc:, c].any()      # scored through its truncating step, then left alone
        for i, k in enumerate(TRACK_METRICS):
            cnt = {3: max(Fc - 1, 0), 4: max(Fc - 2, 0)}.get(i, Fc)
            want = per[k][off[k]:off[k] + cnt]
            off[k] += cnt
            vals = got[Fc - cnt:, i]
            assert np.isnan(got[:Fc - cnt, i]).all(), (k, c)
            err = np.abs(vals - want)
            assert (err <= TOL[i]).all(), (k, c, err.max(), np.argmax(err))
            assert abs(sums[c, i] - want.sum()) <= TOL[i] * max(cnt, 1), (k, c)
    assert ev.frames.cpu().numpy().tolist() == F.tolist() and ev.success.cpu().numpy().tolist() == [1] * len(F)
    # the frame-weighted means over the clips are the reference's concatenated means
    cnt = np.array([F.sum()] * 3 + [np.maximum(F - 1, 0).sum(), np.maximum(F - 2, 0).sum(), F.sum()])
    for i, k in enumerate(TRACK_METRICS):
        assert abs(sums[:, i].sum() / cnt[i] - float(z[f"{tag}_mean_{k}"])) <= TOL[i], k


def test_procrustes_special_frames(backend):
    """The planted frames of the long SMPL clip: a scaled, rotated copy aligns to ~0, a reflected copy is fitted by a proper rotation
    (the reference's sign_detR), a collinear frame and rotations near pi are scored as the reference scores them."""
    fx = FixtureClips(backend, "b24")
    ev = Eval(backend, fx.b, fx.nb, dt=float(fx.dt))
    fm, _ = fx.run(ev)
    c = int(np.argmax(fx.F))
    start = int(fx.starts_fix[c])
    pa = fx.z["b24_mpjpe_pa"]
    assert fm[5, c, 2] < 1e-3 and abs(fm[5, c, 2] - pa[start + 5]) <= TOL_MM
    assert pa[start + 9] > 100 and abs(fm[9, c, 2] - pa[start + 9]) <= TOL_MM      # a reflection would fit to ~10 mm
    assert abs(fm[13, c, 2] - pa[start + 13]) <= TOL_MM
    assert abs(fm[17, c, 5] - (np.pi - 1e-3)) < 2e-5


def test_scoring_window_and_success(backend):
    """Scoring stops on the terminating / truncating step, which is scored; inactive envs are untouched; vel / accel counts are
    frames - 1 / frames - 2; both flags on one step is a failure."""
    fx = FixtureClips(backend, "b24")              # clips of 1, 2, 3, 41, 12 frames
    ev = Eval(backend, fx.b, fx.nb, dt=float(fx.dt))
    n = len(fx.F)
    ev.active[4] = 0                               # env 4 never scored: its state is a sentinel
    ev.frames[4] = 77; ev.sums[4] = 1.5; ev.success[4] = 9; ev.prev[4] = 2.5
    term_at = np.array([10 ** 6, 2, 3, 5, 10 ** 6])
    trunc_at = np.array([1, 10 ** 6, 3, 8, 12])
    fm, act = fx.run(ev, term_at=term_at, trunc_at=trunc_at, steps=14)
    frames = ev.frames.cpu().numpy()
    assert frames.tolist() == [1, 2, 3, 5, 77]
    assert ev.success.cpu().numpy().tolist() == [1, 0, 0, 0, 9]     # env 2: terminated and truncated on step 3 -> failed
    assert ev.active.cpu().numpy().tolist() == [0] * n
    assert (ev.sums[4] == 1.5).all() and (ev.prev[4] == 2.5).all() and np.isnan(fm[:, 4]).all()
    for e in range(4):
        f = frames[e]
        assert act[:f, e].all() and not act[f:, e].any()
        assert np.isfinite(fm[:f, e, [0, 1, 2, 5]]).all() and np.isnan(fm[f:, e]).all()
        assert np.isfinite(fm[:f, e, 3]).sum() == f - 1 and np.isfinite(fm[:f, e, 4]).sum() == max(f - 2, 0)
        sums = ev.sums[e].cpu().numpy()
        assert np.allclose(sums, np.nansum(fm[:f, e], 0), rtol=1e-12, atol=0)


def make_env(backend, n, robot="smpl_humanoid", clips=5, frames=8, seed=0, **ov):
    cfg = make_cfg(env="im", robot=robot, overrides={f"env.{k}": x for k, x in ov.items()})
    return HumanoidImB200(cfg, lambda b: synthetic_tables(b, num_clips=clips, frames=frames, seed=3), num_envs=n, seed=seed,
                          batch_factory=backend.batch)


@pytest.mark.parametrize("interp", [0, 1])
def test_mpjpe_g_is_the_imitation_tasks(backend, interp):
    """On a stepped SMPL batch, frame_metrics[:, mpjpe_g] is 1000 x HumanoidImB200.mpjpe of the same step, bit for bit (the same
    frame rule, differences, norms and sum order), with and without interpolated reference states."""
    n = 16
    env = make_env(backend, n, im_interpolate=bool(interp))
    rng = np.random.default_rng(1)
    env.reset(None, motion_ids=backend.t(np.arange(n) % 5, torch.int32), motion_times=backend.t(rng.uniform(0, 0.1, n)))
    ev = Eval(backend, env.batch, env.model.nbody, interpolate=interp)
    zero = torch.zeros(n, dtype=torch.uint8, device=env.device)
    for _ in range(3):
        env.step(backend.t(np.clip(rng.normal(size=(n, env.num_actions)) * 0.5, -1, 1)))
        assert ev(env._tab, env.motion_ids, env.motion_start_times, env.batch.progress_buf, env.batch._aux, zero, zero) == 0
        assert torch.equal(ev.fm[:, 0], 1000 * env.mpjpe)
        assert torch.isfinite(ev.fm[:, [0, 1, 2, 5]]).all()


# ------------------------------------------------------------------ evaluate end to end
def policy_of(env):
    W = torch.as_tensor(np.random.default_rng(7).normal(size=(env.num_obs, env.num_actions)) * 0.02, dtype=torch.float32, device=env.device)
    return lambda obs: 0.1 * torch.tanh(obs @ W)


def hand_loop(env, clip_ids, policy, termination_distance):
    """The waves of evaluate written out: per wave one masked reset at clip time 0, then the fixed step count, each step recording the
    simulated poses, the reference row the task kernel compared (ref_frames[:, 0]) and the flags; scored by restate_clip."""
    from smplsim_b200.abi import SmplsimImitationCfgC
    N, dv, nb = env.num_envs, env.device, env.model.nbody
    steps = env.clip_steps(clip_ids)
    icfg = SmplsimImitationCfgC()
    ctypes.memmove(ctypes.byref(icfg), ctypes.byref(env._icfg), ctypes.sizeof(icfg))
    icfg.termination_distance = termination_distance
    icfg.episode_length = max(icfg.episode_length, int(steps.max()))
    TX = env.lib.tables["xpos"].cpu().numpy().astype(np.float64).reshape(-1, nb, 3)
    TQ = env.lib.tables["xquat"].cpu().numpy().astype(np.float64).reshape(-1, nb, 4)
    res = []
    for w0 in range(0, len(clip_ids), N):
        ids = clip_ids[w0:w0 + N]
        c = len(ids)
        mask = torch.zeros(N, dtype=torch.uint8, device=dv); mask[:c] = 1
        wid = torch.zeros(N, dtype=torch.int32, device=dv); wid[:c] = torch.as_tensor(ids, dtype=torch.int32)
        env.reset(mask, motion_ids=wid, motion_times=torch.zeros(N, device=dv))
        rec = []
        with torch.no_grad():
            for _ in range(int(steps[w0:w0 + c].max())):
                env.batch.step(torch.clamp(policy(env.obs_buf), -1, 1))
                env._task(None, obs_only=False, icfg=icfg)
                rec.append([x.cpu().numpy().astype(np.float64) if x.dtype == torch.float32 else x.cpu().numpy().copy()
                            for x in (env.batch.xpos, env.batch.xquat, env.ref_frames[:, 0], env.terminate_buf, env.truncate_buf)])
        for e in range(c):
            xs, ys, qr, qs = [], [], [], []
            ok = False
            for xp, xq, row, te, tr in rec:
                xs.append(TX[row[e]]); qr.append(TQ[row[e]]); ys.append(xp[e]); qs.append(xq[e])
                if te[e] or tr[e]:
                    ok = bool(tr[e]) and not bool(te[e])
                    break
            res.append((len(xs), ok, restate_clip(np.array(xs), np.array(ys), np.array(qr), np.array(qs))))
    return res


def test_evaluate_matches_hand_written_waves(backend):
    clip_ids = [0, 1, 2, 3, 4]                     # 5 clips on 2 envs: three waves, the last one ragged
    td = 0.25                                      # clips of 5 frames (4 steps): some reach their end, some terminate
    ref_env = make_env(backend, 2, frames=5)
    want = hand_loop(ref_env, clip_ids, policy_of(ref_env), td)
    env = make_env(backend, 2, frames=5)
    env.reset()
    ep, tm = env.clip_episodes.clone(), env.clip_terminations.clone()
    res = env.evaluate(policy_of(env), motion_ids=clip_ids, termination_distance=td)
    assert torch.equal(env.clip_episodes, ep) and torch.equal(env.clip_terminations, tm)
    assert (env.reset_buf == 1).all()
    assert res.frames.tolist() == [w[0] for w in want] and res.success.tolist() == [w[1] for w in want]
    m = res.metrics
    for c, (f, ok, per) in enumerate(want):
        for i, k in enumerate(TRACK_METRICS):
            vals = per[:, i][np.isfinite(per[:, i])]
            if vals.size == 0:
                assert np.isnan(float(m[k][c])), (k, c)
            else:
                assert abs(float(m[k][c]) - vals.mean()) <= TOL[i], (k, c, float(m[k][c]), vals.mean())
    assert 0 < sum(w[1] for w in want) < len(want), "the threshold should give both outcomes"
    assert res.failed_keys == [res.keys[c] for c in range(5) if not want[c][1]]
    s = res.summary()
    allf = np.concatenate([w[2] for w in want])
    for i, k in enumerate(TRACK_METRICS):
        v = allf[:, i][np.isfinite(allf[:, i])]
        assert abs(s[k] - v.mean()) <= TOL[i], k
    assert s["success_rate"] == np.mean([w[1] for w in want]) and s["num_clips"] == 5
    ss = res.summary(successful_only=True)
    okf = np.concatenate([w[2] for w in want if w[1]])
    assert abs(ss["mpjpe_g"] - okf[:, 0].mean()) <= TOL_MM and ss["num_clips"] == sum(w[1] for w in want)
    # the failed clips are what hard PMCP sampling trains on
    env.lib.update_hard_sampling_weight(res.failed_keys)
    prob = env.lib._sampling_batch_prob.cpu().numpy()
    failed = [c for c in range(5) if not want[c][1]]
    assert (prob[failed] > 0).all() and np.isclose(prob.sum(), 1.0) and (np.delete(prob, failed) == 0).all()
    # the training loop carries on: reset_done starts every env on a clip
    env.reset_done()
    assert (env.progress_buf == 0).all()


def test_evaluate_whole_library_and_eval_bodies(backend):
    env = make_env(backend, 4, clips=6, frames=6)
    res = env.evaluate(policy_of(env), termination_distance=100.0, eval_bodies=["Pelvis", "L_Wrist", "R_Wrist", "Head"])
    steps = env.clip_steps()
    assert res.motion_ids.tolist() == list(range(6)) and res.success.all() and res.frames.tolist() == steps.tolist()
    assert res.failed_keys == [] and res.keys == [str(k) for k in env.lib._motion_data_keys]
    s = res.summary()
    assert all(np.isfinite(s[k]) for k in TRACK_METRICS) and s["success_rate"] == 1.0 and s["frames"] == int(steps.sum())
    with pytest.raises(_lib.SmplsimError, match="num_bodies"):
        env.evaluate(policy_of(env), eval_bodies=[0, 1])
    with pytest.raises(ValueError, match="motion_ids"):
        env.evaluate(policy_of(env), motion_ids=[6])


def run_eval(backend, n, clips, seed):
    env = make_env(backend, n, clips=clips, frames=10, seed=seed)
    res = env.evaluate(policy_of(env), termination_distance=0.15)
    return res.sums, res.frames, res.success


def test_two_evaluations_are_bit_identical(backend):
    a, b = run_eval(backend, 3, 7, 2), run_eval(backend, 3, 7, 2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu_only
def test_two_evaluations_are_bit_identical_large(backend):
    a, b = run_eval(backend, 512, 1100, 2), run_eval(backend, 512, 1100, 2)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and a[1].sum() > 0


# ------------------------------------------------------------------ arguments / ABI
def test_bad_arguments_are_refused(backend):
    fx = FixtureClips(backend, "b24")
    ev = Eval(backend, fx.b, fx.nb)
    call = lambda cfg=None, tab=None, st=None, aux=None: ev(tab or fx.tab, fx.ids, fx.t0, fx.progress, aux or fx.aux, fx.term, fx.trunc,  # noqa: E731
                                                           cfg=cfg, st=st)
    L = fx.b._L()

    def variant(struct, **kw):
        c = type(struct)()
        ctypes.memmove(ctypes.byref(c), ctypes.byref(struct), ctypes.sizeof(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    assert call() == 0
    bad_body = np.array([0, 24, 3], dtype=np.int32)
    for kw in (dict(cfg=variant(ev.cfg, num_bodies=2, bodies=np.array([0, 1], np.int32).ctypes.data)), dict(cfg=variant(ev.cfg, num_bodies=25)),
               dict(cfg=variant(ev.cfg, num_bodies=3, bodies=bad_body.ctypes.data)), dict(cfg=variant(ev.cfg, num_bodies=5)),
               dict(cfg=variant(ev.cfg, interpolate=2)), dict(cfg=variant(ev.cfg, dt=-1.0)), dict(cfg=variant(ev.cfg, dt=float("nan"))),
               dict(tab=variant(fx.tab, nbody=52)), dict(tab=variant(fx.tab, num_motions=0)), dict(tab=variant(fx.tab, xquat=None)),
               dict(st=variant(ev.st, sums=None)), dict(st=variant(ev.st, active=None)), dict(aux=SmplsimAuxC(xpos=_ptr(fx.xpos)))):
        assert call(**kw) == -1 and b"smplsim_track_eval" in L.smplsim_last_error(), kw
    b = fx.b
    assert b._L().smplsim_track_eval(b._h, None, ctypes.byref(fx.tab), _ptr(fx.ids), _ptr(fx.t0), _ptr(fx.progress), ctypes.byref(fx.aux),
                                     _ptr(fx.term), _ptr(fx.trunc), ctypes.byref(ev.st), b._stream()) == -1
    assert call(st=variant(ev.st, frame_metrics=None)) == 0            # frame_metrics is optional


def test_abi_structs_and_version():
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "smplsim.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %d\\n", '
           'sizeof(SmplsimTrackEvalCfg), sizeof(SmplsimTrackEvalState), offsetof(SmplsimTrackEvalCfg, bodies), offsetof(SmplsimTrackEvalCfg, dt), '
           'offsetof(SmplsimTrackEvalState, sums), offsetof(SmplsimTrackEvalState, frame_metrics), SMPLSIM_TRACK_NMETRIC);return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        sizes = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    assert sizes == [ctypes.sizeof(SmplsimTrackEvalCfgC), ctypes.sizeof(SmplsimTrackEvalStateC), SmplsimTrackEvalCfgC.bodies.offset,
                     SmplsimTrackEvalCfgC.dt.offset, SmplsimTrackEvalStateC.sums.offset, SmplsimTrackEvalStateC.frame_metrics.offset,
                     len(TRACK_METRICS)]
    L = ctypes.CDLL(_lib.build())
    L.smplsim_version.restype = ctypes.c_int
    assert L.smplsim_version() == 300
