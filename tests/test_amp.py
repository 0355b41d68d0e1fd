"""Adversarial motion priors (smplsim_amp_obs / smplsim_amp_demo, smplsim_b200.amp): the per-frame feature against an fp64 numpy
restatement of include/smplsim.h, the restatement against the reference's own compute_humanoid_observations_smpl (tests/golden/
amp_obs.npz); the history push / fill / MoCap fill and the demonstration rows on stepped states; masks, determinism, argument checks;
the discriminator's reward and loss terms against hand-written autograd, the replay buffer, the gradient average over ranks.  Every
kernel test runs on the GPU and on the host emulator."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from smplsim_b200 import _lib  # noqa: E402
from smplsim_b200.amp import (AMP_DEFAULTS, AMPDiscriminator, AMPLearner, AMPReplayBuffer, HumanoidAmpB200, amp_c_cfg,  # noqa: E402
                              disc_loss_terms, disc_total_loss)
from smplsim_b200.cfg import make_cfg  # noqa: E402
from smplsim_b200.imitation import HumanoidImB200  # noqa: E402
from smplsim_b200.motion_lib import MotionLibB200, synthetic_tables  # noqa: E402

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "amp_obs.npz")
KEYS = ["R_Ankle", "L_Ankle", "R_Wrist", "L_Wrist"]
TOL = 2e-5          # fp32 kernel vs fp64 restatement, relative to max(1, |row|_inf)
GUARD = 1e-6        # exp-map norms within this of the 1e-5 threshold (or of 2 pi multiples) are not compared


# ------------------------------------------------------------------ fp64 restatement (wxyz)
def qmul(a, b):
    aw, ax, ay, az = np.moveaxis(a, -1, 0)
    bw, bx, by, bz = np.moveaxis(b, -1, 0)
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], -1)


def qrot(q, v):
    w, u = q[..., :1], q[..., 1:]
    return v * (2 * w * w - 1) + 2 * w * np.cross(u, v) + 2 * u * np.sum(u * v, -1, keepdims=True)


def tan_norm(q):
    e = np.zeros(q.shape[:-1] + (3,))
    x, z = e.copy(), e.copy()
    x[..., 0] = 1
    z[..., 2] = 1
    return np.concatenate([qrot(q, x), qrot(q, z)], -1)


def heading_inv(r):
    d = qrot(r, np.broadcast_to([1.0, 0, 0], r.shape[:-1] + (3,)))
    hd = np.arctan2(d[..., 1], d[..., 0])
    return np.stack([np.cos(-hd / 2), 0 * hd, 0 * hd, np.sin(-hd / 2)], -1)


def exp_map_quat(e):
    a = np.linalg.norm(e, axis=-1)
    w = np.arctan2(np.sin(a), np.cos(a))
    ax = e / np.maximum(a, 1e-300)[..., None]
    q = np.concatenate([np.cos(w / 2)[..., None], ax * np.sin(w / 2)[..., None]], -1)
    q[np.abs(w) <= 1e-5] = [1, 0, 0, 0]
    return q


def amp_frame(root_pos, root_rot, root_vel, root_ang_vel, dof_pos, dof_vel, key_pos, upright, local, root_h):
    """One AMP frame per row, as include/smplsim.h states it (rows: leading axis; quaternions wxyz)."""
    r = root_rot if upright else qmul(root_rot, np.broadcast_to([0.5, -0.5, -0.5, -0.5], root_rot.shape))
    h = heading_inv(r)
    m = root_pos.shape[0]
    parts = [root_pos[:, 2:3]] if root_h else []
    parts += [tan_norm(qmul(h, r) if local else r), qrot(h, root_vel), qrot(h, root_ang_vel),
              tan_norm(exp_map_quat(dof_pos.reshape(m, -1, 3))).reshape(m, -1), dof_vel,
              qrot(h[:, None], key_pos - root_pos[:, None]).reshape(m, -1)]
    return np.concatenate(parts, -1)


def near_threshold(dof_pos):
    a = np.linalg.norm(dof_pos.reshape(dof_pos.shape[0], -1, 3), axis=-1)
    w = np.abs(np.arctan2(np.sin(a), np.cos(a)))
    return (np.abs(w - 1e-5) < GUARD).any(-1)


def test_restatement_matches_reference_golden():
    """The restatement above against compute_humanoid_observations_smpl run by the reference's own code (fp64, xyzw converted at the
    boundary): random states, the zero pose, exp-map norms just above / below 1e-5 and above pi, upright_start / local_root_obs /
    root_height_obs on and off, SMPL and SMPL-X widths."""
    g = np.load(GOLDEN)
    seen = set()
    for i, (nb, upright, local, root_h) in enumerate(g["cases"]):
        s = {k: g[f"c{i}_{k}"] for k in ("root_pos", "root_rot", "root_vel", "root_ang_vel", "dof_pos", "dof_vel", "key_pos")}
        got = amp_frame(**s, upright=upright, local=local, root_h=root_h)
        want = g[f"c{i}_obs"]
        assert got.shape == want.shape == (24, root_h + 12 + 6 * (nb - 1) + 3 * (nb - 1) + 12)
        assert np.abs(got - want).max() < 1e-10, i
        seen.add((int(nb), int(upright), int(local), int(root_h)))
    assert len(seen) == 10 and (24, 0, 1, 1) in seen and (52, 0, 1, 1) in seen
    widths = {(int(c[0]), int(c[3])): g[f"c{i}_obs"].shape[1] for i, c in enumerate(g["cases"])}
    assert widths[(24, 1)] == 232 and widths[(52, 1)] == 484


# ------------------------------------------------------------------ envs
def tables_for(b, clips=6, frames=14, seed=3):
    return synthetic_tables(b, num_clips=clips, frames=frames, seed=seed)


def batch_env(backend, n, robot="smpl_humanoid", v=2, env="speed", seed=0, **kw):
    cfg = make_cfg(env=env, robot=robot, overrides={"env.self_obs_v": v, "robot.create_vel_sensors": v == 2})
    return backend.batch(cfg, n, seed=seed, **kw)


def im_env(backend, n, robot="smpl_humanoid", seed=0, clips=6, frames=14):
    cfg = make_cfg(env="im", robot=robot)
    return HumanoidImB200(cfg, lambda b: tables_for(b, clips, frames), num_envs=n, seed=seed, batch_factory=backend.batch)


def sim_frame(b, amp, upright):
    """The restated frame of every env from the batch's post-step tensors."""
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    xp, xq, qp, qv = f64(b.xpos), f64(b.xquat), f64(b.qpos), f64(b.qvel)
    keys = amp._keys
    return amp_frame(xp[:, 0], xq[:, 0], qv[:, :3], qrot(xq[:, 0], qv[:, 3:6]), qp[:, 7:], qv[:, 6:], xp[:, keys], upright,
                     amp.cfg["local_root_obs"], amp.cfg["root_height_obs"]), near_threshold(qp[:, 7:])


def ref_frame(lib, ids, times, amp_cfg, upright):
    """The restated frame of clip ids[i] at times[i] from the table rows the gather picks (the frame rule is held to the gather in
    test_imitation.py)."""
    ids_t = torch.as_tensor(np.asarray(ids), dtype=torch.int32, device=lib.env.device)
    t_t = torch.as_tensor(np.asarray(times), dtype=torch.float32, device=lib.env.device)
    s = lib.get_motion_state_intervaled(ids_t, t_t)
    f64 = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    xp, xq = f64(s["xpos"]), f64(s["xquat"])
    keys = amp_c_cfg(lib.env.model, amp_cfg)[1]
    return amp_frame(xp[:, 0], xq[:, 0], f64(s["root_vel"]), f64(s["root_ang_vel"]), f64(s["dof_pos"]), f64(s["dof_vel"]), xp[:, keys],
                     upright, amp_cfg["local_root_obs"], amp_cfg["root_height_obs"]), near_threshold(f64(s["dof_pos"]))


def close(got, want, skip=None):
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want).max(axis=-1, keepdims=True))
    if skip is not None:
        err = err[~skip]
    assert err.max() < TOL, err.max()


def fma32(k, dt, t0):
    return np.float32(np.float64(np.float32(k)) * np.float64(np.float32(dt)) + np.float64(np.float32(t0)))


def actions(env, backend, rng, sigma=0.5):
    return backend.t(np.clip(rng.normal(size=(env.num_envs, env.num_actions)) * sigma, -1, 1))


@pytest.mark.parametrize("robot,v,shapes,selfcol", [("smpl_humanoid", 2, False, False), ("smpl_humanoid", 1, False, False),
                                                     ("smplx_humanoid", 2, False, False), ("smpl_humanoid", 2, True, False),
                                                     ("smpl_humanoid", 2, False, True)])
def test_push_and_fill_match_restatement(backend, robot, v, shapes, selfcol):
    n = 16 if robot == "smpl_humanoid" else 8
    kw = {}
    if shapes:      # a second body shape: longer limbs, heavier bodies (same tree, joints and geom layout)
        import dataclasses
        from smplsim_b200.abi import model_from_cfg
        m0 = model_from_cfg(make_cfg(env="speed", robot=robot))
        m1 = dataclasses.replace(m0, body_pos=m0.body_pos * 1.08, body_mass=m0.body_mass * 1.2, body_inertia=m0.body_inertia * 1.2)
        kw = dict(models=[m0, m1], env_model=[i % 2 for i in range(n)])
    if selfcol:
        b = backend.batch(make_cfg(env="speed", robot=robot, overrides={"env.self_collision": True}), n, seed=0)
    else:
        b = batch_env(backend, n, robot=robot, v=v, **kw)
    amp = HumanoidAmpB200(b, amp_cfg=dict(num_amp_obs_steps=4))
    K, F = 4, amp.amp_frame_dim
    assert F == (232 if robot == "smpl_humanoid" else 484) and amp.amp_obs.shape == (n, K * F)
    up = bool(b.cfg.robot.has_upright_start)
    amp.reset()
    want, skip = sim_frame(b, amp, up)
    got = amp.amp_obs_buf.cpu().numpy()
    for k in range(K):
        close(got[:, k], want, skip)
        assert np.array_equal(got[:, k], got[:, 0])
    rng = np.random.default_rng(1)
    hist = [got[:, 0].copy()]
    for step in range(5):
        amp.step(actions(b, backend, rng))
        want, skip = sim_frame(b, amp, up)
        got = amp.amp_obs_buf.cpu().numpy()
        close(got[:, 0], want, skip)
        hist.insert(0, got[:, 0].copy())
        for k in range(1, K):       # frame k is frame 0 of k steps ago, bit for bit (the oldest fill repeats)
            assert np.array_equal(got[:, k], hist[min(k, len(hist) - 1)])


def test_masked_rows_are_untouched(backend):
    n = 16
    b = batch_env(backend, n)
    amp = HumanoidAmpB200(b, amp_cfg=dict(num_amp_obs_steps=3))
    amp.reset()
    rng = np.random.default_rng(2)
    amp.step(actions(b, backend, rng))
    before = amp.amp_obs_buf.clone()
    mask = torch.zeros(n, dtype=torch.uint8, device=b.device)
    mask[[0, 3, 9]] = 1
    amp.reset(mask)
    o = ~mask.bool()
    assert torch.equal(amp.amp_obs_buf[o], before[o])
    m = mask.bool()
    assert torch.equal(amp.amp_obs_buf[m][:, 1], amp.amp_obs_buf[m][:, 0]) and not torch.equal(amp.amp_obs_buf[m], before[m])
    # PUSH through the C call with a mask: only those rows move
    from smplsim_b200.abi import AMP_PUSH
    before = amp.amp_obs_buf.clone()
    amp._amp(mask, AMP_PUSH)
    assert torch.equal(amp.amp_obs_buf[o], before[o]) and torch.equal(amp.amp_obs_buf[m][:, 1:], before[m][:, :-1])
    # index-tensor reset
    before = amp.amp_obs_buf.clone()
    amp.reset(torch.tensor([5], device=b.device))
    assert torch.equal(amp.amp_obs_buf[:5], before[:5]) and torch.equal(amp.amp_obs_buf[6:], before[6:])


@pytest.mark.parametrize("robot", ["smpl_humanoid", "smplx_humanoid"])
def test_fill_ref_and_demo_match_restatement(backend, robot):
    n = 8
    env = im_env(backend, n, robot=robot)
    amp = HumanoidAmpB200(env)
    K, F, lib, dt = amp.num_amp_obs_steps, amp.amp_frame_dim, env.lib, env.dt
    up = bool(env.cfg.robot.has_upright_start)
    ids = backend.t(np.arange(n) % lib.num_motions(), torch.int32)
    t0 = backend.t(np.array([0.0, 0.05, 0.1, 0.2, 0.31, 0.4, 0.02, 0.43]))      # several start inside the history span: clamped at 0
    amp.reset(None, motion_ids=ids, motion_times=t0)
    got = amp.amp_obs_buf.cpu().numpy()
    want0, skip0 = sim_frame(env.batch, amp, up)
    close(got[:, 0], want0, skip0)
    idn, tn = ids.cpu().numpy(), t0.cpu().numpy()
    for k in range(1, K):
        times = [fma32(-k, dt, x) for x in tn]
        want, skip = ref_frame(lib, idn, times, amp.cfg, up)
        close(got[:, k], want, skip)
    # DEMO: explicit rows, including times before a clip's start and past its end
    L = float(lib._motion_lengths[0])
    times = np.array([0.0, 0.01, L, L + 0.5, -0.2, L / 2, 0.3, 0.12], dtype=np.float32)
    demo = lib.amp_obs_demo(motion_ids=ids, motion_times=backend.t(times)).cpu().numpy()
    assert demo.shape == (n, K, F)
    for k in range(K):
        want, skip = ref_frame(lib, idn, [fma32(-k, dt, x) for x in times], amp.cfg, up)
        close(demo[:, k], want, skip)
    # the same rows into a caller buffer: bit-identical, and sampled rows stay on their clip
    out = torch.zeros(n, K, F, device=env.device)
    r = lib.amp_obs_demo(motion_ids=ids, motion_times=backend.t(times), out=out)
    assert r is out and np.array_equal(out.cpu().numpy(), demo)
    s = lib.amp_obs_demo(32)
    assert s.shape == (32, K, F) and torch.isfinite(s).all()


def test_amp_calls_leave_the_stepper_alone(backend):
    n = 8
    plain = batch_env(backend, n)
    b = batch_env(backend, n)
    amp = HumanoidAmpB200(b)
    plain.reset(); amp.reset()
    rng = np.random.default_rng(3)
    for _ in range(3):
        a = actions(b, backend, rng)
        plain.step(a); amp.step(a)
        for k in ("qpos", "qvel", "obs_buf", "rew_buf", "terminate_buf", "truncate_buf", "xpos", "xquat"):
            assert torch.equal(getattr(plain, k), getattr(b, k)), k
        assert torch.equal(amp.rew_buf, plain.rew_buf) and torch.equal(amp.obs_buf, plain.obs_buf)


def run_fixed(backend, n, steps):
    env = im_env(backend, n, clips=8, frames=12, seed=4)
    env.lib._gen.manual_seed(11)
    amp = HumanoidAmpB200(env)
    amp.reset()
    rng = np.random.default_rng(4)
    out = []
    for _ in range(steps):
        amp.step(actions(env, backend, rng))
        out.append(amp.amp_obs.clone())
        amp.reset_done()
        out.append(amp.amp_obs.clone())
    out.append(env.lib.amp_obs_demo(16).reshape(16, -1))
    return torch.cat(out)


def test_two_runs_are_bit_identical(backend):
    assert torch.equal(run_fixed(backend, 8, 12), run_fixed(backend, 8, 12))


def test_bad_arguments_are_refused(backend):
    n = 4
    b = batch_env(backend, n)
    with pytest.raises(ValueError, match="unknown key body"):
        HumanoidAmpB200(b, amp_cfg=dict(key_bodies=["Tail"]))
    with pytest.raises(ValueError, match="unknown AMP key"):
        HumanoidAmpB200(b, amp_cfg=dict(num_steps=3))
    with pytest.raises(_lib.SmplsimError, match="key body out of range"):
        HumanoidAmpB200(b, amp_cfg=dict(key_bodies=[0, 24]))
    with pytest.raises(_lib.SmplsimError, match="num_steps"):
        HumanoidAmpB200(b, amp_cfg=dict(num_amp_obs_steps=0))
    env = im_env(backend, n)
    amp = HumanoidAmpB200(env)
    eb, L = env.batch, env.batch._L()
    from smplsim_b200.abi import SmplsimAmpTablesC, SmplsimMotionTablesC
    from smplsim_b200.batched import _ptr

    def obs(cfg=amp._ccfg, tab=amp._tab, mode=2, ids=env.motion_ids, out=amp.amp_obs_buf):
        return L.smplsim_amp_obs(eb._h, ctypes.byref(cfg) if cfg is not None else None, ctypes.byref(eb._state), ctypes.byref(eb._aux),
                                 ctypes.byref(tab) if tab is not None else None, _ptr(ids), _ptr(env.motion_start_times), None, mode, _ptr(out),
                                 eb._stream())

    def variant(struct, **kw):
        c = type(struct)()
        ctypes.memmove(ctypes.byref(c), ctypes.byref(struct), ctypes.sizeof(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    assert obs() == 0 and obs(mode=0) == 0 and obs(mode=1, tab=None, ids=None) == 0
    mt = SmplsimMotionTablesC.from_address(amp._tab.motion)
    mt52, mt0 = variant(mt, nbody=52), variant(mt, num_motions=0)      # named: the structs must outlive the calls that point at them
    for kw in (dict(cfg=None), dict(mode=3), dict(mode=-1), dict(out=None), dict(tab=None), dict(ids=None),
               dict(cfg=variant(amp._ccfg, num_steps=0)), dict(cfg=variant(amp._ccfg, num_key_bodies=25)),
               dict(cfg=variant(amp._ccfg, key_bodies=None)),
               dict(tab=variant(amp._tab, dof_vel=None)),
               dict(tab=SmplsimAmpTablesC(motion=ctypes.addressof(mt52), dof_pos=amp._tab.dof_pos, dof_vel=amp._tab.dof_vel)),
               dict(tab=SmplsimAmpTablesC(motion=ctypes.addressof(mt0), dof_pos=amp._tab.dof_pos, dof_vel=amp._tab.dof_vel))):
        assert obs(**kw) == -1, kw
        assert b"smplsim_amp_obs" in L.smplsim_last_error()
    bad = np.array([0, -1], dtype=np.int32)
    assert obs(cfg=variant(amp._ccfg, key_bodies=bad.ctypes.data, num_key_bodies=2)) == -1
    d = lambda **kw: L.smplsim_amp_demo(eb._h, ctypes.byref(kw.get("cfg", amp._ccfg)), ctypes.byref(kw["tab"]) if kw.get("tab") else None,  # noqa: E731
                                        _ptr(env.motion_ids), _ptr(env.motion_start_times), kw.get("n", n), _ptr(amp.amp_obs_buf), eb._stream())
    assert d(tab=amp._tab) == 0 and d(tab=amp._tab, n=0) == 0 and d(tab=None) == -1 and d(tab=amp._tab, n=-1) == -1
    assert d(tab=amp._tab, cfg=variant(amp._ccfg, num_steps=0)) == -1
    assert L.smplsim_amp_obs_dim(eb._h, ctypes.byref(amp._ccfg)) == 232
    assert L.smplsim_amp_obs_dim(eb._h, ctypes.byref(variant(amp._ccfg, root_height_obs=0, num_key_bodies=0))) == 219


def test_abi_structs_and_version():
    from smplsim_b200.abi import SmplsimAmpCfgC, SmplsimAmpTablesC
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "smplsim.h"\nint main(){printf("%zu %zu %zu %zu %zu %d %d %d\\n", '
           'sizeof(SmplsimAmpCfg), sizeof(SmplsimAmpTables), offsetof(SmplsimAmpCfg, key_bodies), offsetof(SmplsimAmpCfg, root_height_obs), '
           'offsetof(SmplsimAmpTables, dof_vel), SMPLSIM_AMP_PUSH, SMPLSIM_AMP_FILL, SMPLSIM_AMP_FILL_REF);return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        sizes = list(map(int, subprocess.check_output([os.path.join(d, "t")]).split()))
    from smplsim_b200.abi import AMP_FILL, AMP_FILL_REF, AMP_PUSH
    assert sizes == [ctypes.sizeof(SmplsimAmpCfgC), ctypes.sizeof(SmplsimAmpTablesC), SmplsimAmpCfgC.key_bodies.offset,
                     SmplsimAmpCfgC.root_height_obs.offset, SmplsimAmpTablesC.dof_vel.offset, AMP_PUSH, AMP_FILL, AMP_FILL_REF]
    L = ctypes.CDLL(_lib.build())
    L.smplsim_version.restype = ctypes.c_int
    assert L.smplsim_version() >= 280
    assert AMP_DEFAULTS["num_amp_obs_steps"] == 10 and AMP_DEFAULTS["key_bodies"] == KEYS and AMP_DEFAULTS["disc_units"] == [1024, 512]
    assert (AMP_DEFAULTS["task_reward_w"], AMP_DEFAULTS["disc_reward_w"], AMP_DEFAULTS["disc_reward_scale"]) == (0.5, 0.5, 2.0)


# ------------------------------------------------------------------ discriminator and learner (CPU)
def tiny_disc(dim=5, seed=0):
    torch.manual_seed(seed)
    return AMPDiscriminator(dim, units=(4, 3), activation="relu", normalize=False).double()


def test_reward_and_loss_terms_against_hand_written_autograd():
    d = tiny_disc()
    g = torch.Generator().manual_seed(1)
    agent = torch.randn(7, 5, generator=g, dtype=torch.float64)
    demo = torch.randn(6, 5, generator=g, dtype=torch.float64) + 0.5
    W = [(l.weight, l.bias) for l in d.mlp.affine_layers] + [(d.logits.weight, d.logits.bias)]

    def D(x):
        for w, b in W[:-1]:
            x = torch.relu(x @ w.T + b)
        return x @ W[-1][0].T + W[-1][1]

    la = D(agent)
    # reward: -log(max(1 - sigmoid(l), 1e-4)) * scale, with the clamp active for a large logit
    x = torch.cat([agent, agent[:1] * 40])
    lx = D(x).squeeze(-1)
    want_r = -torch.log(torch.clamp(1 - 1 / (1 + torch.exp(-lx)), min=1e-4)) * 2.0
    assert torch.allclose(d.reward(x, 2.0), want_r, atol=1e-12, rtol=0)
    terms = disc_loss_terms(d, agent, demo)
    demo_in = demo.clone().requires_grad_(True)
    ld = D(demo_in)
    bce = lambda l, y: torch.mean(-(y * torch.log(torch.sigmoid(l)) + (1 - y) * torch.log(1 - torch.sigmoid(l))))  # noqa: E731
    want_loss = 0.5 * (bce(la, 0.0) + bce(ld, 1.0))
    gd = torch.autograd.grad(ld.sum(), demo_in, create_graph=True)[0]
    want_gp = (gd ** 2).sum(-1).mean()
    want_lr = (W[-1][0] ** 2).sum()
    want_wd = sum((w ** 2).sum() for w, _ in W)
    for k, want in (("loss", want_loss), ("grad_penalty", want_gp), ("logit_reg", want_lr), ("weight_decay", want_wd)):
        assert torch.allclose(terms[k], want, atol=1e-12, rtol=1e-10), k
    c = dict(AMP_DEFAULTS)
    total = disc_total_loss(terms, c)
    want_total = 5.0 * (want_loss + 0.01 * want_lr + 5.0 * want_gp + 1e-4 * want_wd)
    assert torch.allclose(total, want_total, atol=1e-12, rtol=1e-10)
    # the gradient of the total (the penalty's double backward included) equals the hand-written one
    ga = torch.autograd.grad(total, [p for p in d.parameters()], retain_graph=True)
    gw = torch.autograd.grad(want_total, [p for p in d.parameters()])
    assert all(torch.allclose(a, b, atol=1e-12, rtol=1e-9) for a, b in zip(ga, gw))
    assert float(terms["agent_acc"]) == float((la < 0).double().mean()) and float(terms["demo_acc"]) == float((ld > 0).double().mean())


def test_normalisation_uses_merged_moments_and_never_syncs_in_forward():
    d = AMPDiscriminator(3, units=(4,), normalize=True).double()
    x = torch.randn(10, 3, dtype=torch.float64)
    assert torch.equal(d.normalize(x), x)           # no moments yet: identity
    d.update_norm(x)
    want = ((x - x.mean(0)) / (x.var(0, unbiased=False).sqrt() + 1e-8)).clamp(-5, 5)
    assert torch.allclose(d.normalize(x), want, atol=1e-12)
    d.train()
    y = d(x)
    assert int(d.norm.n) == 10 and y.shape == (10, 1)   # a training-mode forward does not move the moments


def test_replay_buffer_keep_probability_bookkeeping():
    g = torch.Generator().manual_seed(0)
    r = AMPReplayBuffer(100, 2, 0.25, "cpu", g)
    r.store(torch.arange(60.0).view(30, 2))
    assert (r.count, r.total, r.head) == (30, 30, 30)
    r.store(torch.zeros(90, 2) + 7)                     # total 30 <= 100 when it arrives: every row kept, 90 > 100 - 30 so it wraps
    assert (r.count, r.total, r.head) == (100, 120, 20)
    r.store(torch.ones(250, 2))                         # more than a buffer's worth seen: about a quarter kept
    assert 40 <= r.total - 120 <= 85 and r.count == 100
    before = r.total
    r.store(torch.ones(4000, 2) * 3)                    # kept rows beyond the buffer size: a random `size` of them
    assert r.total - before == 100 and r.count == 100
    assert r.sample(17).shape == (17, 2)


def test_learner_update_runs_on_cpu_and_separates():
    torch.manual_seed(0)
    d = AMPDiscriminator(4, units=(32, 16), normalize=True)
    g = torch.Generator().manual_seed(0)
    learner = AMPLearner(d, lambda n: torch.randn(n, 4, generator=g) + 3.0, dict(amp_minibatch_size=64, lr=1e-3, amp_replay_buffer_size=512), g)
    info = None
    for _ in range(30):
        info = learner.update(torch.randn(256, 4, generator=g))
    assert info["disc_agent_acc"] > 0.9 and info["disc_demo_acc"] > 0.9 and learner.replay.total > 0


def _dist_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)
    d = AMPDiscriminator(3, units=(4,), normalize=False).double()
    p0 = [p.detach().clone() for p in d.parameters()]
    agent = torch.full((8, 3), float(rank + 1), dtype=torch.float64)
    demo = lambda n: torch.full((n, 3), -float(rank + 1), dtype=torch.float64)  # noqa: E731
    learner = AMPLearner(d, demo, dict(amp_minibatch_size=8, lr=0.0))
    captured = {}
    orig = learner.optimizer.step

    def step(*a, **k):
        captured["g"] = [p.grad.detach().clone() for p in d.parameters()]
        return orig(*a, **k)

    learner.optimizer.step = step
    learner.update(agent)
    # this rank's own gradient, without the average
    own = AMPDiscriminator(3, units=(4,), normalize=False).double()
    with torch.no_grad():
        for p, v in zip(own.parameters(), p0):
            p.copy_(v)
    t = disc_total_loss(disc_loss_terms(own, agent, demo(8)), learner.cfg)
    og = torch.autograd.grad(t, list(own.parameters()))
    q.put((rank, [x.numpy() for x in captured["g"]], [x.numpy() for x in og]))
    dist.destroy_process_group()


def test_discriminator_gradients_are_averaged_over_ranks():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_dist_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = dict((r, (g, o)) for r, g, o in (q.get(timeout=120) for _ in ps))
    for p in ps:
        p.join(timeout=60)
    for i in range(len(res[0][0])):
        mean = 0.5 * (res[0][1][i] + res[1][1][i])
        assert np.allclose(res[0][0][i], mean, atol=1e-12) and np.allclose(res[1][0][i], mean, atol=1e-12)
    assert not np.allclose(res[0][1][0], res[1][1][0])


# ------------------------------------------------------------------ the wrapper with a discriminator (GPU)
@pytest.mark.gpu
def test_reward_mix_and_protocol_on_gpu():
    from conftest import Backend
    backend = Backend("gpu")
    n = 64
    env = im_env(backend, n)
    amp = HumanoidAmpB200(env)
    amp.make_learner()
    from smplsim_b200.batched import GymVectEnvB200
    from smplsim_b200.learning import BatchedSampler
    amp.reset()
    rng = np.random.default_rng(0)
    for _ in range(3):
        amp.step(actions(env, backend, rng))
        c = amp.cfg
        task, disc = amp.extras["task_rew_buf"], amp.extras["disc_rew_buf"]
        assert task is env.rew_buf
        assert torch.equal(amp.rew_buf, task * c["task_reward_w"] + disc * c["disc_reward_w"])
        assert torch.equal(disc, amp.discriminator.reward(amp.amp_obs, c["disc_reward_scale"]))
        amp.reset_done()
    assert amp.drain_amp_obs().shape == (3, n, amp.num_amp_obs) and amp.drain_amp_obs().shape[0] == 0
    venv = GymVectEnvB200(amp)
    obs, _ = venv.reset()
    obs, rew, term, trunc, info = venv.step(actions(env, backend, rng))
    assert obs.shape == (n, amp.num_obs) and torch.isfinite(rew).all()
    gen = torch.Generator(device=env.device); gen.manual_seed(0)
    batch = BatchedSampler(amp, lambda o: 0.3 * torch.randn(n, amp.num_actions, generator=gen, device=env.device)).sample(8)
    assert batch["rewards"].shape == (8, n) and torch.isfinite(batch["rewards"]).all()


AMP_SEPARATION_UPDATES = 20


@pytest.mark.gpu
def test_discriminator_separates_random_actions_from_demo_rows():
    """256 speed envs under random actions: within AMP_SEPARATION_UPDATES discriminator updates (one 16-step rollout each, default
    hyper-parameters except the learning rate 1e-4 and minibatches of 1024 rows) the accuracy on agent and demo rows passes 0.9."""
    from conftest import Backend
    backend = Backend("gpu")
    n = 256
    b = batch_env(backend, n)
    lib = MotionLibB200(b, tables_for(b, clips=16, frames=120))
    amp = HumanoidAmpB200(b, lib)
    g = torch.Generator(device=b.device); g.manual_seed(0)
    torch.manual_seed(0)
    learner = amp.make_learner(generator=g)
    learner.cfg["amp_minibatch_size"] = 1024
    for grp in learner.optimizer.param_groups:
        grp["lr"] = 1e-4
    rng = np.random.default_rng(0)
    amp.reset()
    info = {}
    for _ in range(AMP_SEPARATION_UPDATES):
        for _ in range(16):
            amp.step(actions(b, backend, rng, 1.0))
            amp.reset_done()
        info = learner.update(amp.drain_amp_obs())
        if info["disc_agent_acc"] > 0.9 and info["disc_demo_acc"] > 0.9:
            break
    assert info["disc_agent_acc"] > 0.9 and info["disc_demo_acc"] > 0.9, info
