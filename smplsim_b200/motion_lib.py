"""Reference-pose feed (SURVEY.md 8 a12): device-resident motion tables + ``get_motion_state_intervaled``.

Replaces ``MotionLibBase.get_motion_state_intervaled`` / ``_calc_frame_blend`` (smpl_sim/smpllib/motion_lib_base.py:313-354,
448-458): the flat per-frame tables (``gts, grs, gvs, gavs, dof_pos, dvs, qpos, qvel`` + ``length_starts``, built in
``load_motions`` :173-198) live on the GPU and one CUDA kernel does the nearest-frame gather for all envs.  The AMASS
loader itself (SMPL pkl files, ``smplx``) is a "next" row (f3); ``synthetic_tables`` builds the BASELINE config-4 stand-in
(K clips x F frames of sinusoidal joint angles, tables from this repo's own FK with finite-difference + gaussian velocities,
following smpl_sim/smpllib/torch_smpl_humanoid_batch.py:118-228).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from .abi import SmplsimAmpTablesC, SmplsimMotionTablesC
from .batched import HumanoidBatchB200

TABLE_KEYS = ("qpos", "qvel", "xpos", "xquat", "body_vel", "body_ang_vel", "dof_pos", "dof_vel")
OPTIONAL_KEYS = ("motion_aa",)
# value kind of each table in get_motion_state / blend_into (abi.BLEND_*: 0 LERP, 1 POS, 2 SLERP, 3 QPOS, 4 ROW0); the rest are LERP
BLEND_KINDS = {"xpos": 1, "xquat": 2, "qpos": 3, "motion_aa": 4}          # per-frame axis-angle pose of the source clip (motion_lib_base.py:340-354 returns it)


def _gauss1d(x, sigma):
    from scipy.ndimage import gaussian_filter1d
    return gaussian_filter1d(x, sigma, axis=0, mode="nearest")


def synthetic_tables(env: HumanoidBatchB200, num_clips: int = 64, frames: int = 300, fps: float = 30.0, seed: int = 4) -> Dict[str, np.ndarray]:
    """Config-4 synthetic clip tables (SURVEY.md 8d): 3 sinusoids per joint, root on a 1 m/s straight path at fixed height."""
    m = env.model
    rng = np.random.default_rng(seed)
    K, F, nu = num_clips, frames, m.nu
    t = np.arange(F) / fps
    amp = rng.uniform(0, 0.4, (K, 3, nu))
    frq = rng.uniform(0.2, 1.5, (K, 3, nu))
    ph = rng.uniform(0, 2 * np.pi, (K, 3, nu))
    dof = (amp[:, :, None, :] * np.sin(2 * np.pi * frq[:, :, None, :] * t[None, None, :, None] + ph[:, :, None, :])).sum(1) / 3.0   # [K,F,nu]
    qpos = np.zeros((K, F, m.nq))
    qpos[..., 0] = t[None, :] * 1.0
    qpos[..., 2] = 0.94
    qpos[..., 3:7] = 0.5
    qpos[..., 7:] = dof
    flat_q = qpos.reshape(K * F, m.nq)
    xpos, xquat = env.kinematics(torch.as_tensor(flat_q, dtype=torch.float32))
    xpos = xpos.cpu().numpy().reshape(K, F, m.nbody, 3)
    xquat = xquat.cpu().numpy().reshape(K, F, m.nbody, 4)
    dt = 1.0 / fps
    body_vel = np.stack([_gauss1d(np.gradient(xpos[k], dt, axis=0), 2) for k in range(K)])
    dof_vel = np.stack([_gauss1d(np.gradient(dof[k], dt, axis=0), 2) for k in range(K)])
    # angular velocity from consecutive quaternions (world frame), gaussian filtered
    def qmul(a, b):
        w1, x1, y1, z1 = np.moveaxis(a, -1, 0); w2, x2, y2, z2 = np.moveaxis(b, -1, 0)
        return np.stack([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                         w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2], -1)
    qn = np.concatenate([xquat[:, 1:], xquat[:, -1:]], 1)
    qc = xquat * np.array([1, -1, -1, -1.0])
    dq = qmul(qn, qc)
    dq *= np.sign(dq[..., :1] + 1e-12)
    ang = 2 * np.arctan2(np.linalg.norm(dq[..., 1:], axis=-1), dq[..., 0])
    ax = dq[..., 1:] / np.maximum(np.linalg.norm(dq[..., 1:], axis=-1, keepdims=True), 1e-9)
    body_ang_vel = np.stack([_gauss1d((ax * ang[..., None] / dt)[k], 2) for k in range(K)])
    qvel = np.zeros((K, F, m.nv))
    qvel[..., 0:3] = body_vel[:, :, 0]
    qvel[..., 3:6] = body_ang_vel[:, :, 0]
    qvel[..., 6:] = dof_vel
    f32 = lambda a: np.ascontiguousarray(a.reshape(K * F, -1), dtype=np.float32)  # noqa: E731
    return dict(qpos=f32(qpos), qvel=f32(qvel), xpos=f32(xpos), xquat=f32(xquat), body_vel=f32(body_vel), body_ang_vel=f32(body_ang_vel),
                dof_pos=f32(dof), dof_vel=f32(dof_vel), motion_num_frames=np.full(K, F, np.int32), motion_dt=np.full(K, dt, np.float32),
                motion_lengths=np.full(K, dt * (F - 1), np.float32), length_starts=(np.arange(K) * F).astype(np.int32),
                motion_aa=np.zeros((K * F, 3 * m.nbody), np.float32), motion_bodies=np.zeros((K, 17), np.float32),
                motion_fps=np.full(K, fps, np.float32), motion_keys=np.array([f"synthetic_{k:03d}" for k in range(K)]))


class MotionLibB200:
    """GPU-resident motion tables with the reference's query API."""

    def __init__(self, env: HumanoidBatchB200, tables: Dict[str, np.ndarray]):
        self.env = env
        dv = env.device
        self.tables = {k: torch.as_tensor(tables[k], dtype=torch.float32, device=dv).contiguous() for k in TABLE_KEYS}
        self._motion_num_frames = torch.as_tensor(tables["motion_num_frames"], dtype=torch.int32, device=dv)
        self._motion_dt = torch.as_tensor(tables["motion_dt"], dtype=torch.float32, device=dv)
        self._motion_lengths = torch.as_tensor(tables["motion_lengths"], dtype=torch.float32, device=dv)
        self.length_starts = torch.as_tensor(tables["length_starts"], dtype=torch.int32, device=dv)
        self._keys = TABLE_KEYS + tuple(k for k in OPTIONAL_KEYS if k in tables)
        for k in self._keys[len(TABLE_KEYS):]:
            self.tables[k] = torch.as_tensor(tables[k], dtype=torch.float32, device=dv).contiguous()
        self._ptrs = {}          # tuple of table keys -> (table pointers, widths) of gather_into
        K = int(self._motion_lengths.shape[0])
        # per-motion shape parameters (motion_lib_base.py:_motion_bodies, 17 = 16 betas + gender) and library bookkeeping
        self._motion_bodies = torch.as_tensor(tables["motion_bodies"], dtype=torch.float32, device=dv) if "motion_bodies" in tables else torch.zeros(K, 17, device=dv)
        self._motion_fps = torch.as_tensor(tables["motion_fps"], dtype=torch.float32, device=dv) if "motion_fps" in tables else 1.0 / self._motion_dt
        self._motion_data_keys = np.asarray(tables["motion_keys"]) if "motion_keys" in tables else np.array([f"clip_{i:04d}" for i in range(K)])
        self._num_unique_motions = K
        # sampling weights (PMCP), motion_lib_base.py:102-116,231-270: uniform until evaluation reports failed sequences
        self._sampling_prob = torch.full((K,), 1.0 / K, dtype=torch.float64, device=dv)
        self._sampling_batch_prob = self._sampling_prob.clone()
        self._termination_history = torch.zeros(K, dtype=torch.float64, device=dv)
        self.curr_failed_keys = []
        self._gen = torch.Generator(device=dv)
        self._gen.manual_seed(int(getattr(env, "seed", 0)) & 0x7FFFFFFF)
        # the tables as the imitation, evaluation and AMP entry points take them; they point into the tensors above
        t = self.tables
        self.c_tables = SmplsimMotionTablesC(
            xpos=t["xpos"].data_ptr(), xquat=t["xquat"].data_ptr(), body_vel=t["body_vel"].data_ptr(), body_ang_vel=t["body_ang_vel"].data_ptr(),
            motion_len=self._motion_lengths.data_ptr(), num_frames=self._motion_num_frames.data_ptr(), motion_dt=self._motion_dt.data_ptr(),
            length_starts=self.length_starts.data_ptr(), num_motions=K, nbody=t["xpos"].shape[1] // 3)

    def num_motions(self):
        return int(self._motion_lengths.shape[0])

    def get_motion_length(self, motion_ids=None):
        return self._motion_lengths if motion_ids is None else self._motion_lengths[motion_ids.long()]

    def get_motion_state_intervaled(self, motion_ids: torch.Tensor, motion_times: torch.Tensor, offset=None):
        dv = self.env.device
        ids = motion_ids.to(dv, torch.int32).contiguous()
        tm = motion_times.to(dv, torch.float32).contiguous()
        n = ids.shape[0]
        outs = {k: torch.empty(n, self.tables[k].shape[1], dtype=torch.float32, device=dv) for k in self._keys}
        frame = torch.empty(n, dtype=torch.int32, device=dv)
        self.gather_into(self._keys, ids, tm, [outs[k] for k in self._keys], frame)
        nb = self.env.model.nbody
        xpos = outs["xpos"].view(n, nb, 3)
        if offset is not None:
            xpos = xpos + offset[:, None, :]
        xquat, bv, bav = outs["xquat"].view(n, nb, 4), outs["body_vel"].view(n, nb, 3), outs["body_ang_vel"].view(n, nb, 3)
        return dict(root_pos=xpos[:, 0], root_rot=xquat[:, 0], dof_pos=outs["dof_pos"], root_vel=bv[:, 0], root_ang_vel=bav[:, 0],
                    dof_vel=outs["dof_vel"], xpos=xpos, xquat=xquat, body_vel=bv, body_ang_vel=bav, qpos=outs["qpos"], qvel=outs["qvel"],
                    motion_aa=outs.get("motion_aa"), motion_bodies=self._motion_bodies[ids.long()], frame_idx=frame)

    def gather_into(self, keys, motion_ids: torch.Tensor, motion_times: torch.Tensor, outs, frame_idx=None):
        """The frame gather of ``get_motion_state_intervaled`` for the tables ``keys`` only, into the caller's ``outs`` (one ``[n, width]``
        float32 tensor per key): nothing is allocated.  ``motion_ids`` int32 / ``motion_times`` float32, contiguous, on the env's device."""
        env, n = self.env, motion_ids.shape[0]
        keys = tuple(keys)
        if keys not in self._ptrs:
            self._ptrs[keys] = ((C.c_void_p * len(keys))(*[self.tables[k].data_ptr() for k in keys]),
                                (C.c_int32 * len(keys))(*[self.tables[k].shape[1] for k in keys]))
        tabs, widths = self._ptrs[keys]
        optr = (C.c_void_p * len(keys))(*[o.data_ptr() for o in outs])
        env._check(env._L().smplsim_motion_gather(env._h, motion_ids.data_ptr(), motion_times.data_ptr(), n, self._motion_lengths.data_ptr(),
                                                  self._motion_num_frames.data_ptr(), self._motion_dt.data_ptr(), self.length_starts.data_ptr(),
                                                  len(keys), tabs, widths, optr, None if frame_idx is None else frame_idx.data_ptr(),
                                                  env._stream()))
        env.gpu_launches += 1

    # ------------------------------------------------------------------ blended states (csrc/aux_kernels.cuh k_motion_blend)
    def get_motion_state(self, motion_ids: torch.Tensor, motion_times: torch.Tensor, offset=None):
        """``MotionLibBaseTorch.get_motion_state`` (motion_lib_base_torch.py:434-499): the state at ``motion_times`` blended from the two
        frames around it, positions / velocities / joint angles lerped, body rotations slerped (the reference's slerp, unnormalised).
        ``offset [n, 3]`` (or None) is added to every body position.  The reference's keys, plus ``qpos`` (root quaternion slerped,
        offset on the root position) and ``qvel`` (lerped), this project's extension, and ``frame_idx0`` / ``frame_idx1`` (table rows)
        and ``blend``.  One kernel launch."""
        dv = self.env.device
        ids = motion_ids.to(dv, torch.int32).contiguous()
        tm = motion_times.to(dv, torch.float32).contiguous()
        n = ids.shape[0]
        off = None if offset is None else torch.as_tensor(offset, dtype=torch.float32, device=dv).reshape(n, 3).contiguous()
        outs = {k: torch.empty(n, self.tables[k].shape[1], dtype=torch.float32, device=dv) for k in self._keys}
        f0, f1 = torch.empty(n, dtype=torch.int32, device=dv), torch.empty(n, dtype=torch.int32, device=dv)
        blend = torch.empty(n, dtype=torch.float32, device=dv)
        self.blend_into(self._keys, ids, tm, [outs[k] for k in self._keys], offset=off, frame_idx0=f0, frame_idx1=f1, blend=blend)
        nb = self.env.model.nbody
        xpos, xquat = outs["xpos"].view(n, nb, 3), outs["xquat"].view(n, nb, 4)
        bv, bav = outs["body_vel"].view(n, nb, 3), outs["body_ang_vel"].view(n, nb, 3)
        return dict(root_pos=xpos[:, 0], root_rot=xquat[:, 0], dof_pos=outs["dof_pos"], root_vel=bv[:, 0], root_ang_vel=bav[:, 0],
                    dof_vel=outs["dof_vel"], motion_aa=outs.get("motion_aa"), rg_pos=xpos, rb_rot=xquat, body_vel=bv, body_ang_vel=bav,
                    motion_bodies=self._motion_bodies[ids.long()], qpos=outs["qpos"], qvel=outs["qvel"], frame_idx0=f0, frame_idx1=f1,
                    blend=blend)

    def blend_into(self, keys, motion_ids: torch.Tensor, motion_times: torch.Tensor, outs, offset=None, kinds=None, frame_idx0=None,
                   frame_idx1=None, blend=None):
        """The blend of ``get_motion_state`` for the tables ``keys`` only, into the caller's ``outs`` (one ``[n, width]`` float32 tensor per
        key): nothing is allocated.  ``kinds``: one ``abi.BLEND_*`` per key (default ``BLEND_KINDS``: ``xpos`` POS, ``xquat`` SLERP,
        ``qpos`` QPOS, ``motion_aa`` ROW0, the rest LERP).  ``motion_ids`` int32 / ``motion_times`` float32 / ``offset`` float32 ``[n, 3]``,
        contiguous, on the env's device; ``frame_idx0`` / ``frame_idx1`` int32 and ``blend`` float32 ``[n]`` outputs, or None."""
        env, n = self.env, motion_ids.shape[0]
        keys = tuple(keys)
        kinds = tuple(BLEND_KINDS.get(k, 0) for k in keys) if kinds is None else tuple(int(x) for x in kinds)
        ck = ("blend", keys, kinds)
        if ck not in self._ptrs:
            self._ptrs[ck] = ((C.c_void_p * len(keys))(*[self.tables[k].data_ptr() for k in keys]),
                              (C.c_int32 * len(keys))(*[self.tables[k].shape[1] for k in keys]), (C.c_int32 * len(keys))(*kinds))
        tabs, widths, ckinds = self._ptrs[ck]
        optr = (C.c_void_p * len(keys))(*[o.data_ptr() for o in outs])
        p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        env._check(env._L().smplsim_motion_blend(env._h, motion_ids.data_ptr(), motion_times.data_ptr(), n, self._motion_lengths.data_ptr(),
                                                 self._motion_num_frames.data_ptr(), self._motion_dt.data_ptr(), self.length_starts.data_ptr(),
                                                 len(keys), tabs, widths, ckinds, p(offset), optr, p(frame_idx0), p(frame_idx1), p(blend),
                                                 env._stream()))
        env.gpu_launches += 1

    # ------------------------------------------------------------------ AMP demonstration rows (amp.py, csrc/amp_kernels.cuh)
    def set_amp_cfg(self, amp_cfg=None):
        """The AMP observation ``amp_obs_demo`` produces (keys of ``amp.AMP_DEFAULTS``; ``HumanoidAmpB200`` sets its own)."""
        from .amp import amp_c_cfg, amp_config
        self.amp_cfg = amp_config(amp_cfg)
        self._amp_ccfg, self._amp_keys = amp_c_cfg(self.env.model, self.amp_cfg)

    def _amp_tables(self):
        if getattr(self, "_amp_tab", None) is None:
            t = self.tables
            self._amp_tab = SmplsimAmpTablesC(motion=C.addressof(self.c_tables), dof_pos=t["dof_pos"].data_ptr(), dof_vel=t["dof_vel"].data_ptr())
        return self._amp_tab

    def amp_obs_demo(self, n=None, motion_ids=None, motion_times=None, out=None):
        """Demonstration AMP observations ``[n, K, F]``: row i holds frames ``t_i - k dt`` (k = 0..K-1, dt the env's control period) of
        clip ``motion_ids[i]``, the nearest-frame rows of the tables (blended states with the AMP key ``interpolate``).  Either ``n`` (clips from ``sample_motions``, times from
        ``sample_time(ids, truncate_time=(K-1) dt) + (K-1) dt``, so no frame lies before the clip's start) or ``motion_ids`` (int32) and
        ``motion_times`` (float32), ``[n]`` tensors on the env's device.  One kernel launch; nothing is allocated when ``out`` (float32,
        contiguous) is given along with ids and times of those dtypes."""
        if getattr(self, "amp_cfg", None) is None:
            self.set_amp_cfg()
        env, K = self.env, int(self.amp_cfg["num_amp_obs_steps"])
        if motion_ids is None:
            if n is None:
                raise ValueError("give n or motion_ids / motion_times")
            motion_ids = self.sample_motions(int(n))
            span = (K - 1) * env.dt
            motion_times = self.sample_time(motion_ids, truncate_time=span) + span
        elif motion_times is None:
            raise ValueError("motion_ids needs motion_times")
        ids = motion_ids.to(env.device, torch.int32).contiguous()
        tm = motion_times.to(env.device, torch.float32).contiguous()
        m = ids.shape[0]
        if tm.shape != (m,) or ids.dim() != 1:
            raise ValueError(f"motion_ids and motion_times must be [n] tensors of one length, got {tuple(ids.shape)} / {tuple(tm.shape)}")
        L = env._L()
        F = L.smplsim_amp_obs_dim(env._h, C.byref(self._amp_ccfg))
        if out is None:
            out = torch.empty(m, K, F, dtype=torch.float32, device=env.device)
        elif tuple(out.shape) != (m, K, F) or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous float32 tensor of shape {(m, K, F)}")
        env._check(L.smplsim_amp_demo(env._h, C.byref(self._amp_ccfg), C.byref(self._amp_tables()), ids.data_ptr(), tm.data_ptr(), m,
                                      out.data_ptr() if m else None, env._stream()))
        env.gpu_launches += 1
        return out

    def inverse_dynamics(self, contact_wrench: bool = False):
        """``env.inverse`` over every frame of the library: ``qfrc_inverse [total_frames, nv]`` (and ``contact_wrench [total_frames,
        nbody, 6]``), indexed like the tables.  ``qfrc_inverse[:, 0:6]`` is the root residual force of each frame.  ``qacc`` is the
        forward difference of ``qvel`` over the clip's ``motion_dt``; a clip's last frame repeats its previous difference (a one-frame clip
        gets zero), so nothing is differenced across clips."""
        return self.env.inverse(self.tables["qpos"], self.tables["qvel"], self._frame_qacc(), contact_wrench=contact_wrench)

    def _frame_qacc(self):
        """qacc of every frame: the forward difference of ``qvel`` over the clip's ``motion_dt``; a clip's last frame repeats its
        previous difference (a one-frame clip gets zero), so nothing is differenced across clips."""
        qvel = self.tables["qvel"]
        idx = torch.arange(qvel.shape[0], device=qvel.device)
        clip = torch.searchsorted(self.length_starts.long(), idx, right=True) - 1
        start, last = self.length_starts.long()[clip], (self.length_starts.long() + self._motion_num_frames.long() - 1)[clip]
        hi = torch.where(idx < last, idx + 1, idx)
        lo = torch.maximum(hi - 1, start)
        return (qvel[hi] - qvel[lo]) / self._motion_dt[clip][:, None]

    def rne_post(self, **kw):
        """``env.rne_post`` over every frame of the library, at the frames' ``qpos`` / ``qvel`` and the ``qacc`` that
        ``inverse_dynamics`` uses: body accelerations, joint reaction wrenches and IMU readings, indexed like the tables.  Keywords go to
        ``rne_post`` (``acc``, ``joint_wrench``, ``imu_sites``, ``xfrc_applied``)."""
        return self.env.rne_post(self.tables["qpos"], self.tables["qvel"], self._frame_qacc(), **kw)

    def centroidal(self, **kw):
        """``env.centroidal`` over every frame of the library: subtree centres of mass, their velocities, angular momenta, the
        centroidal momentum matrix and its bias, and COM Jacobians of the frames' ``qpos`` / ``qvel``, indexed like the tables.  Keywords
        go to ``centroidal`` (``com``, ``velocity``, ``cmm``, ``jac_com_bodies``)."""
        return self.env.centroidal(self.tables["qpos"], self.tables["qvel"], **kw)

    def render_clip(self, motion_id: int, camera="side", width: int = 320, height: int = 240, **kw):
        """``env.render`` of every frame of clip ``motion_id`` from the library's ``xpos`` / ``xquat`` tables: ``rgb [F, H, W, 3]``
        uint8 (F = the clip's frame count).  Further keywords go to ``render`` (``geom_rgb``).  Needs a one-shape batch."""
        K = self.num_motions()
        if not 0 <= int(motion_id) < K:
            raise ValueError(f"motion_id must be in [0, {K}), got {motion_id}")
        s = int(self.length_starts[int(motion_id)].item())
        f = int(self._motion_num_frames[int(motion_id)].item())
        nb = self.env.model.nbody
        xpos = self.tables["xpos"][s:s + f].view(f, nb, 3)
        xquat = self.tables["xquat"][s:s + f].view(f, nb, 4)
        return self.env.render(camera=camera, width=width, height=height, xpos=xpos, xquat=xquat, **kw)["rgb"]

    # ------------------------------------------------------------------ sampling (motion_lib_base.py:231-312), on the device
    def _uniform(self):
        K = self._num_unique_motions
        self._sampling_prob = torch.full((K,), 1.0 / K, dtype=torch.float64, device=self._sampling_prob.device)

    def _key_indexes(self, failed_keys):
        all_keys = self._motion_data_keys.tolist()
        return [all_keys.index(k) for k in failed_keys]

    def update_hard_sampling_weight(self, failed_keys):
        """Auto PMCP, hard: train only on the failed sequences (motion_lib_base.py:231-243)."""
        if len(failed_keys) > 0:
            idx = self._key_indexes(failed_keys)
            self._sampling_prob.zero_()
            self._sampling_prob[idx] = 1.0 / len(idx)
        else:
            self._uniform()
        self._sampling_batch_prob = self._sampling_prob / self._sampling_prob.sum()

    def update_soft_sampling_weight(self, failed_keys):
        """Auto PMCP, soft: weights proportional to the termination history (motion_lib_base.py:245-262)."""
        if len(failed_keys) > 0:
            self.curr_failed_keys = list(failed_keys)
            self._termination_history[self._key_indexes(failed_keys)] += 1
            self.update_sampling_prob(self._termination_history)
        else:
            self._uniform()
        self._sampling_batch_prob = self._sampling_prob / self._sampling_prob.sum()

    def update_sampling_prob(self, termination_history):
        th = torch.as_tensor(termination_history, dtype=torch.float64, device=self._sampling_prob.device)
        if th.numel() != self._sampling_prob.numel():
            return False
        self._sampling_prob = th / th.sum()
        self._termination_history = th.clone()
        self._sampling_batch_prob = self._sampling_prob.clone()
        return True

    def set_termination_history(self, termination_history):
        self._termination_history = torch.as_tensor(termination_history["termination_history"], dtype=torch.float64, device=self._sampling_prob.device)
        self.curr_failed_keys = termination_history["failed_keys"]
        self.update_sampling_prob(self._termination_history)

    def sample_motions(self, n: int = 1):
        """np.random.choice(p=_sampling_batch_prob, replace=True) of the reference (:272-274) as a device multinomial (its own
        Philox stream: distributional parity, the reference draws from the global numpy RNG)."""
        return torch.multinomial(self._sampling_batch_prob.float(), int(n), replacement=True, generator=self._gen).to(torch.int32)

    def sample_time(self, motion_ids, truncate_time=None):
        phase = torch.rand(motion_ids.shape, generator=self._gen, device=self._motion_lengths.device)
        motion_len = self._motion_lengths[motion_ids.long()].clone()
        if truncate_time is not None:
            assert truncate_time >= 0.0
            motion_len -= truncate_time
        return phase * motion_len

    def sample_time_interval(self, motion_ids, truncate_time=None):
        curr_fps = 1.0 / 30.0
        t = self.sample_time(motion_ids, truncate_time)
        return (t / curr_fps).long().float() * curr_fps

    def get_motion_num_steps(self, motion_ids=None):
        nf = self._motion_num_frames if motion_ids is None else self._motion_num_frames[motion_ids.long()]
        fps = self._motion_fps if motion_ids is None else self._motion_fps[motion_ids.long()]
        return (nf.float() * 30.0 / fps).to(torch.int32)
