"""Motion-imitation env on the batched tensor protocol: every env tracks one clip of a ``MotionLibB200``.

``HumanoidImB200`` owns a ``HumanoidBatchB200`` whose stepper runs without a task (self observation only) and adds the task with one
CUDA kernel per call (``smplsim_imitation``, csrc/imitation_kernels.cuh) that reads the library's tables in place: tracking
observation, reward, early termination, truncation at the clip's end and the mean per-joint position error.  The definitions are
stated in include/smplsim.h and DESIGN.md 2; the reference ships no imitation task in its MuJoCo env layer (SURVEY.md 3.4), they
follow the published PHC formulation.  Envs that finish are put back on a reference frame of a newly drawn clip (MoCap init)."""
from __future__ import annotations

import ctypes as C
from typing import Any, Callable, Optional, Sequence, Union

import numpy as np
import torch

from .abi import SmplsimImitationCfgC, SmplsimMotionTablesC
from .batched import HumanoidBatchB200, _ptr
from .motion_lib import MotionLibB200


class HumanoidImB200:
    """N SMPL humanoids, each tracking a motion-library clip.  The tensor protocol of ``HumanoidBatchB200`` (``num_envs, num_obs,
    num_actions, device, obs_buf, rew_buf, terminate_buf, truncate_buf, reset_buf, progress_buf, extras, step, reset, reset_done``), so
    ``GymVectEnvB200`` and ``BatchedSampler`` take it as they take a batch; plus ``motion_ids`` / ``motion_start_times`` (the clip and
    the clip time at which each env's episode started), ``mpjpe`` (metres, of the last step) and ``ref_frames`` (the two table rows the
    last call used: now, next).

    ``cfg``: ``make_cfg(env="im")`` (gains ``im_k_*``, weights ``im_w_*``, ``termination_distance``, ``tracked_bodies``, ``episode_length``).
    ``motion``: the library's tables (the dict ``synthetic_tables`` / ``amass_tables`` return), or a callable ``batch -> tables`` (the
    synthetic tables need the batch's kinematics), or a ``MotionLibB200`` built on ``batch``.
    ``tracked_bodies``: body names or indices (default ``cfg.env.tracked_bodies``, None = all bodies).
    ``batch_factory(cfg, num_envs, **kw)`` builds the owned batch (default ``HumanoidBatchB200``); further keywords go to it."""

    def __init__(self, cfg: Any, motion: Union[dict, Callable, MotionLibB200], num_envs: Optional[int] = None, device: str = "cuda:0",
                 seed: Optional[int] = None, tracked_bodies: Optional[Sequence] = None, batch_factory: Optional[Callable] = None, **batch_kw):
        e = cfg.env
        if e.get("task", None) != "HumanoidIm":
            raise ValueError(f"HumanoidImB200 needs cfg.env.task == 'HumanoidIm' (make_cfg(env='im')), got {e.get('task', None)!r}")
        if isinstance(motion, MotionLibB200):
            self.batch = motion.env
            self.lib = motion
        else:
            if batch_factory is None:
                self.batch = HumanoidBatchB200(cfg, num_envs=num_envs, device=device, seed=seed, **batch_kw)
            else:
                self.batch = batch_factory(cfg, num_envs, seed=seed, **batch_kw)
            self.lib = MotionLibB200(self.batch, motion(self.batch) if callable(motion) else motion)
        b, lib = self.batch, self.lib
        if b._aux.body_linvel is None or b._aux.xpos is None:
            raise ValueError("HumanoidImB200 needs the batch's side outputs (with_aux=True): body poses and velocities")
        self.cfg, self.model, self.device, self.num_envs, self.num_actions, self.dt = cfg, b.model, b.device, b.num_envs, b.num_actions, b.dt
        self.max_episode_length = int(e.episode_length)
        m, N, dv = b.model, b.num_envs, b.device
        for k, w in (("xpos", 3), ("xquat", 4), ("body_vel", 3), ("body_ang_vel", 3)):
            if lib.tables[k].shape[1] != w * m.nbody:
                raise ValueError(f"motion table {k!r} has {lib.tables[k].shape[1]} columns, the model needs {w * m.nbody}")
        tb = tracked_bodies if tracked_bodies is not None else e.get("tracked_bodies", None)
        bodies = list(range(m.nbody)) if tb is None else [self._body_index(x) for x in tb]
        self.tracked_bodies = bodies
        self._bodies = np.ascontiguousarray(np.asarray(bodies, dtype=np.int32))
        L = b._L()
        self._icfg = SmplsimImitationCfgC(
            k_pos=float(e.im_k_pos), k_rot=float(e.im_k_rot), k_vel=float(e.im_k_vel), k_angvel=float(e.im_k_angvel),
            w_pos=float(e.im_w_pos), w_rot=float(e.im_w_rot), w_vel=float(e.im_w_vel), w_angvel=float(e.im_w_angvel),
            termination_distance=float(e.termination_distance), episode_length=self.max_episode_length, self_obs_dim=int(b.num_obs),
            num_tracked=len(bodies), tracked_bodies=self._bodies.ctypes.data if len(bodies) else None)
        self._tab = SmplsimMotionTablesC(
            xpos=lib.tables["xpos"].data_ptr(), xquat=lib.tables["xquat"].data_ptr(), body_vel=lib.tables["body_vel"].data_ptr(),
            body_ang_vel=lib.tables["body_ang_vel"].data_ptr(), motion_len=lib._motion_lengths.data_ptr(),
            num_frames=lib._motion_num_frames.data_ptr(), motion_dt=lib._motion_dt.data_ptr(), length_starts=lib.length_starts.data_ptr(),
            num_motions=lib.num_motions(), nbody=lib.tables["xpos"].shape[1] // 3)
        self.num_obs = L.smplsim_imitation_obs_dim(b._h, len(bodies))
        f32 = dict(dtype=torch.float32, device=dv)
        u8 = dict(dtype=torch.uint8, device=dv)
        self.obs_buf = torch.zeros(N, max(self.num_obs, 0), **f32)
        self.rew_buf = torch.zeros(N, **f32)
        self.mpjpe = torch.zeros(N, **f32)
        self.terminate_buf = torch.zeros(N, **u8)
        self.truncate_buf = torch.zeros(N, **u8)
        self.reset_buf = torch.ones(N, **u8)
        self.progress_buf = b.progress_buf
        self.motion_ids = torch.zeros(N, dtype=torch.int32, device=dv)
        self.motion_start_times = torch.zeros(N, **f32)
        self.ref_frames = torch.zeros(N, 2, dtype=torch.int32, device=dv)
        self.extras = {"terminate": self.terminate_buf, "sim_warning": b.status, "mpjpe": self.mpjpe}
        # reference state of a reset (gathered rows of the qpos / qvel tables) and per-clip statistics
        self._qpos0 = torch.zeros(N, m.nq, **f32)
        self._qvel0 = torch.zeros(N, m.nv, **f32)
        self._ids64 = torch.zeros(N, dtype=torch.int64, device=dv)
        self._done_f = torch.zeros(N, dtype=torch.float64, device=dv)
        self._term_f = torch.zeros(N, dtype=torch.float64, device=dv)
        K = lib.num_motions()
        self.clip_episodes = torch.zeros(K, dtype=torch.float64, device=dv)       # episodes that ended on each clip
        self.clip_terminations = torch.zeros(K, dtype=torch.float64, device=dv)   # ... of which by early termination
        self._task(None, obs_only=True)      # argument check up front (a bad tracked body is refused here, not at the first step)

    def _body_index(self, x):
        m = self.batch.model
        if isinstance(x, str):
            if x not in m.body_names:
                raise ValueError(f"unknown body name {x!r}")
            return list(m.body_names).index(x)
        if isinstance(x, bool) or not isinstance(x, (int, np.integer)):
            raise ValueError(f"tracked_bodies entries must be body names or indices, got {x!r}")
        return int(x)

    @property
    def gpu_launches(self) -> int:
        return self.batch.gpu_launches

    def _task(self, mask: Optional[torch.Tensor], obs_only: bool):
        b = self.batch
        b._check(b._L().smplsim_imitation(b._h, C.byref(self._icfg), C.byref(self._tab), _ptr(self.motion_ids), _ptr(self.motion_start_times),
                                          _ptr(b.progress_buf), C.byref(b._aux), _ptr(b.obs_buf), _ptr(mask), int(obs_only),
                                          _ptr(self.obs_buf), _ptr(self.rew_buf), _ptr(self.terminate_buf), _ptr(self.truncate_buf),
                                          _ptr(self.mpjpe), _ptr(self.ref_frames), b._stream()))
        b.gpu_launches += 1

    def step(self, actions: torch.Tensor):
        """The batch's physics step, then the task kernel: ``obs_buf, rew_buf, terminate_buf, truncate_buf, reset_buf, mpjpe`` updated in
        place.  In stream order, no host sync, nothing allocated."""
        self.batch.step(actions)
        self._task(None, obs_only=False)
        torch.bitwise_or(self.terminate_buf, self.truncate_buf, out=self.reset_buf)
        self._done_f.copy_(self.reset_buf)
        self._term_f.copy_(self.terminate_buf)
        self.clip_episodes.index_add_(0, self._ids64, self._done_f)
        self.clip_terminations.index_add_(0, self._ids64, self._term_f)
        return self.obs_buf, self.rew_buf, self.terminate_buf, self.truncate_buf

    def reset(self, env_ids: Optional[torch.Tensor] = None, motion_ids: Optional[torch.Tensor] = None,
              motion_times: Optional[torch.Tensor] = None):
        """Put the envs ``env_ids`` (None = all; an index tensor or a uint8 / bool mask) on a reference frame: a clip from
        ``lib.sample_motions`` and a start time from ``lib.sample_time`` (at least one control period before the clip's end), or the
        caller's ``motion_ids`` / ``motion_times`` (full ``[num_envs]`` tensors; rows outside ``env_ids`` are ignored).  Masked and in
        stream order: the other envs keep their state, observation row, clip and start time."""
        b, lib, N, dv = self.batch, self.lib, self.num_envs, self.device
        mask = None
        if env_ids is not None:
            if env_ids.dtype in (torch.bool, torch.uint8) and env_ids.numel() == N:
                mask = env_ids.to(dv, torch.uint8).contiguous()
            else:
                if env_ids.numel() == 0:
                    return self.obs_buf
                mask = torch.zeros(N, dtype=torch.uint8, device=dv)
                mask[env_ids.to(dv).long()] = 1
        ids = lib.sample_motions(N) if motion_ids is None else motion_ids.to(dv, torch.int32)
        if ids.shape != (N,):
            raise ValueError(f"motion_ids must have shape ({N},), got {tuple(ids.shape)}")
        t0 = lib.sample_time(ids, truncate_time=self.dt).clamp_(min=0.0) if motion_times is None else motion_times.to(dv, torch.float32)
        if t0.shape != (N,):
            raise ValueError(f"motion_times must have shape ({N},), got {tuple(t0.shape)}")
        if mask is None:
            self.motion_ids.copy_(ids)
            self.motion_start_times.copy_(t0)
        else:
            sel = mask.bool()
            torch.where(sel, ids, self.motion_ids, out=self.motion_ids)
            torch.where(sel, t0, self.motion_start_times, out=self.motion_start_times)
        self._ids64.copy_(self.motion_ids)
        lib.gather_into(("qpos", "qvel"), self.motion_ids, self.motion_start_times, (self._qpos0, self._qvel0))
        b.reset(mask, init_mode=2, qpos0=self._qpos0, qvel0=self._qvel0)
        self._task(mask, obs_only=True)
        self._keep = mask
        return self.obs_buf

    def reset_done(self):
        """Reset every env whose reset_buf is set (in-stream, no host sync)."""
        return self.reset(self.reset_buf)

    def termination_history(self) -> torch.Tensor:
        """Early terminations per clip since construction (float64 ``[num_motions]``), the argument of
        ``MotionLibB200.update_sampling_prob``: clips that fail more are drawn more (PMCP).  ``clip_episodes`` holds the episode counts."""
        return self.clip_terminations.clone()
