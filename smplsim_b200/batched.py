"""Batched tensor protocol (boundary B2, SURVEY.md 8b): the reference's own GPU-sim surface
(smpl_sim/envs/nv/base_task.py:97-124,294-313, smpl_sim/envs/nv/humanoid.py:2127-2143) backed by
libsmplsim_b200.so instead of Isaac Gym, with MuJoCo-env semantics (smpl_sim/envs/humanoid_env.py).

PyTorch owns every tensor (device memory, streams); the C ABI receives raw pointers per call.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence, Any, Optional

import numpy as np
import torch

from . import _lib
from .abi import SmplsimAuxC, SmplsimEnvParamsC, SmplsimFdCfgC, SmplsimInverseFdCfgC, SmplsimStateC, env_cfg_from, model_from_cfg
from .model import ModelDesc


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _fd_eps(**eps: float):
    """The finite-difference steps of ``transition_fd`` / ``inverse_fd`` as floats, in the order given; raises unless each is finite and > 0."""
    for name, e in eps.items():
        if not (np.isfinite(e) and e > 0):
            raise ValueError(f"{name} must be finite and > 0, got {e!r}")
    return [float(e) for e in eps.values()]


_NO_ENVS = object()     # HumanoidBatchB200._env_mask of an empty index tensor: the call selects no env


class HumanoidBatchB200:
    """N independent SMPL humanoid envs stepped in lockstep on one GPU.

    Attributes mirroring the reference's tensor API: ``num_envs, num_obs, num_actions, device, obs_buf,
    rew_buf, reset_buf, progress_buf, extras`` (+ ``terminate_buf, truncate_buf``).  State lives in the
    SoA tensors ``qpos[N,nq], qvel[N,nv]`` etc.
    """

    def __init__(self, cfg: Any, num_envs: Optional[int] = None, device: str = "cuda:0", seed: Optional[int] = None,
                 model: Optional[ModelDesc] = None, rank: int = 0, with_aux: bool = True,
                 models: Optional[Sequence[ModelDesc]] = None, env_model: Optional[Sequence[int]] = None,
                 contact_wrench: bool = False):
        """``models`` + ``env_model`` ([num_envs] indices into models): per-env body shapes in one batch -- what one SMPL_Robot per
        env process gives the reference (humanoid_env.py:219-250).  Same tree / joints / geom layout in every model.

        ``contact_wrench=True`` allocates ``self.contact_wrench`` ``[num_envs, nbody, 6]`` float32 on the device (also with
        ``with_aux=False``), which ``step`` / ``mj_step`` fill with the per-body contact wrench of the last forward pass (last substep,
        before integration; the pass ``contact_mask`` and ``qacc`` describe): rows indexed like ``xpos`` (row 0 = root / Pelvis),
        ``[..., 0:3]`` the world-frame force the floor and geom-geom contacts apply to the body, ``[..., 3:6]`` the torque of those forces
        about the body's centre of mass -- the convention of ``xfrc_applied``.  ``contact_wrench[..., :3]`` is the layout of Isaac's
        ``net_contact_force`` ([N, nbody, 3]).  Bodies without contact force read exact zeros; ``reset`` zeroes the rows of the envs it
        resets.  False (the default): ``self.contact_wrench`` is None and the kernels skip it."""
        self._require_device(device)
        self.cfg = cfg
        e = cfg.env
        self.num_envs = int(num_envs if num_envs is not None else (e.get("num_envs", 1) if hasattr(e, "get") else 1))
        self.device = torch.device(device)
        self.models = list(models) if models is not None else None
        if self.models is not None:
            if env_model is None or len(env_model) != self.num_envs:
                raise ValueError("models= needs env_model with one entry per env")
            model = self.models[0]
        self.model = model if model is not None else model_from_cfg(cfg)
        seed = int(cfg.get("seed", 0) if seed is None and hasattr(cfg, "get") else (seed or 0))
        self.seed = (seed + 0x9E3779B97F4A7C15 * rank) & 0xFFFFFFFFFFFFFFFF      # per-rank Philox key (env sharding)
        self.envcfg = env_cfg_from(cfg, self.model, seed=self.seed)
        self._cmodel = self.model.c_struct()
        self._h = C.c_void_p()
        L = self._L()
        dev_index = self._device_index()
        if self.models is None:
            self._check(L.smplsim_create(C.addressof(self._cmodel), C.addressof(self.envcfg), self.num_envs, dev_index, C.byref(self._h)))
            self.env_model = None
        else:
            self._cmodels_each = [m.c_struct() for m in self.models]          # keeps the arrays the structs point at alive
            arr = (type(self._cmodel) * len(self.models))(*self._cmodels_each)
            em = np.ascontiguousarray(np.asarray(env_model, dtype=np.int32))
            self._check(L.smplsim_create_shapes(C.addressof(arr), len(self.models), C.c_void_p(em.ctypes.data), C.addressof(self.envcfg),
                                                self.num_envs, dev_index, C.byref(self._h)))
            self.env_model = em
        self.num_obs = L.smplsim_obs_dim(self._h)
        self.num_actions = self.model.nu
        self.dt = float(self.model.timestep * self.envcfg.nsubsteps)
        self.max_episode_length = int(e.episode_length)
        N, m, dv = self.num_envs, self.model, self.device
        f32 = dict(dtype=torch.float32, device=dv)
        i32 = dict(dtype=torch.int32, device=dv)
        self.qpos = torch.zeros(N, m.nq, **f32)
        self.qpos[:, 3] = 1.0
        self.qvel = torch.zeros(N, m.nv, **f32)
        self.qpos_fwd = self.qpos.clone()
        self.qvel_fwd = torch.zeros(N, m.nv, **f32)
        self.qacc_warm = torch.zeros(N, m.nv, **f32)
        self.task_target = torch.zeros(N, 4, **f32)
        self.task_change_step = torch.zeros(N, **i32)
        self.progress_buf = torch.zeros(N, **i32)
        self.recovery = torch.zeros(N, **i32)
        self.rng_counter = torch.zeros(N, **i32)
        self.pid_integral = torch.zeros(N, m.nu, **f32)              # SimplePID state (simple_pid only; survives reset, like the reference object)
        self.pid_last_error = torch.full((N, m.nu), float('nan'), **f32)   # NaN = None
        self.obs_buf = torch.zeros(N, self.num_obs, **f32)
        self.rew_buf = torch.zeros(N, **f32)
        self.terminate_buf = torch.zeros(N, dtype=torch.uint8, device=dv)
        self.truncate_buf = torch.zeros(N, dtype=torch.uint8, device=dv)
        self.reset_buf = torch.ones(N, dtype=torch.uint8, device=dv)
        # side outputs of the last forward pass
        self.xpos = torch.zeros(N, m.nbody, 3, **f32)
        self.xquat = torch.zeros(N, m.nbody, 4, **f32)
        self.body_linvel = torch.zeros(N, m.nbody, 3, **f32)
        self.body_angvel = torch.zeros(N, m.nbody, 3, **f32)
        self.contact_mask = torch.zeros(N, dtype=torch.int64, device=dv)
        self.qacc = torch.zeros(N, m.nv, **f32)
        self.ctrl = torch.zeros(N, m.nu, **f32)
        self.solver_iter = torch.zeros(N, **i32)
        self.status = torch.zeros(N, dtype=torch.uint8, device=dv)   # mj_warning bits of the last call (1 qpos, 2 qvel, 4 qacc)
        self.extras = {"terminate": self.terminate_buf, "sim_warning": self.status}
        self._state = SmplsimStateC(*[t.data_ptr() for t in (self.qpos, self.qvel, self.qpos_fwd, self.qvel_fwd, self.qacc_warm,
                                                             self.task_target, self.task_change_step, self.progress_buf,
                                                             self.recovery, self.rng_counter, self.pid_integral, self.pid_last_error)])
        self._aux = SmplsimAuxC(*[t.data_ptr() for t in (self.xpos, self.xquat, self.body_linvel, self.body_angvel,
                                                         self.contact_mask, self.qacc, self.ctrl, self.solver_iter, self.status)])
        if not with_aux:        # throughput runs: skip the side outputs (NULL pointers), keep the 1-byte status
            self._aux = SmplsimAuxC(status=self.status.data_ptr())
        self.contact_wrench = torch.zeros(N, m.nbody, 6, **f32) if contact_wrench else None   # per-body contact wrench (see above)
        if self.contact_wrench is not None:
            self._aux.contact_wrench = self.contact_wrench.data_ptr()
        self._xfrc = None           # mj_data.xfrc_applied (None: no external wrench; see xfrc_applied)
        self._cams = {}             # named cameras of render(), resolved once (a tracking camera's offset needs host kinematics)
        self.gpu_launches = 0

    def __del__(self):
        try:
            if self._h:
                self._L().smplsim_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass

    # ------------------------------------------------------------------ binding to libsmplsim_b200.so (CUDA only)
    def _require_device(self, device):
        if not torch.cuda.is_available():
            raise RuntimeError("HumanoidBatchB200 needs a CUDA device (there is no CPU fallback for the stepper)")

    def _L(self):
        return _lib.lib()

    def _check(self, rc):
        if rc != 0:
            raise _lib.SmplsimError(f"libsmplsim_b200 error {rc}: {self._L().smplsim_last_error().decode()}")

    def _device_index(self):
        return self.device.index if self.device.index is not None else torch.cuda.current_device()

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ------------------------------------------------------------------ reference tensor API
    def reset(self, env_ids: Optional[torch.Tensor] = None, init_mode: int = -1, qpos0: Optional[torch.Tensor] = None,
              qvel0: Optional[torch.Tensor] = None):
        """HumanoidTask.reset for ``env_ids`` (None = all; an index tensor or a uint8/bool mask)."""
        mask = self._env_mask(env_ids)
        if mask is _NO_ENVS:
            return self.obs_buf
        if qpos0 is not None:
            qpos0 = qpos0.to(self.device, torch.float32).contiguous()
            qvel0 = qvel0.to(self.device, torch.float32).contiguous()
        self._check(self._L().smplsim_reset(self._h, C.byref(self._state), _ptr(mask), int(init_mode), _ptr(qpos0), _ptr(qvel0),
                                            _ptr(self.obs_buf), C.byref(self._aux), self._stream()))
        self.gpu_launches += 1
        self._keep = (mask, qpos0, qvel0)
        return self.obs_buf

    def _env_mask(self, env_ids):
        """The uint8 [num_envs] mask of an env selection: None (all envs) stays None, a bool / uint8 mask of num_envs entries is
        converted where it is (a contiguous uint8 mask is returned as it is, so ``reset(self.reset_buf)`` allocates, copies and syncs
        nothing), an index tensor is scattered into a new mask on this batch's device, and an empty index tensor gives ``_NO_ENVS``."""
        if env_ids is None:
            return None
        if env_ids.dtype in (torch.bool, torch.uint8) and env_ids.numel() == self.num_envs:
            return env_ids.to(torch.uint8).contiguous()
        if env_ids.numel() == 0:
            return _NO_ENVS
        mask = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
        mask[env_ids.long()] = 1
        return mask

    def reset_done(self):
        """Reset every env whose reset_buf is set (in-stream, no host sync)."""
        return self.reset(self.reset_buf)

    def step(self, actions: torch.Tensor):
        """BaseEnv.step for all envs: obs_buf, rew_buf, terminate/truncate/reset_buf, progress_buf updated in place."""
        a = actions.to(self.device, torch.float32)
        if bool(self.cfg.env.clip_actions):
            a = torch.clamp(a, -1.0, 1.0)      # action_space Box(-1,1) (humanoid_env.py:180-184; agent.py:153-161)
        a = a.contiguous()
        assert a.shape == (self.num_envs, self.num_actions)
        self._set_xfrc()
        self._check(self._L().smplsim_step(self._h, C.byref(self._state), _ptr(a), _ptr(self.obs_buf), _ptr(self.rew_buf),
                                           _ptr(self.terminate_buf), _ptr(self.truncate_buf), C.byref(self._aux), self._stream()))
        self.gpu_launches += 1
        torch.bitwise_or(self.terminate_buf, self.truncate_buf, out=self.reset_buf)
        self._keep_a = a
        return self.obs_buf, self.rew_buf, self.terminate_buf, self.truncate_buf

    # ------------------------------------------------------------------ external body wrenches (mj_data.xfrc_applied)
    @property
    def xfrc_applied(self) -> Optional[torch.Tensor]:
        """External wrench per robot body and env: None (none, the default) or a caller-owned contiguous float32 tensor
        ``[num_envs, nbody, 6]`` on this batch's device, indexed like ``xpos`` (row 0 = root / Pelvis).  Each row is a world-frame force
        ``(fx, fy, fz)`` acting at the body's centre of mass and a world-frame torque ``(tx, ty, tz)``, as MuJoCo's
        ``mj_data.xfrc_applied``.  ``step`` and ``mj_step`` read it on every call and hold it constant over all substeps of the call; it
        enters the dynamics (qfrc_smooth) but not the bias forces the stable-PD controller reads.  ``reset`` ignores it.  An env that
        auto-resets on a bad state inside a call runs the rest of that call without it (mj_resetData zeroes xfrc_applied); the tensor
        itself is never written.  Assign None to clear it."""
        return self._xfrc

    @xfrc_applied.setter
    def xfrc_applied(self, t: Optional[torch.Tensor]):
        shape = (self.num_envs, self.model.nbody, 6)
        self._xfrc = self._checked("xfrc_applied", t, shape, optional=True, want=f"{shape} (envs, robot bodies, force + torque)")

    def _set_xfrc(self):
        """The wrench pointer of this call (NULL: none); the tensor is kept referenced until the next call."""
        self._state.xfrc_applied = None if self._xfrc is None else self._xfrc.data_ptr()
        self._keep_xfrc = self._xfrc

    # ------------------------------------------------------------------ per-env physics parameters (domain randomization)
    ENV_PARAMS = ("friction", "gravity", "kp", "kd", "torque_limit", "body_mass_scale")

    def _env_param_shapes(self):
        m, N = self.model, self.num_envs
        return {"friction": (N,), "gravity": (N, 3), "kp": (N, m.nu), "kd": (N, m.nu), "torque_limit": (N, m.nu),
                "body_mass_scale": (N, m.nbody)}

    def set_env_params(self, env_ids: Optional[torch.Tensor] = None, *, friction: Optional[torch.Tensor] = None,
                       gravity: Optional[torch.Tensor] = None, kp: Optional[torch.Tensor] = None, kd: Optional[torch.Tensor] = None,
                       torque_limit: Optional[torch.Tensor] = None, body_mass_scale: Optional[torch.Tensor] = None):
        """Per-env physics parameters for domain randomization.  For the envs in ``env_ids`` (None = all; an index tensor or a
        bool/uint8 mask, as in ``reset``) each given value replaces that env's parameter; a parameter left None keeps its current value.
        Env ``e`` is then simulated as the model (its own shape with per-env shapes) with these fields replaced, as MuJoCo does when
        ``MjModel`` fields are edited in place without ``mj_setConst``:

        - ``friction [N]``: sliding friction of every floor and geom-geom contact;
        - ``gravity [N, 3]``;
        - ``kp``, ``kd``, ``torque_limit [N, nu]``: the gains and torque limits the configured controller reads (``model.act_kp`` /
          ``act_kd`` / ``act_torque_lim``; in torque mode only the clamp);
        - ``body_mass_scale [N, nbody]``: each body's mass and rotational inertia times the scale; its centre of mass stays.

        The invweight0 values, and with them the constraint regularisation, stay the nominal model's.  Values are full
        ``[num_envs, ...]`` float32 tensors on this batch's device; rows outside ``env_ids`` are ignored.  Raises ``ValueError`` for a
        wrong shape, dtype or device, non-finite values, ``friction < 1e-5``, ``kp`` or ``kd < 0``, ``torque_limit <= 0`` or
        ``body_mass_scale <= 0`` in the selected rows.  Checking the values costs one host sync: call this at reset time, not every
        step.  ``step``, ``mj_step``, ``reset``, ``inverse``, ``dynamics`` and ``render`` (TRACKCOM) use the values from the next call on;
        ``inverse`` and ``dynamics`` then take ``n == num_envs`` rows (row i = env i).  ``clear_env_params`` goes back to the model."""
        vals = {"friction": friction, "gravity": gravity, "kp": kp, "kd": kd, "torque_limit": torque_limit, "body_mass_scale": body_mass_scale}
        shapes = self._env_param_shapes()
        given = {name: self._checked(name, t, shapes[name], copy=True, want=str(shapes[name])) for name, t in vals.items() if t is not None}
        mask = self._env_mask(None if env_ids is None else env_ids.to(self.device))
        if mask is _NO_ENVS or not given:
            return
        sel = None if mask is None else mask.bool()
        bad = []
        for name, x in given.items():   # elementwise on the device; the one host sync is the .cpu() below
            b = ~torch.isfinite(x)
            if name == "friction":
                b = b | (x < 1e-5)
            elif name in ("kp", "kd"):
                b = b | (x < 0)
            elif name in ("torque_limit", "body_mass_scale"):
                b = b | (x <= 0)
            if sel is not None:
                b = b & sel.view((-1,) + (1,) * (b.dim() - 1))
            bad.append(b.any())
        flags = torch.stack(bad).cpu().tolist()
        rules = {"friction": "finite and >= 1e-5", "gravity": "finite", "kp": "finite and >= 0", "kd": "finite and >= 0",
                 "torque_limit": "finite and > 0", "body_mass_scale": "finite and > 0"}
        for name, f in zip(given, flags):
            if f:
                raise ValueError(f"{name} must be {rules[name]} in the selected envs")
        p = SmplsimEnvParamsC(**{k: v.data_ptr() for k, v in given.items()})
        self._check(self._L().smplsim_set_env_params(self._h, C.byref(p), _ptr(mask), self._stream()))
        self.gpu_launches += 1
        self._keep_prm = (mask, given)

    @property
    def env_params(self) -> dict:
        """The current per-env parameters as a dict of new ``[num_envs, ...]`` float32 tensors (keys as ``set_env_params`` takes them);
        the model's values (each env's shape) where nothing has been set."""
        out = {k: torch.empty(s, dtype=torch.float32, device=self.device) for k, s in self._env_param_shapes().items()}
        self._check(self._L().smplsim_get_env_params(self._h, *[_ptr(out[k]) for k in self.ENV_PARAMS], self._stream()))
        self.gpu_launches += 1
        return out

    def clear_env_params(self):
        """Drop every per-env parameter: the batch simulates the model again, exactly as before the first ``set_env_params``
        (synchronizes with the device)."""
        self._check(self._L().smplsim_clear_env_params(self._h))

    # ------------------------------------------------------------------ raw physics / kinematics (parity + tools)
    def mj_step(self, ctrl: torch.Tensor, nsub: int = 1):
        """data.ctrl[:] = ctrl; mujoco.mj_step x nsub."""
        c = ctrl.to(self.device, torch.float32).contiguous()
        self._set_xfrc()
        self._check(self._L().smplsim_mj_step(self._h, C.byref(self._state), _ptr(c), int(nsub), C.byref(self._aux), self._stream()))
        self.gpu_launches += 1
        self._keep_a = c

    def kinematics(self, qpos: torch.Tensor):
        q = qpos.to(self.device, torch.float32).contiguous()
        n = q.shape[0]
        xpos = torch.empty(n, self.model.nbody, 3, dtype=torch.float32, device=self.device)
        xquat = torch.empty(n, self.model.nbody, 4, dtype=torch.float32, device=self.device)
        self._check(self._L().smplsim_kinematics(self._h, _ptr(q), _ptr(xpos), _ptr(xquat), n, self._stream()))
        self.gpu_launches += 1
        return xpos, xquat

    def _checked(self, name, t, shape, copy=False, optional=False, want=None):
        """Caller tensor ``t`` checked for ``shape`` (None entries free), float32 and this batch's device, and returned.  A tensor that is
        not contiguous is refused, or with ``copy`` returned as a contiguous copy (for inputs the call only reads; a tensor the batch
        keeps, as ``xfrc_applied``, must stay the caller's).  With ``optional`` None (the argument left out) is returned as None.
        ``want``: the shape as the refusal states it (default: ``shape``, free entries as n)."""
        if t is None and optional:
            return None
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch.Tensor{' or None' if optional else ''}, got {type(t).__name__}")
        if t.dim() != len(shape) or any(s is not None and t.shape[i] != s for i, s in enumerate(shape)):
            want = want or "[" + ", ".join("n" if s is None else str(s) for s in shape) + "]"
            raise ValueError(f"{name} must have shape {want}, got {tuple(t.shape)}")
        if t.dtype != torch.float32:
            raise ValueError(f"{name} must be float32, got {t.dtype}")
        dv = self.device
        if t.device.type != dv.type or (dv.index is not None and t.device.index != dv.index):
            raise ValueError(f"{name} must live on {dv}, got {t.device}")
        if t.is_contiguous():
            return t
        if not copy:
            raise ValueError(f"{name} must be contiguous")
        return t.contiguous()

    def _rows(self, *rows, n=None, optional=False):
        """Caller state rows ``(name, tensor, width)``, each ``[n, width]`` with the n of qpos (``n``, or the first row's), checked by
        ``_checked`` and returned contiguous; with ``optional`` a row given as None is returned as None."""
        out = []
        for name, t, w in rows:
            t = self._checked(name, t, (n, w), copy=True, optional=optional, want=f"[n, {w}] with the same n as qpos")
            if n is None:
                n = t.shape[0]
            out.append(t)
        return out

    def inverse(self, qpos: torch.Tensor, qvel: torch.Tensor, qacc: torch.Tensor, contact_wrench: bool = False):
        """mujoco.mj_inverse on caller rows: ``qfrc_inverse [n, nv]`` (and ``contact_wrench [n, nbody, 6]`` when asked), the generalized
        force that produces ``qacc`` at ``(qpos, qvel)``: ``M qacc + qfrc_bias - J^T f`` with the soft-constraint forces
        ``f = -D min(0, J qacc - aref)`` of the floor contacts and joint limits.  ``qfrc_inverse[:, 0:6]`` is the root residual (world-frame
        force, torque about the root body's axes), ``[:, 6:]`` the joint torques.  ``contact_wrench`` uses the convention of
        ``self.contact_wrench``.  Float32 tensors on this batch's device, ``[n, nq]`` / ``[n, nv]`` / ``[n, nv]``; any n on a one-shape
        batch, n == num_envs with per-env shapes (row i uses env i's shape).  Reads no env state and changes none; ``xfrc_applied``
        is not taken.  Not available with ``cfg.env.self_collision``."""
        m = self.model
        q, v, a = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv), ("qacc", qacc, m.nv))
        n = q.shape[0]
        out = torch.empty(n, m.nv, dtype=torch.float32, device=self.device)
        cw = torch.empty(n, m.nbody, 6, dtype=torch.float32, device=self.device) if contact_wrench else None
        self._check(self._L().smplsim_inverse(self._h, _ptr(q), _ptr(v), _ptr(a), _ptr(out), _ptr(cw), n, self._stream()))
        self.gpu_launches += 1
        return (out, cw) if contact_wrench else out

    def forward(self, qpos: torch.Tensor, qvel: torch.Tensor, ctrl: torch.Tensor, qacc_warmstart: Optional[torch.Tensor] = None,
                contact_wrench: bool = False):
        """mujoco.mj_forward on caller rows: the accelerations of ``(qpos, qvel)`` under the raw joint torques ``ctrl`` (as ``mj_step``
        takes them, not clamped), with the floor contacts and joint limits of that state.  ``qacc_warmstart`` (None: zeros) is where the
        constraint solve starts.  Returns a dict of ``qacc [n, nv]``, ``contact_mask [n]`` (int64 bits as ``self.contact_mask``),
        ``solver_iter [n]``, ``status [n]`` (bits as ``self.status``) and, when asked, ``contact_wrench [n, nbody, 6]`` (as
        ``self.contact_wrench``).  The pass is the first substep of ``mj_step(ctrl, 1)`` without the integration, from empty working-set
        memory.  A row with a non-finite input gets its status bits and unspecified values in that row only; there is no auto-reset.
        Float32 tensors on this batch's device; row rules of ``inverse``.  Reads no env state and changes none; ``xfrc_applied`` is not
        taken.  Not available with ``cfg.env.self_collision``."""
        m = self.model
        q, v, u = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv), ("ctrl", ctrl, m.nu))
        n, dv = q.shape[0], self.device
        (w,) = self._rows(("qacc_warmstart", qacc_warmstart, m.nv), n=n, optional=True)
        out = {"qacc": torch.empty(n, m.nv, dtype=torch.float32, device=dv), "contact_mask": torch.empty(n, dtype=torch.int64, device=dv),
               "solver_iter": torch.empty(n, dtype=torch.int32, device=dv), "status": torch.empty(n, dtype=torch.uint8, device=dv)}
        if contact_wrench:
            out["contact_wrench"] = torch.empty(n, m.nbody, 6, dtype=torch.float32, device=dv)
        self._check(self._L().smplsim_forward(self._h, _ptr(q), _ptr(v), _ptr(u), _ptr(w), n, _ptr(out["qacc"]), _ptr(out["contact_mask"]),
                                              _ptr(out["solver_iter"]), _ptr(out["status"]), _ptr(out.get("contact_wrench")), self._stream()))
        self.gpu_launches += 1
        return out

    FD_EPS = (1e-2, 1e-1, 1.0)   # eps_qpos (rad / m), eps_qvel, eps_ctrl (N m): the fp32 steps DESIGN.md 2 measured

    def transition_fd(self, qpos: torch.Tensor, qvel: torch.Tensor, ctrl: torch.Tensor, eps_qpos: float = FD_EPS[0],
                      eps_qvel: float = FD_EPS[1], eps_ctrl: float = FD_EPS[2], centered: bool = True, dqacc: bool = False):
        """Finite-difference derivatives of one ``mj_step`` substep at caller rows, as ``mujoco.mjd_transitionFD`` without sensors.
        State tangent ``x = [dq (nv) ; qvel (nv)]`` (root rotation tangent in the body frame, ``q * exp(d)``), input ``u = ctrl (nu)``.
        Returns a dict of

        - ``qacc [n, nv]``: the nominal forward pass;
        - ``A [n, 2nv, 2nv]``, ``B [n, 2nv, nu]``: ``dx'/dx``, ``dx'/du`` in MuJoCo's layout, assembled from ``dqacc`` and the
          semi-implicit Euler step;
        - ``flags [n, 2nv + nu]`` uint8 per column: 1 the two solves ended on different active sets (the column straddles a contact or
          joint-limit switch; never set with ``centered=False``), 2 a solve hit the iteration cap, dropped rows or saw a non-finite value;
        - ``dqacc [n, nv, 2nv + nu]`` when asked: ``d qacc / d [dq, qvel, ctrl]``.

        ``eps_*`` are the perturbations; MuJoCo's fp64 default of 1e-6 is rounding noise in fp32, and the defaults are the measured
        choice.  ``centered=False`` differences against the nominal (half the passes).  Float32 tensors on this batch's device, any n;
        single-shape batches without per-env parameters (raises otherwise), not with ``cfg.env.self_collision``.  Reads no env state and
        changes none."""
        m = self.model
        eps = _fd_eps(eps_qpos=eps_qpos, eps_qvel=eps_qvel, eps_ctrl=eps_ctrl)
        q, v, u = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv), ("ctrl", ctrl, m.nu))
        n, nx, f32 = q.shape[0], 2 * m.nv, dict(dtype=torch.float32, device=self.device)
        ncol = nx + m.nu
        out = {"qacc": torch.empty(n, m.nv, **f32), "A": torch.empty(n, nx, nx, **f32), "B": torch.empty(n, nx, m.nu, **f32),
               "flags": torch.empty(n, ncol, dtype=torch.uint8, device=self.device)}
        if dqacc:
            out["dqacc"] = torch.empty(n, m.nv, ncol, **f32)
        cfg = SmplsimFdCfgC(*eps, 1 if centered else 0, 0)
        self._check(self._L().smplsim_transition_fd(self._h, C.byref(cfg), _ptr(q), _ptr(v), _ptr(u), n, _ptr(out["qacc"]), _ptr(out.get("dqacc")),
                                                    _ptr(out["A"]), _ptr(out["B"]), _ptr(out["flags"]), self._stream()))
        self.gpu_launches += 1
        return out

    INVFD_EPS = (1e-3, 1e-2, 1.0)   # eps_qpos (rad / m), eps_qvel, eps_qacc: the fp32 steps DESIGN.md 2 measured

    def inverse_fd(self, qpos: torch.Tensor, qvel: torch.Tensor, qacc: torch.Tensor, eps_qpos: float = INVFD_EPS[0],
                   eps_qvel: float = INVFD_EPS[1], eps_qacc: float = INVFD_EPS[2], centered: bool = True):
        """Finite-difference derivatives of ``inverse`` at caller rows, as ``mujoco.mjd_inverseFD`` without sensors or ``DmDq``.  Input
        tangent ``x = [dq (nv) ; qvel (nv) ; qacc (nv)]`` (root rotation tangent in the body frame, ``q * exp(d)``).  Returns a dict of

        - ``qfrc_inverse [n, nv]``: the nominal pass, bit for bit what ``inverse`` gives;
        - ``dfrc [n, nv, 3nv]``: ``d qfrc_inverse / d [dq, qvel, qacc]``, ``dfrc[i, k, j] = d f_k / d x_j`` (the layout of
          ``transition_fd``'s ``dqacc``; ``mjd_inverseFD``'s ``DfDq``, ``DfDv``, ``DfDa`` are its three blocks transposed);
        - ``flags [n, 3nv]`` uint8 per column: 1 the two passes ended on different row sets (a contact appeared or went, or a row's
          ``r < 0`` status flipped; never set with ``centered=False``), 2 a pass dropped joint-limit rows or saw a non-finite value.

        ``eps_*`` are the perturbations; the defaults are the measured choice (fp32: MuJoCo's 1e-6 is rounding noise).  ``qfrc_inverse``
        is affine in ``qacc`` for a fixed row set, so ``eps_qacc`` costs no accuracy.  ``centered=False`` differences against the nominal
        (half the passes).  Float32 tensors on this batch's device, any n; single-shape batches without per-env parameters (raises
        otherwise), not with ``cfg.env.self_collision``.  Reads no env state and changes none."""
        m = self.model
        eps = _fd_eps(eps_qpos=eps_qpos, eps_qvel=eps_qvel, eps_qacc=eps_qacc)
        q, v, a = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv), ("qacc", qacc, m.nv))
        n, ncol, f32 = q.shape[0], 3 * m.nv, dict(dtype=torch.float32, device=self.device)
        out = {"qfrc_inverse": torch.empty(n, m.nv, **f32), "dfrc": torch.empty(n, m.nv, ncol, **f32),
               "flags": torch.empty(n, ncol, dtype=torch.uint8, device=self.device)}
        cfg = SmplsimInverseFdCfgC(*eps, 1 if centered else 0, 0)
        self._check(self._L().smplsim_inverse_fd(self._h, C.byref(cfg), _ptr(q), _ptr(v), _ptr(a), n, _ptr(out["qfrc_inverse"]),
                                                 _ptr(out["dfrc"]), _ptr(out["flags"]), self._stream()))
        self.gpu_launches += 1
        return out

    ROLLOUT_MODES = {"action": 0, "ctrl": 1}   # SMPLSIM_ROLLOUT_ACTION / SMPLSIM_ROLLOUT_CTRL

    def rollout(self, qpos: torch.Tensor, qvel: torch.Tensor, control: torch.Tensor, *, mode: str = "action", nsub: Optional[int] = None,
                qacc_warmstart: Optional[torch.Tensor] = None, qpos_fwd: Optional[torch.Tensor] = None, qvel_fwd: Optional[torch.Tensor] = None,
                body_poses: bool = False, status: bool = True, gains: Optional[torch.Tensor] = None, qpos_ref: Optional[torch.Tensor] = None,
                qvel_ref: Optional[torch.Tensor] = None):
        """Roll ``n`` control sequences forward from caller start states in one kernel launch, as ``mujoco.rollout.rollout``.  Row ``i``
        starts at ``(qpos[i], qvel[i])`` and takes one step per control row ``control[i, t]`` (``control`` is ``[n, T, nu]``):

        - ``mode="action"``: ``step`` -- a policy action (clamped to [-1, 1] with ``cfg.env.clip_actions``, as ``step`` does) through the
          configured controller for ``cfg.env.nsubsteps`` substeps; ``nsub`` must be None; ``simple_pid`` is refused (its integral /
          last error are env state);
        - ``mode="ctrl"``: ``mj_step(control[i, t], nsub)`` -- raw joint torques, not clamped, held for ``nsub`` substeps (None: 1,
          MuJoCo's rollout).

        Each step is bit for bit what that call does on a fresh batch after ``set_state(qpos[i], qvel[i])`` with ``qacc_warm =
        qacc_warmstart[i]``, keeping only the physics: no task target, observation, reward or termination.  ``qacc_warmstart`` (None:
        zeros) seeds the constraint solve; ``qpos_fwd`` / ``qvel_fwd`` (None: the start state, as ``set_state`` marks) are the state of
        the last forward pass that stable PD with stale inertia reads.  Passing an env's own ``qpos, qvel, qacc_warm, qpos_fwd,
        qvel_fwd`` continues its physics up to the solver's tolerance (the rollout starts from empty working-set memory).

        Returns a dict of ``qpos [n, T, nq]`` and ``qvel [n, T, nv]`` (the state after each step), ``status [n, T]`` uint8 (with
        ``status``: the bits of ``self.status`` the step raises -- a row whose state turns non-finite auto-resets and carries on; the
        self-contact bit is not evaluated) and, with ``body_poses``, ``xpos [n, T, nbody, 3]`` / ``xquat [n, T, nbody, 4]`` (the post-step
        poses of ``self.xpos`` / ``self.xquat``; asking for them changes no bit of the trajectory).  Float32 tensors on this batch's
        device; any n on a one-shape batch without per-env parameters, n == num_envs otherwise (row i uses env i's shape and
        parameters).  Reads no env state and changes none; ``xfrc_applied`` is not taken.  Not available with
        ``cfg.env.self_collision``.

        Closed loop (``gains`` given; ``qpos_ref`` and ``qvel_ref`` then required): ``control`` is the feedforward ``ubar`` and step ``t``
        applies ``u_t = ubar_t + K_t dx_t`` with ``K_t = gains[r, t]`` (``[nu, 2 nv]``), ``dx_t = differentiate_pos(qpos_ref[r, t], q_t)``
        stacked on ``qvel_t - qvel_ref[r, t]``, where ``(q_t, qvel_t)`` is the state before step ``t`` (the start state, then the output row
        ``t - 1``) and ``r`` is 0 when the leading dimension of ``gains`` / ``qpos_ref`` / ``qvel_ref`` is 1 (one schedule for every row)
        or the row when it is ``n``.  ``dx`` is the tangent of ``transition_fd``'s ``A`` and ``B`` (root rotation in the reference's body
        frame, on the shortest arc) and is exactly 0 for a state equal to its reference.  In ``mode="action"`` ``u_t`` is clamped to
        [-1, 1] with ``cfg.env.clip_actions`` (a NaN passes, as ``torch.clamp`` lets it, and resets the row); ctrl mode does not clamp.
        All of it runs in the one launch (an iLQR forward pass with its line-search steps as rows, TVLQR tracking from many starts).
        The result adds ``control [n, T, nu]``, the ``u_t`` each step applied: ``rollout`` on those rows replays the run bit for bit."""
        m = self.model
        if gains is None and (qpos_ref is not None or qvel_ref is not None):
            raise ValueError("qpos_ref / qvel_ref are the reference of the feedback law: give gains with them")
        if mode not in self.ROLLOUT_MODES:
            raise ValueError(f"mode must be 'action' or 'ctrl', got {mode!r}")
        if mode == "action":
            if nsub is not None:
                raise ValueError("nsub is for mode='ctrl'; an action step runs cfg.env.nsubsteps substeps")
            ns = 0
        else:
            ns = 1 if nsub is None else nsub
            if isinstance(ns, bool) or not isinstance(ns, (int, np.integer)) or ns < 1:
                raise ValueError(f"nsub must be an int >= 1, got {nsub!r}")
        q, v = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv))
        n = q.shape[0]
        w, qf, vf = self._rows(("qacc_warmstart", qacc_warmstart, m.nv), ("qpos_fwd", qpos_fwd, m.nq), ("qvel_fwd", qvel_fwd, m.nv), n=n,
                               optional=True)
        u = self._checked("control", control, (n, None, m.nu), copy=True)
        T = u.shape[1]
        if T < 1:
            raise ValueError("control must hold at least one step ([n, T, nu] with T >= 1)")
        if gains is not None:
            if qpos_ref is None or qvel_ref is None:
                raise ValueError("gains need qpos_ref and qvel_ref (the reference state of the feedback law)")
            nx = 2 * m.nv
            K = self._checked("gains", gains, (None, T, m.nu, nx), copy=True)
            r = K.shape[0]
            if r not in (1, n):
                raise ValueError(f"gains, qpos_ref and qvel_ref must have leading dimension 1 (shared) or n = {n}, got {r}")
            qr = self._checked("qpos_ref", qpos_ref, (r, T, m.nq), copy=True)
            vr = self._checked("qvel_ref", qvel_ref, (r, T, m.nv), copy=True)
        elif mode == "action" and bool(self.cfg.env.clip_actions):
            u = torch.clamp(u, -1.0, 1.0)
        dv, f32 = self.device, dict(dtype=torch.float32, device=self.device)
        out = {"qpos": torch.empty(n, T, m.nq, **f32), "qvel": torch.empty(n, T, m.nv, **f32)}
        if status:
            out["status"] = torch.empty(n, T, dtype=torch.uint8, device=dv)
        if body_poses:
            out["xpos"] = torch.empty(n, T, m.nbody, 3, **f32)
            out["xquat"] = torch.empty(n, T, m.nbody, 4, **f32)
        if gains is None:
            self._check(self._L().smplsim_rollout(self._h, self.ROLLOUT_MODES[mode], int(ns), _ptr(q), _ptr(v), _ptr(w), _ptr(qf), _ptr(vf),
                                                  _ptr(u), n, T, _ptr(out["qpos"]), _ptr(out["qvel"]), _ptr(out.get("status")),
                                                  _ptr(out.get("xpos")), _ptr(out.get("xquat")), self._stream()))
        else:
            out["control"] = torch.empty(n, T, m.nu, **f32)
            self._check(self._L().smplsim_rollout_feedback(
                self._h, self.ROLLOUT_MODES[mode], int(ns), _ptr(q), _ptr(v), _ptr(w), _ptr(qf), _ptr(vf), _ptr(u), n, T, _ptr(out["qpos"]),
                _ptr(out["qvel"]), _ptr(out.get("status")), _ptr(out.get("xpos")), _ptr(out.get("xquat")), _ptr(K), _ptr(qr), _ptr(vr), r,
                int(bool(self.cfg.env.clip_actions)), _ptr(out["control"]), self._stream()))
        self.gpu_launches += 1
        return out

    def differentiate_pos(self, qpos_ref: torch.Tensor, qpos: torch.Tensor) -> torch.Tensor:
        """``mj_differentiatePos(qpos_ref -> qpos)`` without the division by dt, batched over leading dimensions: ``[..., nq]`` pairs to
        ``[..., nv]``.  The position part of the tangent of ``transition_fd``'s ``A`` / ``B`` and of ``rollout``'s feedback law: root
        translation difference in the world frame, root rotation ``log(normalise(ref)^-1 * normalise(q))`` on the shortest arc (in the
        reference's body frame), hinge differences.  Any float dtype (fp64 for a Riccati pass); on the inputs' device."""
        qr, q = torch.broadcast_tensors(qpos_ref, qpos)
        if q.shape[-1] != self.model.nq:
            raise ValueError(f"qpos_ref / qpos must end in nq = {self.model.nq}, got {tuple(q.shape)}")
        b = qr[..., 3:7] / torch.linalg.vector_norm(qr[..., 3:7], dim=-1, keepdim=True)
        c = q[..., 3:7] / torch.linalg.vector_norm(q[..., 3:7], dim=-1, keepdim=True)
        bw, bv, cw, cv = b[..., :1], b[..., 1:], c[..., :1], c[..., 1:]
        rw = bw * cw + (bv * cv).sum(-1, keepdim=True)                      # conj(b) * c
        rv = bw * cv - cw * bv - torch.linalg.cross(bv, cv)
        sgn = torch.where(rw < 0, -1.0, 1.0).to(rw.dtype)
        rw, rv = rw * sgn, rv * sgn
        s = torch.linalg.vector_norm(rv, dim=-1, keepdim=True)
        f = torch.where(s > 0, 2 * torch.atan2(s, rw) / torch.where(s > 0, s, torch.ones_like(s)), torch.zeros_like(s))
        return torch.cat([q[..., 0:3] - qr[..., 0:3], f * rv, q[..., 7:] - qr[..., 7:]], dim=-1)

    def integrate_pos(self, qpos: torch.Tensor, dq: torch.Tensor) -> torch.Tensor:
        """``mj_integratePos(qpos, dq, 1)``, the inverse of ``differentiate_pos``: ``[..., nq]`` and ``[..., nv]`` to ``[..., nq]``, the
        root rotation as ``q * exp(dq[3:6])`` (body frame), normalised.  Any float dtype; on the inputs' device."""
        if qpos.shape[-1] != self.model.nq or dq.shape[-1] != self.model.nv:
            raise ValueError(f"qpos must end in nq = {self.model.nq} and dq in nv = {self.model.nv}, got {tuple(qpos.shape)}, {tuple(dq.shape)}")
        lead = torch.broadcast_shapes(qpos.shape[:-1], dq.shape[:-1])
        qpos, dq = qpos.expand(lead + (self.model.nq,)), dq.expand(lead + (self.model.nv,))
        w = dq[..., 3:6]
        th = torch.linalg.vector_norm(w, dim=-1, keepdim=True)
        half = 0.5 * th
        k = torch.where(th > 0, torch.sin(half) / torch.where(th > 0, th, torch.ones_like(th)), torch.full_like(th, 0.5))
        ew, ev = torch.cos(half), k * w                                     # exp(w) = (cos |w|/2, sin |w|/2 w / |w|)
        a = qpos[..., 3:7]
        aw, av = a[..., :1], a[..., 1:]
        rw = aw * ew - (av * ev).sum(-1, keepdim=True)
        rv = aw * ev + ew * av + torch.linalg.cross(av, ev)
        r = torch.cat([rw, rv], dim=-1)
        r = r / torch.linalg.vector_norm(r, dim=-1, keepdim=True)
        return torch.cat([qpos[..., 0:3] + dq[..., 0:3], r, qpos[..., 7:] + dq[..., 6:]], dim=-1)

    def dynamics(self, qpos: torch.Tensor, qvel: Optional[torch.Tensor] = None, mass_matrix: bool = True, bias: bool = True,
                 jac_bodies: Optional[Sequence] = None):
        """Joint-space mass matrix, bias forces and body Jacobians at caller rows ``(qpos, qvel)``, as MuJoCo's ``mj_fullM(qM)``,
        ``qfrc_bias`` and ``mj_jacBody``.  Returns a dict with the outputs asked for:

        - ``qM`` ``[n, nv, nv]`` (``mass_matrix``): dense, armature on the diagonal, exactly symmetric;
        - ``qfrc_bias`` ``[n, nv]`` (``bias``, needs ``qvel``): Coriolis, centrifugal and gravity forces (``mj_rne`` at qacc = 0);
        - ``jacp`` / ``jacr`` ``[n, k, 3, nv]`` (``jac_bodies``: k robot body indices, 0 = root, or body names): the world-frame linear
          velocity of each body's origin (``xpos``) and its angular velocity per unit qvel; both are views of one ``[n, k, 6, nv]`` tensor.

        Root dofs follow the qvel convention: ``[0:3]`` world-frame translation, ``[3:6]`` rotation about the root body's axes.  Float32
        tensors on this batch's device, ``[n, nq]`` / ``[n, nv]``; any n on a one-shape batch, n == num_envs with per-env shapes (row i
        uses env i's shape).  Reads no env state and changes none; every handle kind (self-collision too) is supported."""
        m = self.model
        if bias and qvel is None:
            raise ValueError("bias=True needs qvel")
        (q,) = self._rows(("qpos", qpos, m.nq))
        (v,) = self._rows(("qvel", qvel, m.nv), n=q.shape[0], optional=True)
        bodies = [self._body("jac_bodies entries", b) for b in (jac_bodies if jac_bodies is not None else [])]
        n, f32 = q.shape[0], dict(dtype=torch.float32, device=self.device)
        out = {}
        if mass_matrix:
            out["qM"] = torch.empty(n, m.nv, m.nv, **f32)
        if bias:
            out["qfrc_bias"] = torch.empty(n, m.nv, **f32)
        jac = None
        if jac_bodies is not None:
            jac = torch.empty(n, len(bodies), 6, m.nv, **f32)
            out["jacp"], out["jacr"] = jac[:, :, :3], jac[:, :, 3:]
        if mass_matrix or bias or bodies:
            jb = np.ascontiguousarray(np.asarray(bodies, dtype=np.int32))
            self._check(self._L().smplsim_dynamics(self._h, _ptr(q), _ptr(v), n, _ptr(out.get("qM")), _ptr(out.get("qfrc_bias")),
                                                   C.c_void_p(jb.ctypes.data) if bodies else None, len(bodies),
                                                   _ptr(jac) if bodies else None, self._stream()))
            self.gpu_launches += 1
        return out

    def centroidal(self, qpos: torch.Tensor, qvel: Optional[torch.Tensor] = None, *, com: bool = True, velocity: bool = True, cmm: bool = True,
                   jac_com_bodies: Optional[Sequence] = None):
        """Centre of mass and centroidal momentum at caller rows ``(qpos, qvel)``, as MuJoCo's ``subtree_com``, ``mj_subtreeVel`` and
        ``mj_jacSubtreeCom``, plus the centroidal momentum matrix.  Row ``b`` of the per-body outputs is body ``b``'s subtree; row 0 (the
        root's) is the whole robot.  Returns a dict with the outputs asked for:

        - ``subtree_com`` ``[n, nbody, 3]`` (``com``): the world-frame centre of mass of each subtree;
        - ``subtree_linvel`` / ``subtree_angmom`` ``[n, nbody, 3]`` (``velocity``, needs ``qvel``): its velocity, and the subtree's angular
          momentum about it;
        - ``cmm`` ``[n, 6, nv]`` (``cmm``): the centroidal momentum matrix, linear momentum (rows 0-2) over angular momentum about the
          whole-body centre of mass (rows 3-5) per unit qvel, so ``cmm @ qvel = [m subtree_linvel[:, 0] ; subtree_angmom[:, 0]]``;
        - ``cmm_bias`` ``[n, 6]`` (``cmm`` and ``velocity``): the momentum rate at qacc = 0 without gravity, so that the rate at any qacc is
          ``cmm @ qacc + cmm_bias`` (Newton-Euler: ``[m g + sum of external forces ; their torques about the centre of mass]``);
        - ``jac_com`` ``[n, k, 3, nv]`` (``jac_com_bodies``: k robot body indices, 0 = root, or body names): the velocity of each listed
          body's subtree centre of mass per unit qvel.

        Root dofs follow the qvel convention: ``[0:3]`` world-frame translation, ``[3:6]`` rotation about the root body's axes.  No
        output depends on gravity; per-env mass scales (``set_env_params``) are taken.  Float32 tensors on this batch's device, ``[n, nq]``
        / ``[n, nv]``; any n on a one-shape batch without per-env parameters, n == num_envs otherwise (row i uses env i's shape and
        parameters).  Reads no env state and changes none; every handle kind (self-collision too) is supported."""
        m = self.model
        if velocity and qvel is None:
            raise ValueError("velocity=True needs qvel")
        (q,) = self._rows(("qpos", qpos, m.nq))
        (v,) = self._rows(("qvel", qvel, m.nv), n=q.shape[0], optional=True)
        bodies = [self._body("jac_com_bodies entries", b) for b in (jac_com_bodies if jac_com_bodies is not None else [])]
        n, f32 = q.shape[0], dict(dtype=torch.float32, device=self.device)
        out = {}
        if com:
            out["subtree_com"] = torch.empty(n, m.nbody, 3, **f32)
        if velocity:
            out["subtree_linvel"] = torch.empty(n, m.nbody, 3, **f32)
            out["subtree_angmom"] = torch.empty(n, m.nbody, 3, **f32)
        if cmm:
            out["cmm"] = torch.empty(n, 6, m.nv, **f32)
            if velocity:
                out["cmm_bias"] = torch.empty(n, 6, **f32)
        if jac_com_bodies is not None:
            out["jac_com"] = torch.empty(n, len(bodies), 3, m.nv, **f32)
        if com or velocity or cmm or bodies:
            jb = np.ascontiguousarray(np.asarray(bodies, dtype=np.int32))
            self._check(self._L().smplsim_centroidal(self._h, _ptr(q), _ptr(v), n, _ptr(out.get("subtree_com")), _ptr(out.get("subtree_linvel")),
                                                     _ptr(out.get("subtree_angmom")), _ptr(out.get("cmm")), _ptr(out.get("cmm_bias")),
                                                     C.c_void_p(jb.ctypes.data) if bodies else None, len(bodies),
                                                     _ptr(out["jac_com"]) if bodies else None, self._stream()))
            self.gpu_launches += 1
        return out

    def _body(self, what, b):
        """``ModelDesc.body_index`` of ``b`` checked against [0, nbody); ``what`` names the argument in the messages."""
        rule = f"{what} must be body names or indices in [0, {self.model.nbody})"
        i = self.model.body_index(b, rule)
        if not 0 <= i < self.model.nbody:
            raise ValueError(f"{rule}, got {b!r}")
        return i

    RNE_POST_MAX_SITES = 64

    def _imu_sites(self, imu_sites):
        """(site_body int32 [k], site_pos float32 [k, 3], site_quat float32 [k, 4]) of ``rne_post``'s ``imu_sites``."""
        m = self.model
        if isinstance(imu_sites, str):
            if imu_sites != "bodies":
                raise ValueError(f"imu_sites must be 'bodies' or a sequence of (body, pos, quat), got {imu_sites!r}")
            imu_sites = [(b, (0.0, 0.0, 0.0), (1.0, 0.0, 0.0, 0.0)) for b in range(m.nbody)]
        sites = list(imu_sites)
        if len(sites) > self.RNE_POST_MAX_SITES:
            raise ValueError(f"at most {self.RNE_POST_MAX_SITES} imu_sites, got {len(sites)}")
        sb, sp, sq = [], [], []
        for s in sites:
            if not isinstance(s, (tuple, list)) or len(s) != 3:
                raise ValueError(f"imu_sites entries must be (body name or index, pos[3], quat[4]), got {s!r}")
            b, p, q = s
            b = self._body("imu_sites bodies", b)
            p, q = np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64)
            if p.shape != (3,) or not np.all(np.isfinite(p)):
                raise ValueError(f"imu_sites pos must be 3 finite numbers, got {s[1]!r}")
            if q.shape != (4,) or not abs(float(np.linalg.norm(q)) - 1.0) <= 1e-3:
                raise ValueError(f"imu_sites quat must be a unit quaternion (w, x, y, z), got {s[2]!r}")
            sb.append(b); sp.append(p); sq.append(q)
        return (np.ascontiguousarray(np.asarray(sb, dtype=np.int32)), np.ascontiguousarray(np.asarray(sp, dtype=np.float32).reshape(-1, 3)),
                np.ascontiguousarray(np.asarray(sq, dtype=np.float32).reshape(-1, 4)))

    def rne_post(self, qpos: torch.Tensor, qvel: torch.Tensor, qacc: torch.Tensor, *, acc: bool = True, joint_wrench: bool = True,
                 imu_sites=None, xfrc_applied: Optional[torch.Tensor] = None):
        """Body accelerations, joint reaction wrenches and IMU readings at caller rows ``(qpos, qvel, qacc)``, as MuJoCo's
        ``mj_rnePostConstraint`` (``cacc``, ``cfrc_int``) and its acceleration-stage sensors.  Returns a dict with the outputs asked for
        (world frame, robot body order):

        - ``body_acc`` ``[n, nbody, 6]`` (``acc``): the linear acceleration of each body origin (``xpos``; gravity not included), then
          its angular acceleration;
        - ``joint_wrench`` ``[n, nbody, 6]`` (``joint_wrench``): the force, then the torque about the body origin, that body b's parent
          (the world, for the root) applies to b's subtree through b's joint -- the joint's reaction load, joint-limit forces included;
        - ``accelerometer`` / ``gyro`` / ``force`` / ``torque`` ``[n, k, 3]`` (``imu_sites``): per site, in the site frame, the proper
          acceleration ``R^T (a - g)`` (``+|g|`` upward at rest, zero in free fall), the angular velocity, and the joint wrench of the
          site's body moved to the site (MuJoCo's sensors of those names).  ``imu_sites`` is a sequence of at most 64
          ``(body name or index, pos[3], quat[4])``, position and unit quaternion (w, x, y, z) in the body frame, or ``"bodies"``: one
          site at every body frame.

        The floor-contact and joint-limit forces are ``inverse``'s at the same rows; ``xfrc_applied`` (``[n, nbody, 6]``, the
        convention of ``self.xfrc_applied``; None: none) acts on the bodies as well.  Float32 tensors on this batch's device; any n on a
        one-shape batch without per-env parameters, n == num_envs otherwise (row i uses env i's shape, gravity and mass scales).  Reads no
        env state and changes none.  Not available with ``cfg.env.self_collision``."""
        m = self.model
        q, v, a = self._rows(("qpos", qpos, m.nq), ("qvel", qvel, m.nv), ("qacc", qacc, m.nv))
        n, f32 = q.shape[0], dict(dtype=torch.float32, device=self.device)
        xf = self._checked("xfrc_applied", xfrc_applied, (n, m.nbody, 6), optional=True)
        sb, sp, sq = self._imu_sites(imu_sites) if imu_sites is not None else (None, None, None)
        ns = 0 if sb is None else len(sb)
        out = {}
        if acc:
            out["body_acc"] = torch.empty(n, m.nbody, 6, **f32)
        if joint_wrench:
            out["joint_wrench"] = torch.empty(n, m.nbody, 6, **f32)
        if ns:
            for k in ("accelerometer", "gyro", "force", "torque"):
                out[k] = torch.empty(n, ns, 3, **f32)
        if out:
            hp = (lambda x: C.c_void_p(x.ctypes.data) if ns else None)
            self._check(self._L().smplsim_rne_post(self._h, _ptr(q), _ptr(v), _ptr(a), _ptr(xf), n, _ptr(out.get("body_acc")),
                                                   _ptr(out.get("joint_wrench")), hp(sb), hp(sp), hp(sq), ns, _ptr(out.get("accelerometer")),
                                                   _ptr(out.get("gyro")), _ptr(out.get("force")), _ptr(out.get("torque")), self._stream()))
            self.gpu_launches += 1
        return out

    # ------------------------------------------------------------------ ray casting and cameras (mj_ray, mujoco.Renderer)
    def _poses(self, xpos, xquat):
        """Body poses of the call: the batch's own post-step xpos / xquat by default."""
        if (xpos is None) != (xquat is None):
            raise ValueError("give both xpos and xquat, or neither (the batch's own poses)")
        if xpos is None:
            return self.xpos, self.xquat
        nb = self.model.nbody
        self._checked("xpos", xpos, (None, nb, 3))
        self._checked("xquat", xquat, (xpos.shape[0], nb, 4))
        return xpos, xquat

    def ray(self, pnt: torch.Tensor, vec: torch.Tensor, xpos: Optional[torch.Tensor] = None, xquat: Optional[torch.Tensor] = None,
            flg_static: bool = True, bodyexclude: int = -1):
        """``mujoco.mj_ray`` for every ray of every row: ``pnt`` / ``vec`` ``[n, R, 3]`` against the robot geoms (and the floor with
        ``flg_static``) posed by ``xpos [n, nbody, 3]`` / ``xquat [n, nbody, 4]`` (default: this batch's post-step poses).  Returns
        ``dist [n, R]`` (the hit is at ``pnt + dist * vec``; vec need not be unit) and ``geomid [n, R]`` (0 floor, i + 1 robot geom i),
        -1 / -1 for no hit.  ``bodyexclude`` (-1 none) skips that robot body's geoms.  Any n on a one-shape batch, n == num_envs with
        per-env shapes.  Writes no env state."""
        xpos, xquat = self._poses(xpos, xquat)
        n = xpos.shape[0]
        self._checked("pnt", pnt, (n, None, 3))
        self._checked("vec", vec, (n, pnt.shape[1], 3))
        R = pnt.shape[1]
        dist = torch.empty(n, R, dtype=torch.float32, device=self.device)
        gid = torch.empty(n, R, dtype=torch.int32, device=self.device)
        if n and R:
            self._check(self._L().smplsim_ray(self._h, _ptr(xpos), _ptr(xquat), n, R, _ptr(pnt), _ptr(vec), int(bool(flg_static)),
                                              int(bodyexclude), _ptr(dist), _ptr(gid), self._stream()))
            self.gpu_launches += 1
        return {"dist": dist, "geomid": gid}

    def render(self, camera: Any = "side", width: int = 320, height: int = 240, depth: bool = False, segmentation: bool = False,
               rgb: bool = True, xpos: Optional[torch.Tensor] = None, xquat: Optional[torch.Tensor] = None,
               geom_rgb: Optional[Sequence] = None):
        """One image per row from ``camera`` (a name of ``smplsim_b200.camera``: ``"back"``, ``"side"``, ``"front_side"``, their ids
        0-2, ``"egocentric"``; or a ``camera.Camera``) of the robot posed by ``xpos`` / ``xquat`` (default: this batch's post-step
        poses).  Returns a dict with the outputs asked for: ``depth [n, H, W]`` float32 z-depth in metres (the camera's zfar where
        nothing is hit), ``segmentation [n, H, W]`` int32 MuJoCo geom ids (0 floor, i + 1 robot geom i, -1 none), ``rgb [n, H, W, 3]``
        uint8.  Row 0 is the top of the image.  ``geom_rgb``: ``[ngeom, 3]`` albedo of the robot geoms (default 0.8 0.6 0.4).  The
        shading is this project's, stated in include/smplsim.h; it is not MuJoCo's OpenGL renderer.  Writes no env state."""
        from . import camera as _cam
        if isinstance(camera, (str, int, np.integer)) and not isinstance(camera, bool):
            key = (type(camera).__name__, camera)
            if key not in self._cams:
                self._cams[key] = _cam.named(self.model, camera)
            cam = self._cams[key]
        else:
            cam = _cam.named(self.model, camera)
        xpos, xquat = self._poses(xpos, xquat)
        n, f32 = xpos.shape[0], dict(device=self.device)
        if int(width) <= 0 or int(height) <= 0:
            raise ValueError(f"width and height must be positive, got {width} x {height}")
        H, W = int(height), int(width)
        out = {}
        if depth:
            out["depth"] = torch.empty(n, H, W, dtype=torch.float32, **f32)
        if segmentation:
            out["segmentation"] = torch.empty(n, H, W, dtype=torch.int32, **f32)
        if rgb:
            out["rgb"] = torch.empty(n, H, W, 3, dtype=torch.uint8, **f32)
        if not out:
            raise ValueError("render: ask for at least one of depth / segmentation / rgb")
        tab = None
        if geom_rgb is not None:
            tab = np.ascontiguousarray(np.asarray(geom_rgb, dtype=np.float32))
            if tab.shape != (self.model.ngeom, 3):
                raise ValueError(f"geom_rgb must have shape ({self.model.ngeom}, 3), got {tab.shape}")
        if n:
            cs = cam.c_struct()
            self._check(self._L().smplsim_render(self._h, _ptr(xpos), _ptr(xquat), n, C.byref(cs), W, H,
                                                 C.c_void_p(tab.ctypes.data) if tab is not None else None, _ptr(out.get("depth")),
                                                 _ptr(out.get("segmentation")), _ptr(out.get("rgb")), self._stream()))
            self.gpu_launches += 1
        return out

    def self_obs(self, version: int, xpos, xquat, qvel=None, linvel=None, angvel=None):
        def prep(t):
            return None if t is None else t.to(self.device, torch.float32).contiguous()
        xpos, xquat, qvel, linvel, angvel = map(prep, (xpos, xquat, qvel, linvel, angvel))
        n, nb = xpos.shape[0], self.model.nbody
        dim = (1 if self.envcfg.root_height_obs else 0) + 3 * (nb - 1) + 6 * nb + (6 + self.model.nu if version == 1 else 6 * nb)
        obs = torch.empty(n, dim, dtype=torch.float32, device=self.device)
        self._check(self._L().smplsim_self_obs(self._h, version, _ptr(qvel), _ptr(xpos), _ptr(xquat), _ptr(linvel), _ptr(angvel),
                                               _ptr(obs), n, self._stream()))
        self.gpu_launches += 1
        return obs

    def set_state(self, qpos: torch.Tensor, qvel: torch.Tensor):
        """Write qpos/qvel (and mark them as the last-forward state, as mj_forward would)."""
        self.qpos.copy_(qpos.to(self.device, torch.float32))
        self.qvel.copy_(qvel.to(self.device, torch.float32))
        self.qpos_fwd.copy_(self.qpos)
        self.qvel_fwd.copy_(self.qvel)

    def smem_bytes_per_env(self):
        return self._L().smplsim_smem_bytes_per_env(self._h)

    @property
    def kernel_version(self) -> int:
        """5: lane-chain kernels (csrc/lane_kernels.cuh)."""
        return self._L().smplsim_kernel_version(self._h)

    @property
    def schedule_steps(self) -> int:
        return self._L().smplsim_schedule_steps(self._h)


class GymVectEnvB200:
    """``GymVectEnv`` (smpl_sim/envs/nv/gymwrapper.py:7-65) over a HumanoidBatchB200: gymnasium-vector style
    ``reset`` / ``step`` with autoreset and ``info["final_observation"]``."""

    def __init__(self, env: HumanoidBatchB200, clip_observations: float = float(np.inf)):
        self._env = env
        self._clip_obs = clip_observations
        self.single_observation_shape = (env.num_obs,)
        self.single_action_shape = (env.num_actions,)

    @property
    def num_envs(self) -> int:
        return self._env.num_envs

    def _get_clipped_obs(self):
        return torch.clamp(self._env.obs_buf, -self._clip_obs, self._clip_obs)

    def reset(self, seed=None, options=None):
        self._env.reset(None)
        return self._get_clipped_obs().clone(), {}

    def close(self):
        pass

    def step(self, actions):
        env = self._env
        env.step(actions)
        obs = self._get_clipped_obs().clone()
        reward = env.rew_buf.clone()
        terminated = env.terminate_buf.bool()
        truncated = env.truncate_buf.bool()
        done = env.reset_buf.clone()
        env.reset(done)                         # masked, in-stream; no host sync
        info = {"terminate": terminated, "final_observation": obs, "_final_observation": done.bool()}
        return self._get_clipped_obs().clone(), reward, terminated, truncated, info
