"""Single-env gymnasium protocol (boundary B1, SURVEY.md 8b): what ``smpl_sim/run.py``'s loop talks to
(``Agent.sample_worker``, smpl_sim/agents/agent.py:64-109) -- the API of ``BaseEnv`` / ``HumanoidEnv`` /
``HumanoidTask`` (smpl_sim/envs/base_env.py:64-110, humanoid_env.py:148-184,455-469, humanoid_task.py) backed by a
``num_envs=1`` CUDA handle.  numpy in, numpy out; there is no CPU fallback.

A CUDA context does not survive ``fork()`` (agent.py:130-133 forks its samplers), so use ``num_threads=1`` with these
classes, or the batched surface (``smplsim_b200.batched``) for real throughput.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Optional

import numpy as np
import torch

from .batched import HumanoidBatchB200

try:                                     # gymnasium is optional in this image
    import gymnasium as _gym
    _Box = _gym.spaces.Box
    _EnvBase = _gym.Env
except Exception:                        # pragma: no cover - minimal stand-ins with the attributes the agents read
    _gym = None

    class _Box:                          # noqa: D401
        def __init__(self, low, high, dtype=np.float32):
            self.low, self.high, self.dtype = np.asarray(low, dtype=dtype), np.asarray(high, dtype=dtype), dtype
            self.shape = self.low.shape

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

        def sample(self):
            return np.random.uniform(np.maximum(self.low, -1e3), np.minimum(self.high, 1e3)).astype(self.dtype)

    class _EnvBase:
        pass


class _Contacts:
    """``mj_data.contact.geom1 / geom2`` of the last forward pass (floor contacts only; floor = geom 0)."""

    def __init__(self, mask: int):
        g2 = [g for g in range(1, 64) if (mask >> g) & 1]
        self.geom2 = np.asarray(g2, dtype=np.int32)
        self.geom1 = np.zeros_like(self.geom2)


def _dof_tree(m):
    """MuJoCo's ``dof_parentid``, ``dof_Madr`` and ``nM`` for the model: the compressed ``qM`` holds, for each dof i in turn,
    ``M[i, i]`` followed by ``M[i, j]`` for each ancestor dof j, nearest first."""
    par = np.full(m.nv, -1, dtype=np.int32)
    for b in range(m.nbody):
        d0, nd, p = int(m.body_dofadr[b]), int(m.body_dofnum[b]), int(m.body_parent[b])
        par[d0] = -1 if p < 0 else int(m.body_dofadr[p] + m.body_dofnum[p] - 1)
        par[d0 + 1:d0 + nd] = np.arange(d0, d0 + nd - 1)
    adr = np.zeros(m.nv, dtype=np.int32)
    n = 0
    for i in range(m.nv):
        adr[i] = n
        j = i
        while j >= 0:
            n += 1
            j = par[j]
    return par, adr, n


def _pairs(parentid):
    """(i, j) in qM order: every dof i with itself and its ancestors."""
    for i in range(len(parentid)):
        j = i
        while j >= 0:
            yield i, j
            j = parentid[j]


def mj_fullM(model, dst, qM):
    """``mujoco.mj_fullM``: expand the compressed ``qM`` (``model.dof_Madr`` layout) into the dense symmetric ``dst`` [nv, nv], in place."""
    nv = model.nv
    d = dst.reshape(nv * nv)
    d[:] = 0.0
    for k, (i, j) in enumerate(_pairs(model.dof_parentid)):
        d[i * nv + j] = d[j * nv + i] = qM[k]


def mjd_transitionFD(model, data, eps, flg_centered, A, B, C, D):
    """``mujoco.mjd_transitionFD`` for an env's ``mj_data``: finite-difference ``A = dx'/dx`` [2nv, 2nv] and ``B = dx'/du`` [2nv, nu]
    of one simulation substep at the data's ``qpos`` / ``qvel`` / ``ctrl``, written into ``A`` / ``B`` in place (either may be None).
    ``eps`` is the perturbation of every qpos, qvel and ctrl entry, as in MuJoCo; ``flg_centered`` selects centered differences.  The
    computation is fp32 on the GPU: MuJoCo's usual ``eps = 1e-6`` is rounding noise there, and ``eps = None`` takes the measured
    defaults of ``HumanoidBatchB200.transition_fd`` (1e-2 on qpos, 1e-1 on qvel, 1 N m on ctrl).  Sensor derivatives ``C`` / ``D`` are
    not computed: pass None for both.  ``model`` is accepted for the signature and not read."""
    if C is not None or D is not None:
        raise NotImplementedError("mjd_transitionFD: sensor derivatives (C, D) are not computed; pass None")
    a, b = data._fd_fn(data.qpos, data.qvel, data.ctrl, eps, bool(flg_centered))
    if A is not None:
        A[...] = a.reshape(np.shape(A))
    if B is not None:
        B[...] = b.reshape(np.shape(B))


def mjd_inverseFD(model, data, eps, flg_actuation, DfDq, DfDv, DfDa, DsDq, DsDv, DsDa, DmDq):
    """``mujoco.mjd_inverseFD`` for an env's ``mj_data``: finite-difference derivatives of the inverse dynamics ``qfrc_inverse`` at the
    data's ``qpos`` / ``qvel`` / ``qacc``, written into ``DfDq`` / ``DfDv`` / ``DfDa`` [nv, nv] in place (each may be None) in MuJoCo's
    transposed layout: ``DfDq[j, i] = d qfrc_inverse_i / d q_j`` (root rotation tangent in the body frame).  ``eps`` is the
    perturbation of every qpos, qvel and qacc entry, as in MuJoCo; the differences are centered.  The computation is fp32 on the GPU:
    MuJoCo's usual ``eps = 1e-6`` is rounding noise there, and ``eps = None`` takes the measured defaults of
    ``HumanoidBatchB200.inverse_fd`` (1e-3 on qpos, 1e-2 on qvel, 1 on qacc).  ``flg_actuation`` (subtract ``qfrc_actuator``) is
    accepted and changes nothing: this model's motor forces depend on ``ctrl`` only, so their derivatives by qpos, qvel and qacc are
    zero.  Sensor derivatives ``DsDq`` / ``DsDv`` / ``DsDa`` and ``DmDq`` are not computed: pass None.  ``model`` is accepted for the
    signature and not read."""
    if DsDq is not None or DsDv is not None or DsDa is not None or DmDq is not None:
        raise NotImplementedError("mjd_inverseFD: sensor derivatives (DsDq, DsDv, DsDa) and DmDq are not computed; pass None")
    dfrc = data._invfd_fn(data.qpos, data.qvel, data.qacc, eps)
    nv = dfrc.shape[0]
    for k, out in enumerate((DfDq, DfDv, DfDa)):
        if out is not None:
            out[...] = dfrc[:, k * nv:(k + 1) * nv].T.reshape(np.shape(out))


def rollout(model, data, initial_state, control, nstep=None):
    """``mujoco.rollout.rollout`` for an env's ``mj_data`` [MJ-upstream signature, not checked against a wheel]: ``nroll`` rollouts
    of ``nstep`` ``mj_step`` calls each, one per control row, from caller states, in one kernel launch per row (the env's handle holds
    one env).  ``initial_state`` is ``[nroll, 1 + nq + nv]`` (or one ``[1 + nq + nv]`` state for every row): ``[time, qpos, qvel]``,
    MuJoCo's ``mjSTATE_FULLPHYSICS`` layout for this model, which has no activations or plugins.  ``control`` is ``[nroll, nstep,
    nu]`` (or ``[nstep, nu]`` for every row): raw joint torques as ``data.ctrl`` holds them, not clamped.  Returns ``(state,
    sensordata)`` as MuJoCo does: ``state [nroll, nstep, 1 + nq + nv]`` after each step (time advanced by ``model.opt.timestep``
    per step), and ``sensordata [nroll, nstep, 0]``: sensors are not evaluated.  Each row starts from empty warm start and working-set
    memory; fp32 on the GPU.  ``model`` is accepted for the signature; ``data``'s own state is neither read nor changed."""
    return data._rollout_fn(initial_state, control, nstep)


def mj_differentiatePos(model, qvel, dt, qpos1, qpos2):
    """``mujoco.mj_differentiatePos``: ``qvel = (qpos2 (-) qpos1) / dt`` in place, fp64, for this model's joints (one free root joint,
    then hinges).  The root rotation is ``mju_subQuat``: ``log(normalise(q1)^-1 * normalise(q2))`` on the shortest arc, in ``q1``'s
    body frame -- the tangent of ``mjd_transitionFD`` and of ``HumanoidBatchB200.rollout``'s feedback law.  ``model`` is accepted
    for the signature (the layout follows from the lengths)."""
    q1, q2 = np.asarray(qpos1, dtype=np.float64).ravel(), np.asarray(qpos2, dtype=np.float64).ravel()
    b, c = q1[3:7] / np.linalg.norm(q1[3:7]), q2[3:7] / np.linalg.norm(q2[3:7])
    rw = b[0] * c[0] + b[1:] @ c[1:]
    rv = b[0] * c[1:] - c[0] * b[1:] - np.cross(b[1:], c[1:])
    if rw < 0:
        rw, rv = -rw, -rv
    s = np.linalg.norm(rv)
    d = np.concatenate([q2[0:3] - q1[0:3], rv * (2 * np.arctan2(s, rw) / s) if s > 0 else np.zeros(3), q2[7:] - q1[7:]])
    qvel.reshape(-1)[:] = d / dt


def mj_integratePos(model, qpos, qvel, dt):
    """``mujoco.mj_integratePos``: ``qpos <- qpos (+) qvel dt`` in place, fp64; the root rotation as ``q * exp(qvel[3:6] dt)`` (body
    frame), normalised.  The inverse of ``mj_differentiatePos``.  ``model`` is accepted for the signature."""
    q = qpos.reshape(-1)
    d = np.asarray(qvel, dtype=np.float64).ravel() * dt
    w = d[3:6]
    th = np.linalg.norm(w)
    e = np.concatenate([[np.cos(th / 2)], np.sin(th / 2) / th * w if th > 0 else np.zeros(3)])
    a = q[3:7].astype(np.float64)
    r = np.concatenate([[a[0] * e[0] - a[1:] @ e[1:]], a[0] * e[1:] + e[0] * a[1:] + np.cross(a[1:], e[1:])])
    q[0:3] += d[0:3]
    q[3:7] = r / np.linalg.norm(r)
    q[7:] += d[6:]


def mj_subtreeVel(model, data):
    """``mujoco.mj_subtreeVel`` for an env's ``mj_data``: fills ``data.subtree_linvel`` and ``data.subtree_angmom`` [nbody + 1, 3]
    (MuJoCo body order; row 0, the world's subtree, is the whole robot's), the velocity of each subtree's centre of mass and the
    subtree's angular momentum about it, at the state of the last forward pass as ``subtree_com``.  fp32 on the GPU
    (``HumanoidBatchB200.centroidal``).  ``model`` is accepted for the signature and not read."""
    c = data._cent()
    data.subtree_linvel = c["subtree_linvel"].copy()
    data.subtree_angmom = c["subtree_angmom"].copy()


def mj_jacSubtreeCom(model, data, jacp, body):
    """``mujoco.mj_jacSubtreeCom`` for an env's ``mj_data``: the [3, nv] Jacobian of the centre of mass of MuJoCo body ``body``'s
    subtree (0 = world: the whole robot) at the state of the last forward pass, written into ``jacp`` in place (any shape of 3 nv
    entries).  fp32 on the GPU.  ``model`` is accepted for the signature and not read."""
    nb = data._cent()["subtree_com"].shape[0]
    if isinstance(body, bool) or not isinstance(body, (int, np.integer)) or not 0 <= int(body) < nb:
        raise ValueError(f"body must be a MuJoCo body id in [0, {nb}), got {body!r}")
    jac = data._jac_com_fn(max(int(body) - 1, 0))
    jacp.reshape(jac.size)[:] = jac.ravel()


def mj_rnePostConstraint(model, data):
    """``mujoco.mj_rnePostConstraint`` for an env's ``mj_data``: fills ``data.cacc``, ``data.cfrc_int`` and ``data.cfrc_ext``
    [nbody + 1, 6] in MuJoCo's layout (MuJoCo body order, world row first; rotation first; com-based, i.e. about the root subtree's
    centre of mass ``subtree_com[0]``): each body's spatial acceleration with the ``-g`` offset MuJoCo carries (the world row is
    ``[0 ; -g]``), the wrench its parent applies through its joint, and the external wrench on it (contact forces plus
    ``xfrc_applied``).  Evaluated at the last forward pass (``qpos_fwd``, ``qvel_fwd``, ``data.qacc``) with the env's
    ``xfrc_applied``; fp32 on the GPU (``HumanoidBatchB200.rne_post``), converted on the host.  ``model`` is accepted for the signature
    and not read."""
    r = data._rnep_fn()
    data.cacc, data.cfrc_int, data.cfrc_ext = r["cacc"], r["cfrc_int"], r["cfrc_ext"]


class _MjData(SimpleNamespace):
    """``mj_data`` view.  ``qM`` / ``qfrc_bias`` and ``subtree_com`` cost a kernel call, so they are evaluated on first read."""

    @property
    def subtree_com(self):
        return self._cent()["subtree_com"]

    def _cent(self):
        if "_cent_val" not in self.__dict__:
            self._cent_val = self._cent_fn()
        return self._cent_val

    @property
    def qM(self):
        return self._dyn()[0]

    @property
    def qfrc_bias(self):
        return self._dyn()[1]

    def _dyn(self):
        if "_dyn_val" not in self.__dict__:
            self._dyn_val = self._dyn_fn()
        return self._dyn_val


class HumanoidEnvB200(_EnvBase):
    metadata = {"render_modes": ["human", "rgb_array"], "render_fps": 30}
    TASK = None

    def __init__(self, cfg: Any, device: str = "cuda:0"):
        self.cfg = cfg
        if self.TASK is not None and cfg.env.get("task", self.TASK) != self.TASK:
            raise ValueError(f"{type(self).__name__} expects cfg.env.task == {self.TASK!r}")
        e = cfg.env
        # BaseEnv.__init__ (base_env.py:23-49)
        self.clip_actions = e.clip_actions
        self.render_mode = e.render_mode
        assert self.render_mode is None or self.render_mode in self.metadata["render_modes"]
        self.headless = cfg.headless
        self.sim_timestep_inv = e.sim_timestep_inv
        self.sim_timestep = 1.0 / self.sim_timestep_inv
        self.control_freq_inv = e.control_frequency_inv
        self.cur_t = 0
        self.dt = self.sim_timestep * self.control_freq_inv
        self.paused = False
        self.disable_reset = False
        self.viewer = None
        self.renderer = None
        self.dtype = np.float32
        self._b = self._make_batch(cfg, device)
        m = self._b.model
        # mj_data.xfrc_applied: one persistent array in MuJoCo indexing (row 0 = world, no effect), so that
        # env.mj_data.xfrc_applied[body_id] = (fx, fy, fz, tx, ty, tz) works as it does on an MjData
        self._xfrc_applied = np.zeros((m.nbody + 1, 6))
        self._xfrc_dev = None
        self.control_mode = e.control_mode
        self.max_episode_length = e.episode_length
        self.self_obs_v = e.self_obs_v
        self.humanoid_type = cfg.robot.humanoid_type
        self.body_names_orig = list(m.body_names)
        self.mj_body_names = ["world"] + list(m.body_names)
        self.num_rigid_bodies = m.nbody
        self.dof_names = self.body_names_orig[1:]
        self.actuator_names = list(m.joint_names)
        self.dof_size = m.nu
        self.qpos_lim, self.qvel_lim = m.nq, m.nv
        self.contact_bodies = list(e.contact_bodies)
        self.contact_bodies_ids = [m.geom_names.index(n) + 1 for n in self.contact_bodies]
        self.floor_idx = 0
        self._dof_parentid, self._dof_Madr, self._nM = _dof_tree(m)
        self.jkp, self.jkd, self.torque_lim = m.act_kp.copy(), m.act_kd.copy(), m.act_torque_lim.copy()
        self._pd_action_scale, self._pd_action_offset = m.act_scale.copy(), m.act_offset.copy()
        self.observation_space = _Box(-np.inf * np.ones(self.get_obs_size(), dtype=np.float32),
                                      np.inf * np.ones(self.get_obs_size(), dtype=np.float32), dtype=np.float32)
        lim = np.ones(self.get_action_size(), dtype=np.float32) if self.clip_actions else np.inf * np.ones(self.get_action_size(), dtype=np.float32)
        self.action_space = _Box(-lim, lim, dtype=np.float32)
        self.np_random = np.random.default_rng(int(cfg.get("seed", 0)))
        self.reward_info = {}

    def _make_batch(self, cfg, device):
        """The num_envs=1 handle behind this env (CUDA; there is no CPU path)."""
        return HumanoidBatchB200(cfg, num_envs=1, device=device, seed=int(cfg.get("seed", 0)))

    # ------------------------------------------------------------------ sizes
    def get_action_size(self):
        return self._b.num_actions

    def get_obs_size(self):
        return self._b.num_obs

    # ------------------------------------------------------------------ gym API
    def seed(self, seed: Optional[int] = None):
        """BaseEnv.seed / gym reset(seed=): reseeds np_random AND the device-side task / Fall-init stream (Philox counter jump:
        the key stays (cfg.seed, env id), the per-env counter restarts from a value derived from `seed`)."""
        self.np_random = np.random.default_rng(seed)
        if seed is not None:
            self._b.rng_counter.fill_(int((int(seed) * 2654435761) & 0x7FFFFFFF))

    def reset(self, seed=None, options=None):
        if seed is not None:
            self.seed(seed)
        obs = self._b.reset().cpu().numpy()[0].astype(self.dtype)
        self.cur_t = 0
        return obs, {"critic_state": obs}

    def _upload_xfrc(self):
        """mj_data.xfrc_applied -> the batch's wrench tensor before a step: an all-zero array is no wrench (None)."""
        x = self._xfrc_applied[1:]
        if not np.any(x):
            self._b.xfrc_applied = None
            return
        if self._xfrc_dev is None:
            self._xfrc_dev = torch.zeros(1, self._b.model.nbody, 6, dtype=torch.float32, device=self._b.device)
        self._xfrc_dev.copy_(torch.as_tensor(x, dtype=torch.float32)[None])
        self._b.xfrc_applied = self._xfrc_dev

    def step(self, action):
        a = torch.as_tensor(np.asarray(action, dtype=np.float32)[None, : self.dof_size])
        self._upload_xfrc()
        obs, rew, term, trunc = self._b.step(a)
        obs = obs.cpu().numpy()[0].astype(self.dtype)
        self.cur_t = int(self._b.progress_buf[0].item())
        died, timed_out = bool(term[0].item()), bool(trunc[0].item())
        if self.disable_reset:
            died, timed_out = False, False
        info = dict(self.reward_info)
        info["critic_state"] = obs
        return obs, float(rew[0].item()), died, timed_out, info

    def render(self):
        """``render_mode == "rgb_array"`` and not ``headless``: the ``[240, 320, 3]`` uint8 frame of ``cfg.env.camera`` (a name of
        ``smplsim_b200.camera`` or a MuJoCo camera id 0-2: back, side, front_side) at the current state -- mujoco.Renderer's default
        size (base_env.py:159-162).  Every other configuration returns None: worker 0 calls this every step even when headless
        (agent.py:96-97)."""
        if self.render_mode != "rgb_array" or self.headless:
            return None
        frame = self._b.render(camera=self.cfg.env.camera, width=320, height=240)["rgb"]
        return frame[0].cpu().numpy()

    def close(self):
        pass

    # ------------------------------------------------------------------ mj_data-style views (examples poke env.mj_data)
    @property
    def mj_data(self):
        """``qM`` (compressed, ``mj_model.dof_Madr`` layout), ``qfrc_bias`` and ``subtree_com`` ([nbody + 1, 3], the world row the
        whole robot's) are those of the last forward pass, at ``(qpos_fwd, qvel_fwd)``, as on an MjData after ``mj_step``
        (``mj_kinematics`` does not refresh ``subtree_com``)."""
        b = self._b
        sens = np.concatenate([b.body_linvel[0].cpu().numpy().ravel(), b.body_angvel[0].cpu().numpy().ravel()])
        z3, z4 = np.zeros((1, 3)), np.array([[1.0, 0, 0, 0]])
        return _MjData(_dyn_fn=self._fwd_dynamics, _fd_fn=self._transition_fd, _rollout_fn=self._rollout, _invfd_fn=self._inverse_fd,
                               _cent_fn=self._centroidal, _jac_com_fn=self._jac_com, _rnep_fn=self._rne_post, qpos=b.qpos[0].cpu().numpy().astype(np.float64), qvel=b.qvel[0].cpu().numpy().astype(np.float64),
                               ctrl=b.ctrl[0].cpu().numpy().astype(np.float64), qacc=b.qacc[0].cpu().numpy().astype(np.float64),
                               xpos=np.concatenate([z3, b.xpos[0].cpu().numpy()]), xquat=np.concatenate([z4, b.xquat[0].cpu().numpy()]),
                               sensordata=sens, contact=_Contacts(int(b.contact_mask[0].item())),
                               xfrc_applied=self._xfrc_applied)

    @property
    def mj_model(self):
        """The MjModel attributes the reference reads (humanoid_env.py:262-289,325-370; utils/mujoco_utils.py): sizes, names, joint
        ranges, timestep.  Body / geom 0 is the world / floor, as in MuJoCo."""
        m = self._b.model
        rng = np.asarray(m.dof_range)
        names = ["world"] + list(m.body_names)
        joints = {n: SimpleNamespace(name=n, range=rng[6 + i].copy(), qposadr=np.array([7 + i]), dofadr=np.array([6 + i]))
                  for i, n in enumerate(m.joint_names)}
        return SimpleNamespace(nbody=m.nbody + 1, nq=m.nq, nv=m.nv, nu=m.nu, ngeom=len(m.geom_names) + 1, opt=SimpleNamespace(timestep=self.sim_timestep),
                               body=lambda i: SimpleNamespace(name=names[i], id=i), joint=lambda n: joints[n],
                               geom=lambda i: SimpleNamespace(name=(["floor"] + list(m.geom_names))[i], id=i),
                               body_mass=np.concatenate([[0.0], np.asarray(m.body_mass)]),
                               nM=self._nM, dof_Madr=self._dof_Madr.copy(), dof_parentid=self._dof_parentid.copy())

    def _fwd_dynamics(self):
        """(compressed qM, qfrc_bias) at the state of the last forward pass."""
        b = self._b
        out = b.dynamics(b.qpos_fwd, b.qvel_fwd)
        M = out["qM"][0].cpu().numpy().astype(np.float64)
        qM = np.array([M[i, j] for i, j in _pairs(self._dof_parentid)])
        return qM, out["qfrc_bias"][0].cpu().numpy().astype(np.float64)

    def _centroidal(self):
        """subtree_com, subtree_linvel, subtree_angmom [nbody + 1, 3] at the state of the last forward pass, world row first (fp64)."""
        b = self._b
        out = b.centroidal(b.qpos_fwd, b.qvel_fwd, cmm=False)
        return {k: np.concatenate([v[0, :1], v[0]]).astype(np.float64) for k, v in ((k, v.cpu().numpy()) for k, v in out.items())}

    def _jac_com(self, body):
        """jac_com [3, nv] of robot body ``body``'s subtree at the state of the last forward pass (fp64)."""
        b = self._b
        out = b.centroidal(b.qpos_fwd, None, com=False, velocity=False, cmm=False, jac_com_bodies=[body])
        return out["jac_com"][0, 0].cpu().numpy().astype(np.float64)

    def _rne_post(self):
        """cacc, cfrc_int, cfrc_ext [nbody + 1, 6] (MuJoCo's com-based layout, world row first) at the last forward pass (fp64)."""
        b = self._b
        m = b.model
        q, v, a = b.qpos_fwd, b.qvel_fwd, b.qacc
        xf = torch.as_tensor(self._xfrc_applied[1:], dtype=torch.float32, device=b.device)[None].contiguous()
        out = b.rne_post(q, v, a, xfrc_applied=xf)
        jac = b.dynamics(q, None, mass_matrix=False, bias=False, jac_bodies=list(range(m.nbody)))
        J = torch.cat([jac["jacp"], jac["jacr"]], 2)[0].cpu().numpy().astype(np.float64)
        vel = J @ v[0].cpu().numpy().astype(np.float64)                 # [nb, 6]: origin velocity, angular velocity
        c = b.centroidal(q, None, velocity=False, cmm=False)["subtree_com"][0, 0].cpu().numpy().astype(np.float64)
        xpos, xquat = (x[0].cpu().numpy().astype(np.float64) for x in b.kinematics(q))
        cw = b.inverse(q, v, a, contact_wrench=True)[1][0].cpu().numpy().astype(np.float64)
        g = b.env_params["gravity"][0].cpu().numpy().astype(np.float64)
        acc, jw = (out[k][0].cpu().numpy().astype(np.float64) for k in ("body_acc", "joint_wrench"))
        w, x, y, z = xquat.T / np.linalg.norm(xquat, axis=1)
        R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                      np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                      np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
        xipos = xpos + np.einsum("bij,bj->bi", R, np.asarray(m.body_ipos, dtype=np.float64))
        wb, wd = vel[:, 3:], acc[:, 3:]
        # spatial acceleration about the fixed point c: classical acceleration of the body origin + wd x (c - x) - w x v_origin
        lin = acc[:, :3] + np.cross(wd, c - xpos) - np.cross(wb, vel[:, :3]) - g
        f_ext = cw[:, :3] + xf[0, :, :3].cpu().numpy().astype(np.float64)
        t_ext = cw[:, 3:] + xf[0, :, 3:].cpu().numpy().astype(np.float64) + np.cross(xipos - c, f_ext)
        world = np.zeros((1, 6))
        return {"cacc": np.concatenate([np.concatenate([[0.0, 0.0, 0.0], -g])[None], np.concatenate([wd, lin], 1)]),
                "cfrc_int": np.concatenate([world, np.concatenate([jw[:, 3:] + np.cross(xpos - c, jw[:, :3]), jw[:, :3]], 1)]),
                "cfrc_ext": np.concatenate([world, np.concatenate([t_ext, f_ext], 1)])}

    def _fd_row(self, fd, x, eps, **kw):
        """The batch's ``fd`` (``transition_fd`` / ``inverse_fd``) at one state ``x`` (fp32 rows), eps (None: the defaults); fp64 outputs."""
        dv = self._b.device
        out = fd(*(torch.as_tensor(np.asarray(v, dtype=np.float32)[None], device=dv) for v in x), *(() if eps is None else (eps,) * 3), **kw)
        return {k: v[0].cpu().numpy().astype(np.float64) for k, v in out.items()}

    def _transition_fd(self, qpos, qvel, ctrl, eps, centered):
        """(A, B) of ``mjd_transitionFD`` at one state."""
        out = self._fd_row(self._b.transition_fd, (qpos, qvel, ctrl), eps, centered=centered)
        return out["A"], out["B"]

    def _inverse_fd(self, qpos, qvel, qacc, eps):
        """dfrc [nv, 3nv] of ``mjd_inverseFD`` at one state."""
        return self._fd_row(self._b.inverse_fd, (qpos, qvel, qacc), eps)["dfrc"]

    def _rollout(self, initial_state, control, nstep):
        """(state, sensordata) of ``rollout``: ctrl-mode rollouts of the given rows (fp32 on the device; fp64 copies of the result)."""
        b, m = self._b, self._b.model
        x0 = np.asarray(initial_state, dtype=np.float64)
        u = np.asarray(control, dtype=np.float64)
        x0 = x0[None] if x0.ndim == 1 else x0
        if x0.ndim != 2 or x0.shape[1] != 1 + m.nq + m.nv:
            raise ValueError(f"initial_state must have shape [nroll, {1 + m.nq + m.nv}] ([time, qpos, qvel]), got {np.shape(initial_state)}")
        u = np.broadcast_to(u[None], (x0.shape[0],) + u.shape) if u.ndim == 2 else u
        if u.ndim != 3 or u.shape[0] != x0.shape[0] or u.shape[2] != m.nu:
            raise ValueError(f"control must have shape [nroll, nstep, {m.nu}] or [nstep, {m.nu}], got {np.shape(control)}")
        if nstep is not None and nstep != u.shape[1]:
            raise ValueError(f"nstep = {nstep} does not match the {u.shape[1]} control rows")
        dev = lambda x: torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32), device=b.device)  # noqa: E731
        out = b.rollout(dev(x0[:, 1:1 + m.nq]), dev(x0[:, 1 + m.nq:]), dev(u), mode="ctrl", status=False)
        T = u.shape[1]
        time = x0[:, :1] + self.sim_timestep * np.arange(1, T + 1)[None]
        state = np.concatenate([time[..., None], out["qpos"].cpu().numpy().astype(np.float64), out["qvel"].cpu().numpy().astype(np.float64)], axis=2)
        return state, np.zeros((x0.shape[0], T, 0))

    def get_body_jac_by_id(self, id, jacp=None, jacr=None):
        """``mujoco.mj_jacBody`` at the current qpos for MuJoCo body id ``id`` (0 = world: zeros): the [3, nv] translational and
        rotational Jacobians of the body's frame origin.  Fills ``jacp`` / ``jacr`` in place when given (any shape of 3 nv entries);
        returns (jacp, jacr), new arrays where none were given."""
        nv = self._b.model.nv
        jp, jr = np.zeros((3, nv)), np.zeros((3, nv))
        if id != 0:
            out = self._b.dynamics(self._b.qpos, mass_matrix=False, bias=False, jac_bodies=[int(id) - 1])
            jp, jr = (out[k][0, 0].cpu().numpy().astype(np.float64) for k in ("jacp", "jacr"))
        if jacp is not None:
            jacp.reshape(3 * nv)[:] = jp.ravel()
        if jacr is not None:
            jacr.reshape(3 * nv)[:] = jr.ravel()
        return (jp if jacp is None else jacp), (jr if jacr is None else jacr)

    def get_body_jacp_by_name(self, name, jacp=None, jacr=None):
        """jacp [3, nv] of the named body (``jacr`` filled too when given)."""
        return self.get_body_jac_by_id(self.mj_body_names.index(name), jacp=jacp, jacr=jacr)[0]

    def get_body_xvelp(self, name):
        """World-frame linear velocity of the named body's origin: jacp . qvel."""
        return self.get_body_jacp_by_name(name).reshape(3, -1) @ self.get_qvel()

    def get_body_xvelr(self, name):
        """World-frame angular velocity of the named body: jacr . qvel."""
        return self.get_body_jac_by_id(self.mj_body_names.index(name))[1].reshape(3, -1) @ self.get_qvel()

    def get_qpos(self):
        return self._b.qpos[0].cpu().numpy().astype(np.float64)

    def get_qvel(self):
        return self._b.qvel[0].cpu().numpy().astype(np.float64)

    def get_body_xpos(self):
        return self._b.xpos[0].cpu().numpy().astype(np.float64)

    def get_body_xquat(self):
        return self._b.xquat[0].cpu().numpy().astype(np.float64)

    def get_body_xpos_by_id(self, body_id):
        return self.get_body_xpos()[body_id]

    def get_root_pos(self):
        return self.get_body_xpos()[0].copy()

    def compute_torque(self, ctrl):
        """Torque applied in the last substep for the last action (the reference recomputes it per substep)."""
        return self._b.ctrl[0].cpu().numpy().astype(np.float64)


class HumanoidSpeed(HumanoidEnvB200):
    TASK = "HumanoidSpeed"


class HumanoidReach(HumanoidEnvB200):
    TASK = "HumanoidReach"


class HumanoidGetup(HumanoidEnvB200):
    TASK = "HumanoidGetup"


def make_env(cfg: Any, device: str = "cuda:0"):
    """``eval(cfg.env.task)(cfg)`` of AgentHumanoid.setup_env (agents/agent_humanoid.py:91-92)."""
    return {"HumanoidEnv": HumanoidEnvB200, "HumanoidSpeed": HumanoidSpeed, "HumanoidReach": HumanoidReach,
            "HumanoidGetup": HumanoidGetup}[cfg.env.task](cfg, device=device)
