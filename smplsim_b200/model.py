"""ModelDesc: the constant tree / inertia / geom / gain table the stepper consumes.

This is the host-side replacement for ``mujoco.MjModel`` as far as the hot path
reads it (SURVEY.md section 8 a13) plus the controller constants the reference
derives in ``HumanoidEnv.build_pd_action_scale`` (smpl_sim/envs/humanoid_env.py:325-370)
from its ``GAINS["stablepd"]`` table (smpl_sim/envs/humanoid_env.py:62-84).

All arrays are float64 / int32 numpy; ``c_struct()`` exposes them to the C ABI
(include/smplsim.h: SmplsimModelDesc), which both the CUDA library and the CPU
oracle consume.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import mjcf as _mjcf
from .mjcf import GEOM_BOX, GEOM_CAPSULE, GEOM_PLANE, GEOM_SPHERE, ParsedMJCF, parse_mjcf

_ASSET_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets")

# [kp, kd, torque_lim] per SMPL joint -- the values of the reference's
# GAINS["stablepd"] table (smpl_sim/envs/humanoid_env.py:62-84; column 2, the
# gear, is always 1 and unused).  Keyed by joint-group so L_/R_ share a row.
_PD_GAINS = {
    "Hip": (800.0, 80.0, 1000.0), "Knee": (800.0, 80.0, 1000.0), "Ankle": (800.0, 80.0, 1000.0),
    "Toe": (500.0, 50.0, 500.0),
    "Torso": (1000.0, 100.0, 500.0), "Spine": (1000.0, 100.0, 500.0), "Chest": (1000.0, 100.0, 500.0),
    "Neck": (500.0, 50.0, 250.0), "Head": (500.0, 50.0, 250.0),
    "Thorax": (500.0, 50.0, 1000.0), "Shoulder": (500.0, 50.0, 1000.0),
    "Elbow": (500.0, 50.0, 250.0), "Wrist": (300.0, 30.0, 250.0), "Hand": (300.0, 30.0, 250.0),
}
# SMPL-X finger / jaw / eye joints are absent from the reference's table (the
# reference raises KeyError there, SURVEY.md 7.3-9); we use the GAINS_PHC finger
# row [100, 10, 1, 150] (smpl_sim/smpllib/skeleton_local.py:133-162).
_PD_GAINS_FALLBACK = (100.0, 10.0, 150.0)


def pd_gains_for_joint(joint_name: str):
    """kp, kd, torque_lim for an actuator joint called e.g. ``L_Hip_x``."""
    body = "_".join(joint_name.split("_")[:-1])           # humanoid_env.py:348
    key = body[2:] if body[:2] in ("L_", "R_") else body
    return _PD_GAINS.get(key, _PD_GAINS_FALLBACK)


def _skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=np.float64)


class SmplsimModelDescC(C.Structure):
    """ctypes mirror of include/smplsim.h: SmplsimModelDesc (keep in sync)."""
    _fields_ = [
        ("nbody", C.c_int32), ("nq", C.c_int32), ("nv", C.c_int32), ("nu", C.c_int32), ("ngeom", C.c_int32),
        ("body_parent", C.POINTER(C.c_int32)),
        ("body_dofadr", C.POINTER(C.c_int32)),
        ("body_dofnum", C.POINTER(C.c_int32)),
        ("body_pos", C.POINTER(C.c_double)),
        ("body_quat", C.POINTER(C.c_double)),
        ("body_mass", C.POINTER(C.c_double)),
        ("body_ipos", C.POINTER(C.c_double)),
        ("body_inertia", C.POINTER(C.c_double)),
        ("body_invweight0", C.POINTER(C.c_double)),
        ("dof_axis", C.POINTER(C.c_double)),
        ("dof_armature", C.POINTER(C.c_double)),
        ("dof_invweight0", C.POINTER(C.c_double)),
        ("dof_range", C.POINTER(C.c_double)),
        ("dof_limited", C.POINTER(C.c_int32)),
        ("geom_type", C.POINTER(C.c_int32)),
        ("geom_body", C.POINTER(C.c_int32)),
        ("geom_pos", C.POINTER(C.c_double)),
        ("geom_mat", C.POINTER(C.c_double)),
        ("geom_size", C.POINTER(C.c_double)),
        ("geom_legal", C.POINTER(C.c_int32)),
        ("plane_pos", C.c_double * 3),
        ("plane_normal", C.c_double * 3),
        ("margin", C.c_double),
        ("friction", C.c_double * 3),
        ("solref", C.c_double * 2),
        ("solimp", C.c_double * 5),
        ("impratio", C.c_double),
        ("timestep", C.c_double),
        ("gravity", C.c_double * 3),
        ("act_kp", C.POINTER(C.c_double)),
        ("act_kd", C.POINTER(C.c_double)),
        ("act_torque_lim", C.POINTER(C.c_double)),
        ("act_scale", C.POINTER(C.c_double)),
        ("act_offset", C.POINTER(C.c_double)),
        ("geom_contype", C.POINTER(C.c_int32)),
        ("geom_conaffinity", C.POINTER(C.c_int32)),
        ("nexclude", C.c_int32),
        ("exclude_pairs", C.POINTER(C.c_int32)),
    ]


@dataclass
class ModelDesc:
    body_names: List[str]
    joint_names: List[str]          # hinge joints in dof order (nu)
    geom_names: List[str]           # robot geoms; MuJoCo geom id = index + 1 (floor = 0)
    body_parent: np.ndarray         # [nb] int32, -1 for the root
    body_dofadr: np.ndarray         # [nb]
    body_dofnum: np.ndarray         # [nb]  (6 for the root)
    body_pos: np.ndarray            # [nb,3]
    body_quat: np.ndarray           # [nb,4] wxyz
    body_mass: np.ndarray           # [nb]
    body_ipos: np.ndarray           # [nb,3]
    body_inertia: np.ndarray        # [nb,6] xx yy zz xy xz yz, about COM, body frame
    body_invweight0: np.ndarray     # [nb,2]
    dof_axis: np.ndarray            # [nv,3] (rows 0..5 unused)
    dof_armature: np.ndarray        # [nv]
    dof_invweight0: np.ndarray      # [nv]
    dof_range: np.ndarray           # [nv,2] radians
    dof_limited: np.ndarray         # [nv] int32
    geom_type: np.ndarray
    geom_body: np.ndarray
    geom_pos: np.ndarray            # [ng,3]
    geom_mat: np.ndarray            # [ng,9]
    geom_size: np.ndarray           # [ng,3]
    geom_legal: np.ndarray          # [ng] int32: 1 if floor contact with this geom is legal
    plane_pos: np.ndarray
    plane_normal: np.ndarray
    margin: float
    friction: np.ndarray            # [3] contact friction after max-mixing with the floor
    solref: np.ndarray
    solimp: np.ndarray
    impratio: float
    timestep: float
    gravity: np.ndarray
    act_kp: np.ndarray
    act_kd: np.ndarray
    act_torque_lim: np.ndarray
    act_scale: np.ndarray
    act_offset: np.ndarray
    excludes: List[tuple]
    qpos0: np.ndarray
    geom_contype: Optional[np.ndarray] = None      # [ng] collision filter bits (only the oracle's opt-in self-collision reads them)
    geom_conaffinity: Optional[np.ndarray] = None

    # ------------------------------------------------------------------ sizes
    @property
    def nbody(self):
        return len(self.body_names)

    def body_index(self, body, rule: str, kind: str = "body") -> int:
        """The index of ``body``: a name in ``body_names``, or an integer, returned as an int without a range check (each caller checks
        [0, nbody) or leaves it to the C ABI).  Raises ``ValueError`` for an unknown name (``"unknown {kind} name ..."``) and for a bool
        or any other value (``"{rule}, got ..."``).  ``rule`` is the caller's statement of what its argument must be, naming the
        argument (``"jac_bodies entries must be body names or indices in [0, 24)"``); a range-checking caller raises it too."""
        if isinstance(body, str):
            if body not in self.body_names:
                raise ValueError(f"unknown {kind} name {body!r}")
            return list(self.body_names).index(body)
        if isinstance(body, bool) or not isinstance(body, (int, np.integer)):
            raise ValueError(f"{rule}, got {body!r}")
        return int(body)

    @property
    def nv(self):
        return int(self.dof_armature.shape[0])

    @property
    def nq(self):
        return self.nv + 1

    @property
    def nu(self):
        return self.nv - 6

    @property
    def ngeom(self):
        return int(self.geom_type.shape[0])

    @property
    def total_mass(self):
        return float(self.body_mass.sum())

    def body_depth(self):
        d = np.zeros(self.nbody, dtype=np.int32)
        for b in range(1, self.nbody):
            d[b] = d[self.body_parent[b]] + 1
        return d

    def legal_contact_mask(self) -> int:
        """Bit g set <=> MuJoCo geom id g may touch the floor without terminating."""
        m = 0
        for i, ok in enumerate(self.geom_legal):
            if ok:
                m |= 1 << (i + 1)
        return m

    # ------------------------------------------------------------------ C view
    def c_struct(self) -> SmplsimModelDescC:
        s = SmplsimModelDescC()
        keep = []

        def dptr(a):
            a = np.ascontiguousarray(a, dtype=np.float64)
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_double))

        def iptr(a):
            a = np.ascontiguousarray(a, dtype=np.int32)
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_int32))

        s.nbody, s.nq, s.nv, s.nu, s.ngeom = self.nbody, self.nq, self.nv, self.nu, self.ngeom
        for name in ("body_parent", "body_dofadr", "body_dofnum", "dof_limited", "geom_type", "geom_body", "geom_legal"):
            setattr(s, name, iptr(getattr(self, name)))
        for name in ("body_pos", "body_quat", "body_mass", "body_ipos", "body_inertia", "body_invweight0", "dof_axis",
                     "dof_armature", "dof_invweight0", "dof_range", "geom_pos", "geom_mat", "geom_size", "act_kp",
                     "act_kd", "act_torque_lim", "act_scale", "act_offset"):
            setattr(s, name, dptr(getattr(self, name)))
        s.plane_pos[:] = list(self.plane_pos)
        s.plane_normal[:] = list(self.plane_normal)
        s.margin = self.margin
        s.friction[:] = list(self.friction)
        s.solref[:] = list(self.solref)
        s.solimp[:] = list(self.solimp)
        s.impratio = self.impratio
        s.timestep = self.timestep
        s.gravity[:] = list(self.gravity)
        s.geom_contype = iptr(self.geom_contype)
        s.geom_conaffinity = iptr(self.geom_conaffinity)
        ex = np.array([[self.body_names.index(a), self.body_names.index(b)] for a, b in self.excludes], dtype=np.int32).reshape(-1, 2)
        s.nexclude = int(ex.shape[0])
        s.exclude_pairs = iptr(ex)
        s._keepalive = keep
        return s


# ----------------------------------------------------------------------------
# numpy kinematics helpers (host; used for invweight0 at build time, by the
# motion table builder and by tests -- never on the stepping path)
# ----------------------------------------------------------------------------
def quat_mul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def axis_angle_quat(axis, ang):
    return np.concatenate([[math.cos(ang / 2)], np.asarray(axis) * math.sin(ang / 2)])


def fk_numpy(m: "ModelDesc", qpos: np.ndarray):
    """xpos[nb,3], xquat[nb,4], world joint axes[nv,3] (MuJoCo kinematics, SURVEY.md A.3)."""
    nb = m.nbody
    xpos = np.zeros((nb, 3))
    xquat = np.zeros((nb, 4))
    axes = np.zeros((m.nv, 3))
    q = qpos[3:7] / np.linalg.norm(qpos[3:7])
    xpos[0], xquat[0] = qpos[0:3], q
    R0 = _mjcf.quat_to_mat(q)
    for k in range(3):
        axes[k] = np.eye(3)[k]
        axes[3 + k] = R0[:, k]
    for b in range(1, nb):
        p = m.body_parent[b]
        Rp = _mjcf.quat_to_mat(xquat[p])
        xpos[b] = xpos[p] + Rp @ m.body_pos[b]
        qb = quat_mul(xquat[p], m.body_quat[b])
        for k in range(m.body_dofnum[b]):
            d = m.body_dofadr[b] + k
            axes[d] = _mjcf.quat_to_mat(qb) @ m.dof_axis[d]
            qb = quat_mul(qb, axis_angle_quat(m.dof_axis[d], qpos[d + 1]))
        xquat[b] = qb / np.linalg.norm(qb)
    return xpos, xquat, axes


def mass_matrix_numpy(m: "ModelDesc", qpos: np.ndarray):
    """Dense joint-space inertia M = sum_b J_b^T I_b J_b + diag(armature) and the
    per-body COM Jacobians (jacp, jacr) in MuJoCo's dof convention."""
    xpos, xquat, axes = fk_numpy(m, qpos)
    nb, nv = m.nbody, m.nv
    M = np.diag(m.dof_armature.copy())
    jacs = []
    for b in range(nb):
        R = _mjcf.quat_to_mat(xquat[b])
        com = xpos[b] + R @ m.body_ipos[b]
        ixx, iyy, izz, ixy, ixz, iyz = m.body_inertia[b]
        Ib = np.array([[ixx, ixy, ixz], [ixy, iyy, iyz], [ixz, iyz, izz]])
        Iw = R @ Ib @ R.T
        jp = np.zeros((3, nv))
        jr = np.zeros((3, nv))
        a = b
        while a >= 0:
            for k in range(m.body_dofnum[a]):
                d = m.body_dofadr[a] + k
                if a == 0 and k < 3:
                    jp[:, d] = axes[d]
                else:
                    jr[:, d] = axes[d]
                    jp[:, d] = np.cross(axes[d], com - xpos[a])
            a = m.body_parent[a]
        M += m.body_mass[b] * jp.T @ jp + jr.T @ Iw @ jr
        jacs.append((jp, jr))
    return M, jacs


def _invweight0(m: "ModelDesc"):
    """body_invweight0 / dof_invweight0 at qpos0 (SURVEY.md A.1)."""
    M, jacs = mass_matrix_numpy(m, m.qpos0)
    Minv = np.linalg.inv(M)
    biw = np.zeros((m.nbody, 2))
    for b, (jp, jr) in enumerate(jacs):
        biw[b, 0] = np.trace(jp @ Minv @ jp.T) / 3.0
        biw[b, 1] = np.trace(jr @ Minv @ jr.T) / 3.0
    d = np.diag(Minv).copy()
    diw = d.copy()
    diw[0:3] = d[0:3].mean()
    diw[3:6] = d[3:6].mean()
    return biw, diw


# ----------------------------------------------------------------------------
# build
# ----------------------------------------------------------------------------
def build_model(p: ParsedMJCF, *, timestep: float = 1.0 / 450.0, contact_bodies: Sequence[str] = (),
                control_mode: str = "uhc_pd", clip_actions: bool = True, pdp_scale: float = 1.0,
                pdd_scale: float = 1.0, power_scale: float = 1.0) -> ModelDesc:
    nb = len(p.bodies)
    mass, ipos, inertia = _mjcf.body_inertials(p)
    parent = np.array([b.parent for b in p.bodies], dtype=np.int32)
    dofnum = np.array([6 if b.free else len(b.joint_axes) for b in p.bodies], dtype=np.int32)
    dofadr = np.concatenate([[0], np.cumsum(dofnum)[:-1]]).astype(np.int32)
    nv = int(dofnum.sum())
    dof_axis = np.zeros((nv, 3))
    arm = np.zeros(nv)
    rng = np.zeros((nv, 2))
    lim = np.zeros(nv, dtype=np.int32)
    jnames: List[str] = []
    for bi, b in enumerate(p.bodies):
        if b.free:
            continue
        for k in range(len(b.joint_axes)):
            d = dofadr[bi] + k
            dof_axis[d] = b.joint_axes[k]
            arm[d] = b.joint_armature[k]
            rng[d] = b.joint_range[k]
            lim[d] = int(b.joint_limited[k])
            jnames.append(b.joint_names[k])
    if list(p.actuator_joints) != jnames:
        raise NotImplementedError("actuators must drive every hinge, in joint order")

    ng = len(p.geoms)
    gtype = np.array([g.type for g in p.geoms], dtype=np.int32)
    gbody = np.array([g.body for g in p.geoms], dtype=np.int32)
    gpos = np.array([g.pos for g in p.geoms])
    gmat = np.array([g.mat.reshape(9) for g in p.geoms])
    gsize = np.array([g.size for g in p.geoms])
    gnames = [g.name for g in p.geoms]
    for cb in contact_bodies:
        if cb not in gnames:
            raise KeyError(f"contact body {cb!r} is not a geom name")      # mj_name2id would return -1
    legal = np.array([1 if g.name in set(contact_bodies) else 0 for g in p.geoms], dtype=np.int32)
    margins = {max(g.margin, p.floor.margin) for g in p.geoms}
    if len(margins) != 1:
        raise NotImplementedError("per-geom contact margins")
    fr = np.max(np.array([np.maximum(g.friction, p.floor.friction) for g in p.geoms]), axis=0)
    for g in p.geoms:
        if g.condim != 3 or p.floor.condim != 3:
            raise NotImplementedError("condim != 3")
        if not ((g.contype & p.floor.conaffinity) or (p.floor.contype & g.conaffinity)):
            raise NotImplementedError("geom that does not collide with the floor")
        if not np.allclose(np.maximum(g.friction, p.floor.friction), fr):
            raise NotImplementedError("per-geom friction")

    # controller constants: humanoid_env.py:325-370
    nu = nv - 6
    kp = np.zeros(nu)
    kd = np.zeros(nu)
    tl = np.zeros(nu)
    scale = np.ones(nu)
    offset = np.zeros(nu)
    for i, jn in enumerate(jnames):
        lo, hi = rng[6 + i]
        s = min(1.2 * max(abs(lo), abs(hi)), math.pi)
        if clip_actions:
            scale[i] = 0.5 * (s - (-s))
            offset[i] = 0.5 * (s + (-s))
        g = pd_gains_for_joint(jn)
        if control_mode in ("pd", "uhc_pd", "simple_pid", "torque"):
            kp[i], kd[i], tl[i] = g
    if control_mode in ("pd", "uhc_pd"):
        kp = kp / pdp_scale
        kd = kd / pdd_scale
    if control_mode == "simple_pid":
        # SimplePID(self.jkp/10, ones, self.jkd/10, timestep*control_freq_inv, torque_lim, ...): humanoid_env.py:318-319
        kp = kp / 10.0
        kd = kd / 10.0
    if control_mode == "torque":
        # SimpleTorqueController(power_scale * torque_lim, torque_lim): humanoid_env.py:321.
        # (the reference leaves torque_lim at zero in this mode -- build_pd_action_scale only
        # fills it for pd / uhc_pd / simple_pid; we use the stablepd limits so the mode is usable.)
        scale = power_scale * tl
        offset = np.zeros(nu)

    if control_mode == "default":
        # compute_torque returns the action itself (humanoid_env.py:407-410): torque mode with unit scale and no clipping
        scale = np.ones(nu)
        offset = np.zeros(nu)
        tl = np.full(nu, 3.0e38)

    zaxis = p.floor.mat[:, 2]
    qpos0 = np.zeros(nv + 1)
    qpos0[0:3] = p.bodies[0].pos
    qpos0[3:7] = p.bodies[0].quat
    m = ModelDesc(
        body_names=[b.name for b in p.bodies], joint_names=jnames, geom_names=gnames,
        body_parent=parent, body_dofadr=dofadr, body_dofnum=dofnum,
        body_pos=np.array([b.pos for b in p.bodies]), body_quat=np.array([b.quat for b in p.bodies]),
        body_mass=mass, body_ipos=ipos,
        body_inertia=np.array([[I[0, 0], I[1, 1], I[2, 2], I[0, 1], I[0, 2], I[1, 2]] for I in inertia]),
        body_invweight0=np.zeros((nb, 2)), dof_axis=dof_axis, dof_armature=arm, dof_invweight0=np.zeros(nv),
        dof_range=rng, dof_limited=lim, geom_type=gtype, geom_body=gbody, geom_pos=gpos, geom_mat=gmat,
        geom_size=gsize, geom_legal=legal, plane_pos=p.floor.pos.copy(), plane_normal=zaxis.copy(),
        margin=float(margins.pop()), friction=fr, solref=p.solref.copy(), solimp=p.solimp.copy(), impratio=1.0,
        timestep=float(timestep), gravity=np.array([0.0, 0.0, -9.81]),
        act_kp=kp, act_kd=kd, act_torque_lim=tl, act_scale=scale, act_offset=offset,
        excludes=list(p.excludes), qpos0=qpos0, geom_contype=np.array([g.contype for g in p.geoms], np.int32),
        geom_conaffinity=np.array([g.conaffinity for g in p.geoms], np.int32))
    # body 0 of the tree hangs off the world: MuJoCo root body_quat is applied at qpos0 only
    m.body_quat[0] = np.array([1.0, 0, 0, 0])
    m.body_invweight0, m.dof_invweight0 = _invweight0(m)
    return m


# ----------------------------------------------------------------------------
# assets: derived tables shipped with the package (generated by
# tools/extract_model.py from the reference's MJCF files; no XML is vendored)
# ----------------------------------------------------------------------------
def _to_jsonable(p: ParsedMJCF):
    def g2d(g):
        return dict(name=g.name, type=g.type, body=g.body, pos=g.pos.tolist(), mat=g.mat.reshape(9).tolist(),
                    size=g.size.tolist(), density=g.density, margin=g.margin, friction=g.friction.tolist(),
                    contype=g.contype, conaffinity=g.conaffinity, condim=g.condim)

    return dict(
        bodies=[dict(name=b.name, parent=b.parent, pos=b.pos.tolist(), quat=b.quat.tolist(), free=b.free,
                     joint_names=b.joint_names, joint_axes=[a.tolist() for a in b.joint_axes],
                     joint_range=[r.tolist() for r in b.joint_range], joint_limited=b.joint_limited,
                     joint_armature=b.joint_armature, geoms=b.geoms) for b in p.bodies],
        geoms=[g2d(g) for g in p.geoms], floor=g2d(p.floor), actuator_joints=p.actuator_joints,
        excludes=[list(e) for e in p.excludes], sensors=[list(s) for s in p.sensors],
        solref=p.solref.tolist(), solimp=p.solimp.tolist())


def _from_jsonable(d) -> ParsedMJCF:
    def d2g(g):
        return _mjcf.Geom(name=g["name"], type=g["type"], body=g["body"], pos=np.array(g["pos"]),
                          mat=np.array(g["mat"]).reshape(3, 3), size=np.array(g["size"]), density=g["density"],
                          margin=g["margin"], friction=np.array(g["friction"]), contype=g["contype"],
                          conaffinity=g["conaffinity"], condim=g["condim"])

    bodies = [_mjcf.Body(name=b["name"], parent=b["parent"], pos=np.array(b["pos"]), quat=np.array(b["quat"]),
                         joint_names=list(b["joint_names"]), joint_axes=[np.array(a) for a in b["joint_axes"]],
                         joint_range=[np.array(r) for r in b["joint_range"]], joint_limited=list(b["joint_limited"]),
                         joint_armature=list(b["joint_armature"]), free=b["free"], geoms=list(b["geoms"]))
              for b in d["bodies"]]
    return ParsedMJCF(bodies=bodies, geoms=[d2g(g) for g in d["geoms"]], floor=d2g(d["floor"]),
                      actuator_joints=list(d["actuator_joints"]), excludes=[tuple(e) for e in d["excludes"]],
                      sensors=[tuple(s) for s in d["sensors"]], solref=np.array(d["solref"]),
                      solimp=np.array(d["solimp"]))


def save_asset(p: ParsedMJCF, name: str):
    os.makedirs(_ASSET_DIR, exist_ok=True)
    with open(os.path.join(_ASSET_DIR, f"{name}.model.json"), "w") as f:
        json.dump(_to_jsonable(p), f, indent=None, separators=(",", ":"))


def load_parsed(name_or_path: str) -> ParsedMJCF:
    """``smpl`` / ``smplx`` (shipped tables), a ``*.model.json`` or an MJCF ``*.xml`` path."""
    if name_or_path.endswith(".xml"):
        with open(name_or_path) as f:
            return parse_mjcf(f.read())
    path = name_or_path
    if not os.path.exists(path):
        path = os.path.join(_ASSET_DIR, f"{name_or_path}_humanoid.model.json")
    with open(path) as f:
        return _from_jsonable(json.load(f))


def shape_variant(p: ParsedMJCF, leg: float = 1.0, arm: float = 1.0, trunk: float = 1.0, girth: float = 1.0,
                  density: float = 1.0) -> ParsedMJCF:
    """A differently proportioned body of the same tree: bone offsets of the leg / arm / trunk bodies scaled, geoms moved and
    stretched with their bones, radii / box extents scaled by ``girth``, densities by ``density`` (masses and inertias follow from
    the geoms, as in MuJoCo's compiler).  A stand-in for what SMPL_Robot writes for other betas (smpllib/smpl_local_robot.py:
    1280-1505) where the SMPL model files are not available; feed the results to HumanoidBatchB200(models=, env_model=)."""
    import copy
    q = copy.deepcopy(p)

    def fac(name):
        if any(k in name for k in ("Hip", "Knee", "Ankle", "Toe")):
            return leg
        if any(k in name for k in ("Shoulder", "Elbow", "Wrist", "Hand", "Thorax", "Index", "Middle", "Pinky", "Ring", "Thumb")):
            return arm
        return trunk

    for b in q.bodies:
        b.pos = np.asarray(b.pos, dtype=np.float64) * (leg if b.free else fac(b.name))   # the root's pos is the standing height
    for g in q.geoms:
        f = fac(q.bodies[g.body].name)
        g.pos = np.asarray(g.pos, dtype=np.float64) * f
        sz = np.asarray(g.size, dtype=np.float64).copy()
        if g.type == GEOM_CAPSULE:
            sz[0] *= girth; sz[1] *= f
        else:
            sz *= girth
        g.size = sz
        g.density = float(g.density) * density
    return q


def load_model(name_or_path: str = "smpl", **kw) -> ModelDesc:
    return build_model(load_parsed(name_or_path), **kw)
