"""Cameras of ``HumanoidBatchB200.render`` (``smplsim_render``, include/smplsim.h: SmplsimCamera).

The reference adds three tracking cameras when ``render_mode == "rgb_array"`` (smpl_sim/smpllib/smpl_xml_addons.py:23-29, added by
humanoid_env.py:256-258) and renders ``cfg.env.camera`` of them (base_env.py:159-162).  Their MJCF values are written out below;
``named`` turns them into ``Camera`` values for a model.  ``EGOCENTRIC`` is the head camera that file sketches (line 32).

Camera frame as in MJCF: the camera looks along its -z axis, +y is up, +x is right; ``fovy`` is the vertical field of view in
degrees (MuJoCo's default 45).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional, Sequence, Union

import numpy as np

from .abi import SmplsimCameraC

FIXED, TRACKCOM, BODY = 0, 1, 2
DEFAULT_FOVY = 45.0
DEFAULT_ZFAR = 100.0

# name: (pos, xyaxes) of the trackcom cameras, smpl_xml_addons.py:23-29, in the order the reference adds them (MuJoCo camera ids 0-2)
TRACKING = {
    "back": ((0.0, 3.0, 2.4), (-1.0, 0.0, 0.0, 0.0, -1.0, 2.0)),
    "side": ((-3.0, 0.0, 2.4), (0.0, -1.0, 0.0, 1.0, 0.0, 2.0)),
    "front_side": ((-2.0, -2.0, 0.8), (0.5, -0.5, 0.0, 0.1, 0.1, 1.0)),
}
TRACKING_IDS = tuple(TRACKING)
# the head camera of smpl_xml_addons.py:32-34: body Head, pos 0 0 0, xyaxes -1 0 0 0 1 0, fovy 80
EGOCENTRIC = dict(body="Head", pos=(0.0, 0.0, 0.0), xyaxes=(-1.0, 0.0, 0.0, 0.0, 1.0, 0.0), fovy=80.0)


@dataclass
class Camera:
    """One camera of ``smplsim_render``.  ``mat`` is row-major 3x3 whose columns are the camera's x, y, z axes in the world
    (FIXED, TRACKCOM) or body (BODY) frame.  ``pos``: FIXED world position, TRACKCOM offset from the robot's centre of mass, BODY
    position in the body frame.  ``exclude_body`` (-1 none): that body's geoms are not drawn."""
    mode: int
    pos: np.ndarray
    mat: np.ndarray
    body: int = -1
    exclude_body: int = -1
    fovy: float = DEFAULT_FOVY
    zfar: float = DEFAULT_ZFAR
    name: Optional[str] = field(default=None, compare=False)

    def c_struct(self) -> SmplsimCameraC:
        c = SmplsimCameraC()
        c.mode, c.body, c.exclude_body = int(self.mode), int(self.body), int(self.exclude_body)
        c.pos[:] = [float(x) for x in np.asarray(self.pos, dtype=np.float64).reshape(3)]
        c.mat[:] = [float(x) for x in np.asarray(self.mat, dtype=np.float64).reshape(9)]
        c.fovy, c.zfar = float(self.fovy), float(self.zfar)
        return c


def xyaxes_mat(xyaxes: Sequence[float]) -> np.ndarray:
    """MJCF ``xyaxes`` -> row-major 3x3 with columns x, y, z: x normalised, y orthonormalised against x, z = x cross y
    [MJ-upstream: the compiler's frame from xyaxes]."""
    a = np.asarray(xyaxes, dtype=np.float64).reshape(2, 3)
    x = a[0] / np.linalg.norm(a[0])
    y = a[1] - np.dot(a[1], x) * x
    y /= np.linalg.norm(y)
    return np.stack([x, y, np.cross(x, y)], axis=1)


def lookat_mat(pos, lookat, up=(0.0, 0.0, 1.0)) -> np.ndarray:
    """Axes of a camera at ``pos`` looking at ``lookat`` with ``up`` projected to its +y."""
    f = np.asarray(lookat, dtype=np.float64) - np.asarray(pos, dtype=np.float64)
    if np.linalg.norm(f) == 0.0:
        raise ValueError("lookat equals pos")
    z = -f / np.linalg.norm(f)
    x = np.cross(np.asarray(up, dtype=np.float64), z)
    if np.linalg.norm(x) < 1e-9:
        raise ValueError("up is parallel to the viewing direction: give xyaxes instead")
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], axis=1)


def robot_com(model, qpos) -> np.ndarray:
    """Centre of mass of the robot at ``qpos`` (host fp64 forward kinematics)."""
    from .model import _mjcf, fk_numpy
    xpos, xquat, _ = fk_numpy(model, np.asarray(qpos, dtype=np.float64))
    m = np.asarray(model.body_mass, dtype=np.float64)
    ipos = np.asarray(model.body_ipos, dtype=np.float64)
    com = np.stack([xpos[b] + _mjcf.quat_to_mat(xquat[b]) @ ipos[b] for b in range(model.nbody)])
    return (m[:, None] * com).sum(0) / m.sum()


def fixed(pos, xyaxes=None, lookat=None, fovy: float = DEFAULT_FOVY, zfar: float = DEFAULT_ZFAR) -> Camera:
    """A world-fixed camera, oriented by MJCF ``xyaxes`` or by a point to look at (z up)."""
    if (xyaxes is None) == (lookat is None):
        raise ValueError("fixed() takes exactly one of xyaxes / lookat")
    mat = xyaxes_mat(xyaxes) if xyaxes is not None else lookat_mat(pos, lookat)
    return Camera(FIXED, np.asarray(pos, dtype=np.float64), mat, fovy=fovy, zfar=zfar)


def trackcom(model, pos, xyaxes, fovy: float = DEFAULT_FOVY, zfar: float = DEFAULT_ZFAR, name: Optional[str] = None) -> Camera:
    """An MJCF ``mode="trackcom"`` world camera declared at ``pos``: it keeps its axes and its offset from the robot's centre of mass
    at the model's qpos0 (what mj_setConst stores [MJ-upstream])."""
    off = np.asarray(pos, dtype=np.float64) - robot_com(model, model.qpos0)
    return Camera(TRACKCOM, off, xyaxes_mat(xyaxes), fovy=fovy, zfar=zfar, name=name)


def body(model, name: Union[int, str], pos=(0.0, 0.0, 0.0), xyaxes=(1.0, 0.0, 0.0, 0.0, 1.0, 0.0), fovy: float = DEFAULT_FOVY,
         zfar: float = DEFAULT_ZFAR, exclude: bool = True) -> Camera:
    """A camera riding on robot body ``name`` (pose in the body frame).  ``exclude``: that body's own geoms are not drawn."""
    rule = f"body must be a name or an index in [0, {model.nbody})"
    b = model.body_index(name, rule)
    if not 0 <= b < model.nbody:
        raise ValueError(f"{rule}, got {name!r}")
    return Camera(BODY, np.asarray(pos, dtype=np.float64), xyaxes_mat(xyaxes), body=b, exclude_body=b if exclude else -1, fovy=fovy,
                  zfar=zfar, name=name if isinstance(name, str) else None)


def named(model, cam: Union[str, int, Camera]) -> Camera:
    """``"back"`` / ``"side"`` / ``"front_side"`` (or their MuJoCo ids 0-2), ``"egocentric"``, or a ``Camera`` (returned as is)."""
    if isinstance(cam, Camera):
        return cam
    if isinstance(cam, (int, np.integer)) and not isinstance(cam, bool):
        if not 0 <= int(cam) < len(TRACKING_IDS):
            raise ValueError(f"camera id {int(cam)} is not supported: ids 0-2 are {list(TRACKING_IDS)} (MuJoCo's free camera -1 is not "
                             f"available); names: {supported()}")
        cam = TRACKING_IDS[int(cam)]
    if cam == "egocentric":
        return body(model, EGOCENTRIC["body"], EGOCENTRIC["pos"], EGOCENTRIC["xyaxes"], fovy=EGOCENTRIC["fovy"])
    if cam in TRACKING:
        pos, xy = TRACKING[cam]
        return trackcom(model, pos, xy, name=cam)
    raise ValueError(f"unknown camera {cam!r}: supported cameras are {supported()} (or ids 0-2), or a smplsim_b200.camera.Camera")


def supported():
    return list(TRACKING_IDS) + ["egocentric"]
