"""ctypes mirrors of include/smplsim.h and cfg -> SmplsimEnvCfg translation."""
from __future__ import annotations

import ctypes as C
from typing import Any

from .model import ModelDesc, SmplsimModelDescC  # noqa: F401

TASKS = {"HumanoidEnv": 0, "HumanoidSpeed": 1, "HumanoidReach": 2, "HumanoidGetup": 3,
         "HumanoidIm": 0}   # imitation: the stepper runs SMPLSIM_TASK_NONE, the task is smplsim_imitation (imitation.py)
CTRL_MODES = {"uhc_pd": 0, "pd": 1, "torque": 2, "simple_pid": 3, "default": 2}   # "default": ctrl = action (humanoid_env.py:409-410) = torque mode, scale 1, no limit
STATE_INITS = {"Default": 0, "Fall": 1, "MoCap": 2}
_AVAILABLE_CONTROLLERS = ["uhc_pd", "simple_pid", "pd", "torque", "default"]   # humanoid_env.py:32


class SmplsimEnvCfgC(C.Structure):
    _fields_ = [
        ("task", C.c_int32), ("control_mode", C.c_int32), ("self_obs_v", C.c_int32), ("root_height_obs", C.c_int32),
        ("upright_start", C.c_int32), ("nsubsteps", C.c_int32), ("episode_length", C.c_int32),
        ("state_init", C.c_int32), ("spd_stale", C.c_int32), ("legacy_change_step", C.c_int32),
        ("reach_body", C.c_int32), ("recovery_steps", C.c_int32), ("change_steps_min", C.c_int32),
        ("change_steps_max", C.c_int32),
        ("tar_speed_min", C.c_double), ("tar_speed_max", C.c_double), ("tar_dist_max", C.c_double),
        ("tar_height_min", C.c_double), ("tar_height_max", C.c_double), ("seed", C.c_uint64),
        ("self_collision", C.c_int32), ("pad_", C.c_int32),
    ]


class SmplsimStateC(C.Structure):
    _fields_ = [
        ("qpos", C.c_void_p), ("qvel", C.c_void_p), ("qpos_fwd", C.c_void_p), ("qvel_fwd", C.c_void_p),
        ("qacc_warm", C.c_void_p), ("task_target", C.c_void_p), ("task_change_step", C.c_void_p),
        ("progress", C.c_void_p), ("recovery", C.c_void_p), ("rng_counter", C.c_void_p),
        ("pid_integral", C.c_void_p), ("pid_last_error", C.c_void_p), ("xfrc_applied", C.c_void_p),
    ]


class SmplsimAuxC(C.Structure):
    _fields_ = [
        ("xpos", C.c_void_p), ("xquat", C.c_void_p), ("body_linvel", C.c_void_p), ("body_angvel", C.c_void_p),
        ("contact_mask", C.c_void_p), ("qacc", C.c_void_p), ("ctrl", C.c_void_p), ("solver_iter", C.c_void_p), ("status", C.c_void_p),
        ("contact_wrench", C.c_void_p),
    ]


class SmplsimCameraC(C.Structure):
    _fields_ = [("mode", C.c_int32), ("body", C.c_int32), ("exclude_body", C.c_int32), ("pad_", C.c_int32), ("pos", C.c_float * 3),
                ("mat", C.c_float * 9), ("fovy", C.c_float), ("zfar", C.c_float)]


class SmplsimEnvParamsC(C.Structure):
    _fields_ = [("friction", C.c_void_p), ("gravity", C.c_void_p), ("kp", C.c_void_p), ("kd", C.c_void_p), ("torque_limit", C.c_void_p),
                ("body_mass_scale", C.c_void_p)]


class SmplsimFdCfgC(C.Structure):
    _fields_ = [("eps_qpos", C.c_float), ("eps_qvel", C.c_float), ("eps_ctrl", C.c_float), ("centered", C.c_int32), ("pad_", C.c_int32)]


class SmplsimInverseFdCfgC(C.Structure):
    _fields_ = [("eps_qpos", C.c_float), ("eps_qvel", C.c_float), ("eps_qacc", C.c_float), ("centered", C.c_int32), ("pad_", C.c_int32)]


class SmplsimImitationCfgC(C.Structure):
    _fields_ = [("k_pos", C.c_float), ("k_rot", C.c_float), ("k_vel", C.c_float), ("k_angvel", C.c_float),
                ("w_pos", C.c_float), ("w_rot", C.c_float), ("w_vel", C.c_float), ("w_angvel", C.c_float),
                ("termination_distance", C.c_float), ("episode_length", C.c_int32), ("self_obs_dim", C.c_int32),
                ("num_tracked", C.c_int32), ("tracked_bodies", C.c_void_p), ("interpolate", C.c_int32), ("num_future", C.c_int32),
                ("future_dt", C.c_float)]


class SmplsimImitationRecoveryC(C.Structure):
    _fields_ = [("zero_out_far", C.c_int32), ("far_distance", C.c_float), ("power_coefficient", C.c_float), ("pad_", C.c_int32),
                ("recovery", C.c_void_p), ("goal_dist", C.c_void_p), ("qvel", C.c_void_p), ("power", C.c_void_p)]


class SmplsimMotionTablesC(C.Structure):
    _fields_ = [("xpos", C.c_void_p), ("xquat", C.c_void_p), ("body_vel", C.c_void_p), ("body_ang_vel", C.c_void_p),
                ("motion_len", C.c_void_p), ("num_frames", C.c_void_p), ("motion_dt", C.c_void_p), ("length_starts", C.c_void_p),
                ("num_motions", C.c_int32), ("nbody", C.c_int32)]


class SmplsimTrackEvalCfgC(C.Structure):
    _fields_ = [("num_bodies", C.c_int32), ("bodies", C.c_void_p), ("interpolate", C.c_int32), ("dt", C.c_float)]


class SmplsimTrackEvalStateC(C.Structure):
    _fields_ = [("active", C.c_void_p), ("prev_diff", C.c_void_p), ("frames", C.c_void_p), ("sums", C.c_void_p), ("success", C.c_void_p),
                ("frame_metrics", C.c_void_p)]


# SMPLSIM_TRACK_* columns of SmplsimTrackEvalState.sums / frame_metrics
TRACK_METRICS = ("mpjpe_g", "mpjpe_l", "mpjpe_pa", "vel_dist", "accel_dist", "rot_error")


class SmplsimAmpCfgC(C.Structure):
    _fields_ = [("num_steps", C.c_int32), ("num_key_bodies", C.c_int32), ("key_bodies", C.c_void_p), ("local_root_obs", C.c_int32),
                ("root_height_obs", C.c_int32), ("interpolate", C.c_int32)]


class SmplsimAmpTablesC(C.Structure):
    _fields_ = [("motion", C.c_void_p), ("dof_pos", C.c_void_p), ("dof_vel", C.c_void_p)]


AMP_PUSH, AMP_FILL, AMP_FILL_REF = 0, 1, 2     # SMPLSIM_AMP_* modes of smplsim_amp_obs
BLEND_LERP, BLEND_POS, BLEND_SLERP, BLEND_QPOS, BLEND_ROW0 = 0, 1, 2, 3, 4   # SMPLSIM_BLEND_* value kinds of smplsim_motion_blend


def _get(node: Any, key: str, default=None):
    if hasattr(node, "get"):
        return node.get(key, default)
    return getattr(node, key, default)


def env_cfg_from(cfg: Any, model: ModelDesc, seed: int = 0) -> SmplsimEnvCfgC:
    """Translate ``cfg.env`` / ``cfg.robot`` (reference keys) into the C struct.

    Mirrors the reads in HumanoidEnv.__init__ (humanoid_env.py:153-162), BaseEnv.__init__
    (base_env.py:23-32) and the task constructors (tasks/humanoid_speed.py:51-56,
    humanoid_reach.py:35-46, humanoid_getup.py:29-39).
    """
    e, r = cfg.env, cfg.robot
    mode = e.control_mode
    assert mode in _AVAILABLE_CONTROLLERS, f"{mode} is not a valid controller {_AVAILABLE_CONTROLLERS}"
    if mode not in CTRL_MODES:
        raise NotImplementedError(f"control_mode={mode!r} is not built for the b200 backend (have {list(CTRL_MODES)})")
    task = _get(e, "task", "HumanoidEnv")
    if task not in TASKS:
        raise NotImplementedError(f"task {task!r}")
    if r.humanoid_type not in ("smpl", "smplh", "smplx"):
        raise NotImplementedError(f"humanoid_type: {r.humanoid_type}")
    if _get(r, "has_shape_variation", False) or _get(r, "has_shape_obs", False) or _get(r, "has_weight_obs", False):
        # humanoid_env.py:304-305 only adds 10 to _num_self_obs for has_shape_variation -- compute_proprioception (:372-403) never fills
        # them, so the reference's own MuJoCo path is inconsistent with the flag set; shape / limb-weight obs exist on the Isaac side only.
        raise NotImplementedError("has_shape_variation / has_shape_obs / has_weight_obs change the observation only on the Isaac side of the "
                                  "reference; per-env body shapes themselves: HumanoidBatchB200(models=[...], env_model=[...])")
    v = int(e.self_obs_v)
    if v not in (1, 2):
        raise NotImplementedError(f"self_obs_v: {v}")
    if v == 2:
        assert r.create_vel_sensors            # humanoid_env.py:297
    c = SmplsimEnvCfgC()
    c.task = TASKS[task]
    c.control_mode = CTRL_MODES[mode]
    c.self_obs_v = v
    c.root_height_obs = int(bool(e.root_height_obs))
    c.upright_start = int(bool(r.has_upright_start))
    c.nsubsteps = int(e.control_frequency_inv)
    c.episode_length = int(e.episode_length)
    c.state_init = STATE_INITS[e.state_init]
    c.spd_stale = int(_get(e, "spd_inertia", "stale") == "stale")
    c.legacy_change_step = int(bool(_get(e, "legacy_change_step_bug", True)))
    c.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    c.self_collision = int(bool(_get(e, "self_collision", False)))
    if task == "HumanoidSpeed":
        c.tar_speed_min, c.tar_speed_max = float(e.tar_speed_min), float(e.tar_speed_max)
        c.change_steps_min, c.change_steps_max = int(e.speed_change_steps_min), int(e.speed_change_steps_max)
    elif task == "HumanoidReach":
        c.tar_dist_max = float(e.tar_dist_max)
        c.tar_height_min, c.tar_height_max = float(e.tar_height_min), float(e.tar_height_max)
        c.change_steps_min, c.change_steps_max = int(e.tar_change_steps_min), int(e.tar_change_steps_max)
        c.reach_body = model.body_names.index(e.reach_body_name)
    elif task == "HumanoidGetup":
        c.tar_height_min, c.tar_height_max = float(e.tar_height_min), float(e.tar_height_max)
        c.change_steps_min, c.change_steps_max = int(e.height_change_steps_min), int(e.height_change_steps_max)
        c.recovery_steps = int(e.recovery_steps)
    return c


def model_from_cfg(cfg: Any):
    """Build the ModelDesc the way HumanoidEnv._create_humanoid_robot + create_sim +
    setup_controller do (humanoid_env.py:219-260,312-370; base_env.py:139-142)."""
    from .model import load_model
    e, r = cfg.env, cfg.robot
    src = _get(r, "xml_path", None) or ("smplx" if r.humanoid_type == "smplx" else "smpl")
    return load_model(src, timestep=1.0 / float(e.sim_timestep_inv), contact_bodies=list(e.contact_bodies),
                      control_mode=e.control_mode if e.control_mode in CTRL_MODES else "uhc_pd",
                      clip_actions=bool(e.clip_actions), pdp_scale=float(_get(e, "pdp_scale", 1)),
                      pdd_scale=float(_get(e, "pdd_scale", 1)), power_scale=float(e.power_scale))
