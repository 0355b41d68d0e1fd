"""Config objects accepted by the boundary.

The reference composes ``smpl_sim/data/cfg/config.yaml`` with the ``env`` / ``robot`` /
``learning`` groups through hydra (smpl_sim/run.py:31-35) and reads ``cfg.env.*`` /
``cfg.robot.*`` / ``cfg.headless`` in ``HumanoidEnv.__init__`` (smpl_sim/envs/humanoid_env.py:148-241,
smpl_sim/envs/base_env.py:23-49).  hydra / omegaconf are not part of this image, so the boundary
takes any attribute-style mapping (OmegaConf DictConfig, EasyDict, or the ``Cfg`` below) and this
module re-creates the group composition with the same keys and default values.
"""
from __future__ import annotations

import copy
from typing import Any, Dict, Mapping, Optional


class Cfg(dict):
    """dict with attribute access and ``.get`` (what the reference needs from DictConfig)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    @staticmethod
    def wrap(x):
        if isinstance(x, Mapping):
            return Cfg({k: Cfg.wrap(v) for k, v in x.items()})
        if isinstance(x, (list, tuple)):
            return [Cfg.wrap(v) for v in x]
        return x


# env group -- values of smpl_sim/data/cfg/env/{base_env,speed,reach,getup}.yaml
_ENV_COMMON = dict(
    episode_length=300, sim_timestep_inv=450, control_frequency_inv=15, power_scale=10, root_height_obs=True,
    enable_early_termination=True, self_obs_v=1, kp_scale=1.0, kd_scale=1.0, cycle_motion=False, power_reward=True,
    clip_actions=True, control_mode="uhc_pd", render_mode="human", camera="side", state_init="Default",
    pdp_scale=1, pdd_scale=1, pdi_scale=1)
_FEET = ["R_Ankle", "L_Ankle", "R_Toe", "L_Toe"]
ENV_GROUPS: Dict[str, Dict[str, Any]] = {
    "base_env": dict(_ENV_COMMON, task="HumanoidEnv", contact_bodies=[]),
    "humanoid_env": dict(_ENV_COMMON, task="HumanoidEnv", power_scale=1.0, contact_bodies=list(_FEET)),
    "speed": dict(_ENV_COMMON, task="HumanoidSpeed", tar_speed_min=0.0, tar_speed_max=5.0, speed_change_steps_min=100,
                  speed_change_steps_max=200, contact_bodies=list(_FEET)),
    "reach": dict(_ENV_COMMON, task="HumanoidReach", contact_bodies=list(_FEET), reach_body_name="R_Hand",
                  tar_dist_max=1, tar_height_min=0.2, tar_height_max=2.0, tar_change_steps_min=50,
                  tar_change_steps_max=100),
    "getup": dict(_ENV_COMMON, task="HumanoidGetup", state_init="Fall", recovery_steps=60, tar_height_min=0.5,
                  tar_height_max=1.2, height_change_steps_min=100, height_change_steps_max=200,
                  contact_bodies=list(_FEET)),
    # motion imitation (imitation.py; not a reference group: its MuJoCo env layer ships no imitation task).  reward gains k and
    # weights w over (position, rotation, velocity, angular velocity); tracked_bodies: body names or indices, None = all
    "im": dict(_ENV_COMMON, task="HumanoidIm", state_init="MoCap", self_obs_v=2, create_vel_sensors=True, contact_bodies=list(_FEET),
               im_k_pos=100.0, im_k_rot=10.0, im_k_vel=0.1, im_k_angvel=0.1, im_w_pos=0.5, im_w_rot=0.3, im_w_vel=0.1, im_w_angvel=0.1,
               termination_distance=0.25, tracked_bodies=None,
               # blended reference states (get_motion_state) instead of nearest frames; future targets per observation, 1 / inv s apart
               # (PHC: numTrajSamples, trajSampleTimestepInv)
               im_interpolate=False, num_traj_samples=1, traj_sample_timestep_inv=30),
}
# robot group -- smpl_sim/data/cfg/robot/{smpl,smplx}_humanoid.yaml
_ROBOT_COMMON = dict(
    has_upright_start=False, has_shape_obs=False, has_weight_obs=False, has_shape_variation=False, has_mesh=False,
    replace_feet=True, has_jt_limit=False, height_fix_mode="full", big_ankle=True, remove_toe=False,
    real_weight_porpotion_capsules=True, real_weight_porpotion_boxes=True, real_weight=True, box_body=True,
    smpl_data_dir="data/smpl", create_vel_sensors=False)
ROBOT_GROUPS = {
    "smpl_humanoid": dict(_ROBOT_COMMON, humanoid_type="smpl"),
    "smplx_humanoid": dict(_ROBOT_COMMON, humanoid_type="smplx"),
}
# top level -- smpl_sim/data/cfg/config.yaml
_TOP = dict(notes="Default Notes", exp_name="humanoid_smpl", headless=True, seed=0, no_log=False, resume_str=None,
            num_threads=36, test=False, epoch=0)


def _apply_override(cfg: Cfg, key: str, value):
    node = cfg
    parts = key.split(".")
    for p in parts[:-1]:
        if p not in node:
            node[p] = Cfg()
        node = node[p]
    node[parts[-1]] = value


def make_cfg(env: str = "base_env", robot: str = "smpl_humanoid", overrides: Optional[Mapping[str, Any]] = None,
             **top) -> Cfg:
    """``python smpl_sim/run.py env=speed robot=... key=value`` -> cfg (hydra ``defaults`` composition).

    b200-only additions live under ``cfg.env``: ``self_collision`` (geom-geom contacts between the capsule / sphere pairs MuJoCo's
    filters let through, simulated as two-body rows; default False = detected only, aux.status bit 32), ``num_envs`` (default 1), ``spd_inertia``
    ("stale" = reference quirk Q1 | "fresh"), ``legacy_change_step_bug`` (quirk Q4, default True),
    and ``cfg.robot.xml_path`` (explicit MJCF; default = shipped table for ``humanoid_type``).
    """
    c = Cfg.wrap(copy.deepcopy(_TOP))
    c.update(top)
    c["env"] = Cfg.wrap(copy.deepcopy(ENV_GROUPS[env]))
    c["robot"] = Cfg.wrap(copy.deepcopy(ROBOT_GROUPS[robot]))
    if c["env"].get("create_vel_sensors"):      # an env group that needs the body-velocity sensors (obs v2) turns them on in the robot
        c["robot"]["create_vel_sensors"] = True
    c["output_dir"] = f"outputs/{c['exp_name']}"
    for k, v in (overrides or {}).items():
        _apply_override(c, k, v)
    return c
