"""smplsim_b200 -- H100-native (sm_90a) batched SMPL-humanoid physics stepper.

Drop-in for the hot path of ZhengyiLuo/SMPLSim (``HumanoidEnv.step`` =
15 x [PD torque + mj_step] + obs / reward / reset flags).  See DESIGN.md.
"""
from .model import ModelDesc, load_model  # noqa: F401

__all__ = ["ModelDesc", "load_model", "HumanoidImB200"]


def __getattr__(name):          # the env classes need torch: imported on first use
    if name == "HumanoidImB200":
        from .imitation import HumanoidImB200
        return HumanoidImB200
    raise AttributeError(name)
