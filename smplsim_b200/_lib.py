"""ctypes loader for libsmplsim_b200.so (the CUDA product library).  There is no CPU fallback:
if the library is missing or fails to load, importing / calling raises."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("SMPLSIM_SO") or os.path.join(_HERE, "libsmplsim_b200.so")   # SMPLSIM_SO: debug builds (tools/)
_CSRC = os.path.join(_HERE, "csrc")
_LIB = None

# -ftz / -prec-div / -prec-sqrt: denormals flushed, division and square root at 2 ulp (MUFU + one Newton step instead of the IEEE
# sequences with their slow paths and denormal guards).  FMA contraction and everything else stay as in the default mode; the parity
# tolerances (1e-4 against the fp64 oracle) are met with a wide margin, and the step kernel is faster (fewer instructions on its dependent chains).
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-ftz=true", "-prec-div=false", "-prec-sqrt=false",
              "-shared", "-Xcompiler", "-fPIC"]


def sources():
    import glob
    return sorted(glob.glob(os.path.join(_CSRC, "*.cu")) + glob.glob(os.path.join(_CSRC, "*.cuh")) + glob.glob(os.path.join(_CSRC, "*.hpp"))) + [
        os.path.join(_HERE, "..", "include", "smplsim.h")]


def build(force: bool = False, verbose: bool = False) -> str:
    """nvcc-compile the library in-tree for sm_90a (H100; cross-compiles without a GPU)."""
    newest = max(os.path.getmtime(s) for s in sources())
    if force or not os.path.exists(SO_PATH) or os.path.getmtime(SO_PATH) < newest:
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", SO_PATH, os.path.join(_CSRC, "smplsim_capi.cu"),
                                                                               os.path.join(_CSRC, "rollout_kernels.cu"),
                                                                               os.path.join(_CSRC, "rollout_feedback_kernels.cu"),
                                                                               os.path.join(_CSRC, "inverse_fd_kernels.cu"),
                                                                               os.path.join(_CSRC, "centroidal_kernels.cu"),
                                                                               os.path.join(_CSRC, "rne_post_kernels.cu")]
        subprocess.check_call(cmd, cwd=_CSRC)
    return SO_PATH


_SYMBOLS = {
    "smplsim_last_error": (C.c_char_p, []),
    "smplsim_version": (C.c_int, []),
    "smplsim_create": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "smplsim_create_shapes": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "smplsim_num_shapes": (C.c_int, [C.c_void_p]),
    "smplsim_destroy": (C.c_int, [C.c_void_p]),
    "smplsim_obs_dim": (C.c_int, [C.c_void_p]),
    "smplsim_num_envs": (C.c_int, [C.c_void_p]),
    "smplsim_reset": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_mj_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "smplsim_kinematics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "smplsim_inverse": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "smplsim_dynamics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "smplsim_centroidal": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "smplsim_rne_post": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "smplsim_transition_fd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_inverse_fd": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]),
    "smplsim_rollout": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                 C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_rollout_feedback": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "smplsim_ray": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                             C.c_void_p, C.c_void_p]),
    "smplsim_render": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_set_env_params": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_get_env_params": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_clear_env_params": (C.c_int, [C.c_void_p]),
    "smplsim_self_obs": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "smplsim_motion_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_motion_blend": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "smplsim_imitation_obs_dim": (C.c_int, [C.c_void_p, C.c_int]),
    "smplsim_imitation": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_imitation_recovery": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]),
    "smplsim_track_eval": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p]),
    "smplsim_amp_obs_dim": (C.c_int, [C.c_void_p, C.c_void_p]),
    "smplsim_amp_obs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.c_void_p, C.c_void_p]),
    "smplsim_amp_demo": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "smplsim_gae": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p,
                              C.c_void_p, C.c_void_p]),
    "smplsim_smem_bytes_per_env": (C.c_int, [C.c_void_p]),
    "smplsim_warps_per_block": (C.c_int, [C.c_void_p]),
    "smplsim_kernel_version": (C.c_int, [C.c_void_p]),
    "smplsim_schedule_steps": (C.c_int, [C.c_void_p]),
}
# the entry points include/smplsim.h declares (checked by tests/test_abi.py)
_INTROSPECTION = ("smplsim_smem_bytes_per_env", "smplsim_warps_per_block", "smplsim_kernel_version", "smplsim_schedule_steps")
HEADER_SYMBOLS = [s for s in _SYMBOLS if s not in _INTROSPECTION]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(no CPU fallback exists for the stepper)")
        L = C.CDLL(SO_PATH)
        for name, (res, args) in _SYMBOLS.items():
            fn = getattr(L, name)          # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


class SmplsimError(RuntimeError):
    pass


def check(rc: int):
    if rc != 0:
        raise SmplsimError(f"libsmplsim_b200 error {rc}: {lib().smplsim_last_error().decode()}")
