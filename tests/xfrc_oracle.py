"""TEST INFRASTRUCTURE: ctypes wrapper of tests/xfrc_oracle.c, the fp64 oracle with external body wrenches (mj_data.xfrc_applied).

``XfrcOracleEnv`` is an ``oracle.OracleEnv`` whose ``forward`` / ``mj_step`` / ``step`` add the wrench held in ``xfrc_applied``
([nbody, 6] float64, robot bodies, row 0 = root: force at the centre of mass, then torque, world axes).  Like MuJoCo's
mj_data.xfrc_applied it persists across calls and is zeroed by an auto-reset (mj_resetData).  ``qfrc_applied`` holds J^T of the
wrench of the last forward pass.  ``reset`` is the oracle's own: resets ignore the wrench."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
SO = os.path.join(_HERE, "libxfrc_oracle.so")
_L = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "xfrc_oracle.c")
    deps = [src, os.path.join(_ROOT, "oracle", "mjstep_oracle.c"), os.path.join(_ROOT, "include", "smplsim.h")]
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(p) for p in deps):
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        subprocess.check_call([cc, "-O3", "-march=x86-64-v2", "-fPIC", "-shared", "-o", SO, src, "-lm", "-lpthread"], cwd=_HERE)
    return SO


def lib():
    global _L
    if _L is None:
        L = C.CDLL(build())
        dp = C.POINTER(C.c_double)
        L.orx_forward.argtypes = [C.c_void_p, C.c_void_p, dp, dp]
        L.orx_step.argtypes = [C.c_void_p, C.c_void_p, dp, dp]
        L.orx_env_step.argtypes = [C.c_void_p, C.c_void_p, dp, dp, dp, dp, dp, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _L = L
    return _L


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class XfrcOracleEnv(orc.OracleEnv):
    def __init__(self, om: orc.OracleModel, env_id: int = 0):
        super().__init__(om, env_id)
        self.xfrc_applied = np.zeros((self.m.nbody, 6))
        self.qfrc_applied = np.zeros(self.m.nv)

    def forward(self):
        lib().orx_forward(self.om.ptr, self.ptr, _dp(self.xfrc_applied), _dp(self.qfrc_applied))

    def mj_step(self):
        lib().orx_step(self.om.ptr, self.ptr, _dp(self.xfrc_applied), _dp(self.qfrc_applied))

    def step(self, action):
        a = np.ascontiguousarray(action, dtype=np.float64)
        o = np.zeros(self.om.obs_dim + 8)
        rew = C.c_double()
        term, trunc = C.c_int(), C.c_int()
        n = lib().orx_env_step(self.om.ptr, self.ptr, _dp(a), _dp(self.xfrc_applied), _dp(self.qfrc_applied), _dp(o), C.byref(rew),
                               C.byref(term), C.byref(trunc))
        return o[:n], rew.value, bool(term.value), bool(trunc.value)
