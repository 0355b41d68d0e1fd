"""Shared-memory layout of the step kernels (no GPU: the handle is created through the emulator build of the same sources).

The SMPL env rows must stay small enough that 32 envs (8 warps) and the constant table fit the 227 KB a CTA can opt into on an
H100, so that the headline 4 096-env batch runs as one wave over the 132 SMs."""
import ctypes as C
import os
import sys

import pytest

from smplsim_b200.abi import env_cfg_from, model_from_cfg
from smplsim_b200.cfg import make_cfg

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu_env  # noqa: E402

H100_SMEM_OPTIN = 232448   # bytes per CTA (227 KB)
H100_SMS = 132
SMPL_ENV_BYTES = 6896      # 1724 words: state rows, body rows, mailboxes, 15 contact entries, limit rows, misc


def _create(robot, num_envs):
    L = emu_env.lib()
    cfg = make_cfg(env="speed", robot=robot)
    m = model_from_cfg(cfg)
    ec = env_cfg_from(cfg, m, seed=0)
    cm = m.c_struct()
    h = C.c_void_p()
    rc = L.smplsim_create(C.addressof(cm), C.addressof(ec), num_envs, 0, C.byref(h))
    assert rc == 0, L.smplsim_last_error().decode()
    return L, h


def test_smpl_env_rows_fit_eight_warps():
    L, h = _create("smpl_humanoid", 4096)
    try:
        env_bytes, wpb = L.smplsim_smem_bytes_per_env(h), L.smplsim_warps_per_block(h)
        assert env_bytes == SMPL_ENV_BYTES
        assert (env_bytes // 4) % 8 == 4            # stride: float4 rows, not a multiple of 8 words (bank spread)
        assert 32 * env_bytes + 16 < H100_SMEM_OPTIN
        # the CTA size rule takes the fewest waves: 8 warps x 4 envs, table included, fit -> 128 CTAs, one wave on 132 SMs
        assert wpb == 8
        assert -(-4096 // (wpb * 4)) <= H100_SMS
    finally:
        L.smplsim_destroy(h)


@pytest.mark.parametrize("num_envs, waves", [(2048, 1), (8192, 2)])
def test_smpl_waves(num_envs, waves):
    L, h = _create("smpl_humanoid", num_envs)
    try:
        per = L.smplsim_warps_per_block(h) * 4
        assert -(-(-(-num_envs // per)) // H100_SMS) == waves
    finally:
        L.smplsim_destroy(h)
