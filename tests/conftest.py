import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "gpu_only: no emulator variant of this test (size / timing)")


class Backend:
    """Where a parity test runs the product's kernels: "gpu" = libsmplsim_b200.so on cuda:0 (the parity tests proper, -m gpu),
    "emu" = the same kernel sources on the host SIMT emulator (tests/emu, test infrastructure) so the CPU suite covers the
    kernel logic too."""

    def __init__(self, name):
        self.name = name
        self.device = "cuda:0" if name == "gpu" else "cpu"

    def batch(self, cfg, n, seed=0, **kw):
        if self.name == "gpu":
            from smplsim_b200.batched import HumanoidBatchB200
            return HumanoidBatchB200(cfg, num_envs=n, device="cuda:0", seed=seed, **kw)
        sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
        import emu_env
        return emu_env.EmuBatch(cfg, n, seed=seed, **kw)

    def t(self, x, dtype=None):
        import numpy as np
        import torch
        return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype or torch.float32, device=self.device)


@pytest.fixture(params=[pytest.param("gpu", marks=pytest.mark.gpu), pytest.param("emu")])
def backend(request):
    if request.param == "emu" and request.node.get_closest_marker("gpu_only"):
        pytest.skip("gpu only")
    return Backend(request.param)


def pytest_collection_modifyitems(config, items):
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)
