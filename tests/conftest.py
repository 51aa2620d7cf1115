import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _cuda_device_present() -> bool:
    """True when a CUDA driver and at least one device are there (no torch import: cheap and side-effect free)."""
    try:
        cuda = ctypes.CDLL("libcuda.so.1")
        n = ctypes.c_int(0)
        return cuda.cuInit(0) == 0 and cuda.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a CPU-only host skips the gpu-marked tests instead of failing in them
    (the engine has no CPU fallback: jr_engine_create returns JR_E_NO_DEVICE there)."""
    if _cuda_device_present():
        return
    skip = pytest.mark.skip(reason="no CUDA device: the engine has no CPU fallback")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle_lib():
    from oracle import restated
    return restated.load()
