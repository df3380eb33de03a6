import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


def _has_gpu():
    try:
        import ctypes
        cu = ctypes.CDLL("libcuda.so.1")
        if cu.cuInit(0) != 0:
            return False
        n = ctypes.c_int()
        return cu.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


HAS_GPU = _has_gpu()


def pytest_collection_modifyitems(config, items):
    if HAS_GPU:
        return
    skip = pytest.mark.skip(reason="no GPU in this container (runs under gpurun)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def gx():
    """The libgpuexec context. Fails loudly (never falls back) when the CUDA
    library or the GPU is missing."""
    import opentenbase_b200 as g
    ctx = g.Context(0)
    yield ctx
    ctx.close()
