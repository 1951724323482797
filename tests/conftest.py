import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def _have_gpu():
    try:
        import ctypes
        cuda = ctypes.CDLL("libcuda.so.1")
        if cuda.cuInit(0) != 0:
            return False
        n = ctypes.c_int(0)
        return cuda.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False


HAVE_GPU = _have_gpu()


def pytest_collection_modifyitems(config, items):
    if HAVE_GPU:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    """Build the native library and the oracle once (nvcc/g++ only; cross-compiles without a GPU).
    Where build() has already run this is a no-op."""
    from simlod_b200 import build
    build.build_native()
    build.build_oracle()
