"""pytest configuration: markers, import paths, and building the in-tree libraries once."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "all-is-cubes_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (compute capability 9.0; run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built_libraries():
    import __graft_entry__ as g
    g.build_library()
    g.build_oracle()
    yield


def has_gpu():
    try:
        import ctypes
        lib = ctypes.CDLL("libcuda.so.1")
        if lib.cuInit(0) != 0:
            return False
        n = ctypes.c_int(0)
        return lib.cuDeviceGetCount(ctypes.byref(n)) == 0 and n.value > 0
    except OSError:
        return False
