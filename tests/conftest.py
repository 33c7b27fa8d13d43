import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name))


@pytest.fixture(scope="session")
def bunny():
    return load_golden("bunny.npz")


@pytest.fixture(scope="session")
def syn1500():
    return load_golden("synthetic1500.npz")


@pytest.fixture(scope="session")
def nonrigid_golden():
    return load_golden("nonrigid.npz")


# ---- the CPU emulation of libcpd_b200.so (tests/emu): test infrastructure only --------------------------------------
@pytest.fixture(scope="session")
def emu_lib_path():
    sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
    import build as emu_build

    return emu_build.build()


@pytest.fixture
def emulated(emu_lib_path):
    """Swap the loaded shared library for the CPU emulation for the duration of one test (tests only: the package
    itself never loads it).  Handles remember the library that created them, so late destructors stay correct."""
    from probreg_b200 import _cabi

    saved = _cabi._lib
    _cabi._lib = _cabi._load(emu_lib_path)
    assert ctypes_int(_cabi._lib, "cpd_is_emulation") == 1
    try:
        yield _cabi._lib
    finally:
        _cabi._lib = saved


def ctypes_int(handle, name):
    import ctypes

    fn = getattr(handle, name)
    fn.restype = ctypes.c_int
    return fn()
