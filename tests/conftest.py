import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import fastlivo_loader  # noqa: E402


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


@pytest.fixture(scope="session")
def flb():
    return fastlivo_loader.load()


@pytest.fixture(scope="session")
def po():
    """The CPU oracle (checker)."""
    return fastlivo_loader.oracle()


_frames = {}


@pytest.fixture(scope="session")
def frames(flb):
    def get(name):
        if name not in _frames:
            _frames[name] = flb.synth.make_frame(name)
        return _frames[name]
    return get


@pytest.fixture(scope="session")
def hostemu():
    """The product's per-thread device math compiled for the host (tests/hostemu)."""
    import ctypes as C
    d = os.path.join(ROOT, "tests", "hostemu")
    so = os.path.join(d, "libhostemu.so")
    srcs = [os.path.join(d, "hostemu.cpp"), os.path.join(ROOT, "fast-livo_b200", "csrc", "flb_device.cuh")]
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall",
                               "-Wno-unknown-pragmas", "-shared", "-o", so, srcs[0]])
    return C.CDLL(so)


def has_gpu():
    try:
        import ctypes
        cuda = ctypes.CDLL("libcuda.so.1")
        if cuda.cuInit(0) != 0:
            return False
        n = ctypes.c_int()
        cuda.cuDeviceGetCount(ctypes.byref(n))
        return n.value > 0
    except OSError:
        return False


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)
