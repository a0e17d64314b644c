"""TEST INFRASTRUCTURE -- ctypes binding of the local-map cube checker (tests/oracle_fov/fov_oracle.cpp), a restatement
of lasermap_fov_segment (src/laserMapping.cpp:361-421).  __graft_entry__.build() compiles tests/oracle_fov/
libfov_oracle.so next to the host-emulation library; lib() loads it, and rebuilds it in place only when it is missing
or older than its source (the rule of the hostemu fixture in tests/conftest.py)."""
import ctypes as C
import os
import subprocess

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_fov")
SRC = os.path.join(_DIR, "fov_oracle.cpp")
SO = os.path.join(_DIR, "libfov_oracle.so")
_lib = None

SHIPPED = (20.0, 300.0, 1.5)          # cube_side_length of every shipped config, DET_RANGE, MOV_THRESHOLD


def build(force=False):
    if force or not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(SRC):
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", SO, SRC])
    return SO


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.fovo_create.restype = C.c_void_p
        L.fovo_create.argtypes = [C.c_double, C.c_float, C.c_float]
        L.fovo_destroy.argtypes = [C.c_void_p]
        L.fovo_reset.argtypes = [C.c_void_p]
        L.fovo_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class Tracker:
    """LocalMap_Points + Localmap_Initialized of one node; step() is one lasermap_fov_segment()."""

    def __init__(self, cube_len, det_range=300.0, mov_threshold=1.5):
        self.L = lib()
        self.t = self.L.fovo_create(float(cube_len), float(det_range), float(mov_threshold))

    def step(self, pos):
        """Returns (cub_needrm (n, 6) float32 {min xyz, max xyz}, LocalMap_Points (6,) float32 after the call)."""
        p = np.ascontiguousarray(pos, np.float64).reshape(3)
        boxes = np.zeros((3, 6), np.float32)
        local = np.zeros(6, np.float32)
        n = self.L.fovo_step(self.t, p.ctypes.data_as(C.c_void_p), boxes.ctypes.data_as(C.c_void_p),
                             local.ctypes.data_as(C.c_void_p))
        return boxes[:n].copy(), local

    def reset(self):
        self.L.fovo_reset(self.t)

    def __del__(self):
        if getattr(self, "t", None):
            self.L.fovo_destroy(self.t)
            self.t = None
