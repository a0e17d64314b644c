"""TEST INFRASTRUCTURE -- ctypes binding of tests/oracle_pre/velo_oracle.cpp, the checker of flb_lidar_upload_velodyne:
a restatement of velodyne_handler's non-feature branch (reference src/preprocess.cpp:259-297, :376-428) and the stable
time sort of sync_packages (src/laserMapping.cpp:551).  The library is compiled into a temporary directory on first use,
so the source tree is never written."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_pre", "velo_oracle.cpp")
FIELDS = ("point_step", "off_x", "off_y", "off_z", "off_time", "off_ring", "n_scans", "point_filter_num")
YAW_DEFINED, YAW_ATAN2F = 0, 1        # (float)atan2((double)y, (double)x) | libm's atan2f (the reference as built here)
MIDPOINT_ULPS = 4
_lib = None
_tmp = None


class BadRing(Exception):
    def __init__(self, record):
        super().__init__(f"record {record} has a ring >= n_scans")
        self.record = record


def lib():
    global _lib, _tmp
    if _lib is None:
        _tmp = tempfile.TemporaryDirectory(prefix="velo_oracle_")
        so = os.path.join(_tmp.name, "libvelo_oracle.so")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so, SRC])
        L = C.CDLL(so)
        L.velo_process.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int),
                                   C.POINTER(C.c_int)]
        L.velo_midpoint_flags.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.velo_yaw.argtypes = [C.c_float, C.c_float, C.c_int]
        L.velo_yaw.restype = C.c_double
        _lib = L
    return _lib


def fmt_ints(fmt):
    return np.array([int(fmt[k]) for k in FIELDS], np.int32)


def process(fmt, records, mode=YAW_DEFINED, sort=True):
    """(cloud, yaw_times): pl_surf as (n, 4) float32 x, y, z, curvature, time-sorted when `sort`, and
    !given_offset_time.  fmt: a dict with FIELDS and "blind".  Raises BadRing at a ring >= n_scans on the yaw route."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    out = np.zeros((max(n, 1), 4), np.float32)
    yaw, bad = C.c_int(), C.c_int()
    k = lib().velo_process(fmt_ints(fmt).ctypes.data, float(fmt["blind"]), rec.ctypes.data if rec.size else None, n, int(mode),
                           int(sort), out.ctypes.data, C.byref(yaw), C.byref(bad))
    if k < 0:
        raise BadRing(bad.value)
    return out[:k], bool(yaw.value)


def midpoint_flags(fmt, records, ulps=MIDPOINT_ULPS):
    """bool per record: its double atan2(y, x) lies within `ulps` double ulps of a float rounding midpoint, where a
    double atan2 from another library could round to the other float."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    flags = np.zeros(max(n, 1), np.uint8)
    lib().velo_midpoint_flags(fmt_ints(fmt).ctypes.data, rec.ctypes.data if rec.size else None, n, int(ulps), flags.ctypes.data)
    return flags[:n].astype(bool)


def yaw(x, y, mode=YAW_DEFINED):
    return lib().velo_yaw(float(x), float(y), int(mode))
