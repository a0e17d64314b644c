"""TEST INFRASTRUCTURE -- ctypes binding of tests/oracle_pre/intensity_oracle.cpp, the checker of the intensity uploads:
Preprocess::process's non-feature branches (reference src/preprocess.cpp) and velodyne_handler's yaw route with each
handler's intensity line, then the stable time sort of sync_packages (src/laserMapping.cpp:551).  The library is
compiled into a temporary directory on first use, so the source tree is never written."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_pre", "intensity_oracle.cpp")
PRE_FIELDS = ("kind", "point_step", "off_x", "off_y", "off_z", "off_time", "off_tag", "off_line", "n_scans", "point_filter_num")
VELO_FIELDS = ("point_step", "off_x", "off_y", "off_z", "off_time", "off_ring", "n_scans", "point_filter_num")
YAW_DEFINED = 0               # (float)atan2((double)y, (double)x), the project's yaw (DESIGN §2)
# pcl::PointXYZINormal, the 48-byte record of pl_surf and of the intensity outputs
XYZINORMAL_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<f4"), ("normal", "<f4", 4), ("intensity", "<f4"),
                             ("curvature", "<f4"), ("pad", "<f4", 2)])
_lib = None
_tmp = None


def lib():
    global _lib, _tmp
    if _lib is None:
        _tmp = tempfile.TemporaryDirectory(prefix="intensity_oracle_")
        so = os.path.join(_tmp.name, "libintensity_oracle.so")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so, SRC])
        L = C.CDLL(so)
        L.preo_process_intensity.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.velo_process_intensity.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                             C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _lib = L
    return _lib


def process(fmt, records, off_intensity, sort=True):
    """pl_surf with its intensities (time-sorted when `sort`) as (n,) XYZINORMAL_POINT records.  fmt: a dict with
    PRE_FIELDS and "blind"; off_intensity: the intensity field's byte offset, or -1."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    out = np.zeros(max(n, 1), XYZINORMAL_POINT)
    ints = np.array([int(fmt[k]) for k in PRE_FIELDS], np.int32)
    k = lib().preo_process_intensity(ints.ctypes.data, int(off_intensity), float(fmt["blind"]), rec.ctypes.data if rec.size else None,
                                     n, int(sort), out.ctypes.data)
    assert k >= 0
    return out[:k]


def process_velodyne(fmt, records, off_intensity, mode=YAW_DEFINED, sort=True):
    """velodyne_handler (either time route) with its intensities: (xyzt (n, 4) float32, intensity (n,) float32).  fmt: a
    dict with VELO_FIELDS and "blind"."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    out = np.zeros((max(n, 1), 4), np.float32)
    inten = np.zeros(max(n, 1), np.float32)
    ints = np.array([int(fmt[k]) for k in VELO_FIELDS], np.int32)
    yaw, bad = C.c_int(), C.c_int()
    k = lib().velo_process_intensity(ints.ctypes.data, int(off_intensity), float(fmt["blind"]), rec.ctypes.data if rec.size else None,
                                     n, int(mode), int(sort), out.ctypes.data, inten.ctypes.data, C.byref(yaw), C.byref(bad))
    assert k >= 0
    return out[:k], inten[:k]
