"""TEST INFRASTRUCTURE -- ctypes binding of tests/oracle_pre/pre_oracle.cpp, the checker of flb_lidar_upload: a
restatement of Preprocess::process's non-feature branches (reference src/preprocess.cpp), the time sort of
sync_packages (src/laserMapping.cpp:551, stable) and UndistortPcl's window (src/IMU_Processing.cpp:624-646).  The
library is compiled into a temporary directory on first use, so the source tree is never written."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_pre", "pre_oracle.cpp")
_lib = None
_tmp = None

FIELDS = ("kind", "point_step", "off_x", "off_y", "off_z", "off_time", "off_tag", "off_line", "n_scans", "point_filter_num")


def lib():
    global _lib, _tmp
    if _lib is None:
        _tmp = tempfile.TemporaryDirectory(prefix="pre_oracle_")
        so = os.path.join(_tmp.name, "libpre_oracle.so")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so, SRC])
        L = C.CDLL(so)
        L.preo_process.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.preo_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p]
        _lib = L
    return _lib


def _fmt_ints(fmt):
    return np.array([int(fmt[k]) for k in FIELDS], np.int32)


def process48(fmt, records, sort=True):
    """pl_surf as the reference holds it: (n, 12) float32 pcl::PointXYZINormal (x, y, z at 0..2, curvature at 9),
    time-sorted when `sort`.  fmt: a dict with FIELDS and "blind".  None for a Velodyne cloud without times."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    out = np.zeros((max(n, 1), 12), np.float32)
    ints = _fmt_ints(fmt)
    k = lib().preo_process(ints.ctypes.data, float(fmt["blind"]), rec.ctypes.data if rec.size else None, n, int(sort), out.ctypes.data)
    return None if k < 0 else out[:k]


def process(fmt, records, sort=True):
    """(n, 4) float32 x, y, z, curvature of process48."""
    p = process48(fmt, records, sort)
    return None if p is None else np.ascontiguousarray(p[:, [0, 1, 2, 9]])


def window(points48, index_now, pcl_offset_time):
    """pcl_out of UndistortPcl's window, (n_taken, 12) float32, from lidar_scan_index_now = index_now."""
    p = np.ascontiguousarray(points48, np.float32)
    out = np.zeros((max(len(p) - index_now, 1), 12), np.float32)
    k = lib().preo_window(p.ctypes.data, len(p), int(index_now), float(pcl_offset_time), out.ctypes.data)
    return out[:k]
