"""TEST INFRASTRUCTURE -- ctypes binding of tests/oracle_pre/feat_oracle.cpp, the checker of flb_lidar_upload_features
and flb_lidar_upload_velodyne_features: a sequential restatement of the three feature branches of Preprocess
(reference src/preprocess.cpp:94-135, :174-227, :299-373), give_feature, plane_judge and edge_jump_judge, then the
stable time sort.  The library is compiled into a temporary directory on first use, so the source tree is never written."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_pre", "feat_oracle.cpp")
FIELDS = ("kind", "point_step", "off_x", "off_y", "off_z", "off_time", "off_tag", "off_line", "n_scans", "point_filter_num")
FLAGS = ("step0", "step1", "step2", "edge_plane_join", "real_plane_join", "jump1", "jump2", "jump3", "jump4", "wire",
         "small_fire", "small_alternate", "last_dista", "write_past_end", "nan_group", "head_past_end", "full_chunk",
         "partial_chunk", "partial_dropped", "empty_ring", "line_too_short")
_lib = None
_tmp = None


def lib():
    global _lib, _tmp
    if _lib is None:
        _tmp = tempfile.TemporaryDirectory(prefix="feat_oracle_")
        so = os.path.join(_tmp.name, "libfeat_oracle.so")
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-Wall", "-shared", "-o", so, SRC])
        L = C.CDLL(so)
        L.feat_process.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int)]
        L.feat_n_flags.restype = C.c_int
        assert L.feat_n_flags() == len(FLAGS)
        _lib = L
    return _lib


def fmt_ints(fmt):
    return np.array([int(fmt[k]) for k in FIELDS], np.int32)


def process(fmt, records, dis_b=0.0, sort=True):
    """(pl_surf, ftypes, flags, yaw_times): pl_surf as (n, 4) float32 x, y, z, curvature (time-sorted when `sort`),
    the final type of every line point in line order, and a dict of how often each flagged case occurred."""
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // int(fmt["point_step"])
    out = np.zeros((max(n, 1), 4), np.float32)
    ft = np.zeros(max(n, 1), np.int32)
    nft, yaw = C.c_int(), C.c_int()
    flags = np.zeros(len(FLAGS), np.int64)
    m = lib().feat_process(fmt_ints(fmt).ctypes.data, float(fmt["blind"]), float(dis_b), rec.ctypes.data if rec.size else None, n,
                           int(sort), out.ctypes.data, ft.ctypes.data, C.byref(nft), flags.ctypes.data, C.byref(yaw))
    return out[:m], ft[:nft.value], dict(zip(FLAGS, flags.tolist())), bool(yaw.value)
