"""TEST INFRASTRUCTURE -- the oracle's LIO handle with access to laserCloudOri of its last pass, for the tests of
flb_effect_cloud.  tests/oracle_effect/effect_oracle.cpp compiles the oracle's own sources (oracle/flo_*.cpp, unchanged)
together with the accessor flo_lio_last_ori into a library built once per process in a temporary directory; `Lio` is
pyoracle.Lio on that library, so run_pass / update / update_ikfom are the oracle's, and `last_ori()` reads the rows
(point_selected_surf && res_last <= 2.0) the last of them left."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import fastlivo_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRCS = [os.path.join(ROOT, "tests", "oracle_effect", "effect_oracle.cpp")] + \
       [os.path.join(ROOT, "oracle", f) for f in ("flo_ikfom.cpp", "flo_imu.cpp", "flo_vmap.cpp")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        po = fastlivo_loader.oracle()
        so = os.path.join(tempfile.mkdtemp(prefix="effect_oracle_"), "libeffect_oracle.so")
        # the oracle's flags (oracle/Makefile)
        subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fopenmp", "-fPIC", "-ffp-contract=off", "-Wall", "-shared",
                               "-I" + os.path.join(ROOT, "oracle"), "-o", so] + SRCS)
        L = C.CDLL(so)
        ref = po.lib()
        for name in ("flo_lio_create", "flo_lio_destroy", "flo_lio_pass", "flo_lio_update", "flo_ikfom_update"):
            getattr(L, name).restype = getattr(ref, name).restype
            getattr(L, name).argtypes = getattr(ref, name).argtypes
        L.flo_lio_last_ori.restype = C.c_int
        L.flo_lio_last_ori.argtypes = [C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class Lio(fastlivo_loader.oracle().Lio):
    """pyoracle.Lio (brute-force kNN) on the library above, plus last_ori()."""

    def __init__(self, map_xyz, scan_body):
        po = fastlivo_loader.oracle()
        self.L = lib()
        self.map = po.f32(map_xyz)
        self.scan = po.f32(scan_body)
        self.N = len(self.scan)
        self.tree = None
        self.h = self.L.flo_lio_create(po._p(self.map), len(self.map), po._p(self.scan), self.N, None, None)

    def last_ori(self):
        """laserCloudOri of the last pass run on this handle (run_pass, update or update_ikfom): its scan indices."""
        ori = np.zeros(self.N, np.int32)
        n = self.L.flo_lio_last_ori(self.h, ori.ctypes.data_as(C.c_void_p))
        return ori[:n]
