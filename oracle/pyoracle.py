"""TEST INFRASTRUCTURE -- ctypes binding of oracle/liboracle.so and oracle/_ref/libikdtree_ref.so.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.  The product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "liboracle.so")
_REF = os.path.join(_HERE, "_ref", "libikdtree_ref.so")


class State18(C.Structure):
    """flo_state18 (oracle/flo_oracle.h) == StatesGroup, reference include/common_lib.h:296-381."""
    _fields_ = [("rot", C.c_double * 9), ("pos", C.c_double * 3), ("vel", C.c_double * 3),
                ("bg", C.c_double * 3), ("ba", C.c_double * 3), ("grav", C.c_double * 3),
                ("cov", C.c_double * 324)]

    @classmethod
    def make(cls, R, p, vel=None, bg=None, ba=None, grav=None, cov=None):
        s = cls()
        s.rot[:] = np.asarray(R, np.float64).ravel()
        s.pos[:] = np.asarray(p, np.float64)
        s.vel[:] = np.zeros(3) if vel is None else vel
        s.bg[:] = np.zeros(3) if bg is None else bg
        s.ba[:] = np.zeros(3) if ba is None else ba
        s.grav[:] = np.zeros(3) if grav is None else grav
        s.cov[:] = (np.eye(18) if cov is None else np.asarray(cov, np.float64)).ravel()
        return s

    def copy(self):
        o = State18()
        C.memmove(C.byref(o), C.byref(self), C.sizeof(State18))
        return o

    @property
    def R(self):
        return np.array(self.rot[:]).reshape(3, 3)

    @property
    def p(self):
        return np.array(self.pos[:])

    @property
    def P(self):
        return np.array(self.cov[:]).reshape(18, 18)

    def vector(self):
        """All 18 'coordinates' + rotation entries flattened (for tolerance comparisons)."""
        return np.concatenate([self.rot[:], self.pos[:], self.vel[:], self.bg[:], self.ba[:], self.grav[:]])


class LioParams(C.Structure):
    _fields_ = [("R_LI", C.c_double * 9), ("t_LI", C.c_double * 3), ("laser_point_cov", C.c_double),
                ("max_iteration", C.c_int), ("conv_rot_deg", C.c_double), ("conv_pos_cm", C.c_double),
                ("nthreads", C.c_int)]


class LioReport(C.Structure):
    _fields_ = [("passes", C.c_int), ("knn_passes", C.c_int), ("n_eff_last", C.c_int),
                ("res_mean_last", C.c_double), ("rows_total", C.c_int64), ("converged_last", C.c_int)]


class Cam(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("d", C.c_double * 5)]


class VioParams(C.Structure):
    _fields_ = [("Rcl", C.c_double * 9), ("Pcl", C.c_double * 3), ("R_LI", C.c_double * 9),
                ("t_LI", C.c_double * 3), ("img_point_cov", C.c_double), ("max_iteration", C.c_int),
                ("conv_rot_deg", C.c_float), ("conv_pos_cm", C.c_float), ("force_all_passes", C.c_int)]


class VioReport(C.Structure):
    _fields_ = [("passes", C.c_int * 3), ("last_error", C.c_float * 3), ("rows_total", C.c_int64),
                ("skipped_last", C.c_int), ("cov_updated", C.c_int), ("rejects", C.c_int)]


class StateIkfom(C.Structure):
    """flo_state_ikfom == state_ikfom (include/use-ikfom.hpp:12-21); quaternions (x, y, z, w)."""
    _fields_ = [("pos", C.c_double * 3), ("rot", C.c_double * 4), ("offset_R_L_I", C.c_double * 4),
                ("offset_T_L_I", C.c_double * 3), ("vel", C.c_double * 3), ("bg", C.c_double * 3),
                ("ba", C.c_double * 3), ("grav", C.c_double * 3), ("P", C.c_double * 529)]

    def copy(self):
        o = StateIkfom()
        C.memmove(C.byref(o), C.byref(self), C.sizeof(StateIkfom))
        return o

    def vector(self):
        return np.concatenate([self.pos[:], self.rot[:], self.offset_R_L_I[:], self.offset_T_L_I[:], self.vel[:],
                               self.bg[:], self.ba[:], self.grav[:]])

    @property
    def cov(self):
        return np.array(self.P[:]).reshape(23, 23)


class IkfomParams(C.Structure):
    _fields_ = [("laser_point_cov", C.c_double), ("max_iteration", C.c_int), ("limit", C.c_double * 23),
                ("nthreads", C.c_int)]


class IkfomReport(C.Structure):
    _fields_ = [("passes", C.c_int), ("knn_passes", C.c_int), ("n_eff_last", C.c_int), ("converged_last", C.c_int),
                ("res_mean_last", C.c_double), ("rows_total", C.c_int64)]


class ImuParams(C.Structure):
    """flo_imu_params (oracle/flo_oracle.h): ImuProcess members, reference src/IMU_Processing.cpp:15-20."""
    _fields_ = [("cov_gyr", C.c_double * 3), ("cov_acc", C.c_double * 3), ("cov_bias_gyr", C.c_double * 3),
                ("cov_bias_acc", C.c_double * 3), ("G_m_s2", C.c_double), ("mean_acc_norm", C.c_double),
                ("R_LI", C.c_double * 9), ("t_LI", C.c_double * 3)]


class ImuCarry(C.Structure):
    _fields_ = [("last_lidar_end_time", C.c_double), ("acc_s_last", C.c_double * 3), ("angvel_last", C.c_double * 3)]


def imu_undistort(prm: ImuParams, carry: ImuCarry, v_imu, pcl_beg_time, pcl_end_time, x: State18, pts_xyz, offset_ms):
    """flo_imu_undistort: v_imu (K,7) [t, gyr, acc]; x and carry are updated in place.
    Returns (compensated xyz float32 (n,3), IMUpose (n_poses,22))."""
    v = np.ascontiguousarray(v_imu, np.float64)
    pts = np.ascontiguousarray(pts_xyz, np.float32).copy()
    off = np.ascontiguousarray(offset_ms, np.float32)
    poses = np.zeros((len(v), 22), np.float64)
    n = C.c_int()
    rc = lib().flo_imu_undistort(C.byref(prm), C.byref(carry), _p(v), len(v), float(pcl_beg_time), float(pcl_end_time),
                                 C.byref(x), _p(pts), _p(off), len(pts), C.byref(n), _p(poses))
    if rc:
        raise RuntimeError(f"flo_imu_undistort failed ({rc})")
    return pts, poses[:n.value]


def visual_candidates(cam: dict, Rcw, Pcw, image, world_xyz, grid_size, border, map_value):
    """flo_visual_candidates (first loop of addSparseMap).  Returns (map_value_out, winner) per grid cell."""
    c = make_cam(cam)
    img = np.ascontiguousarray(image, np.uint8)
    pts = np.ascontiguousarray(world_xyz, np.float32)
    mv = np.ascontiguousarray(map_value, np.float32).copy()
    win = np.zeros(len(mv), np.int32)
    lib().flo_visual_candidates(C.byref(c), _p(f64(Rcw)), _p(f64(Pcw)), _p(img), img.shape[1], _p(pts), len(pts),
                                int(grid_size), int(border), _p(mv), _p(win))
    return mv, win


def shi_tomasi(image, u, v):
    img = np.ascontiguousarray(image, np.uint8)
    return np.float32(lib().flo_shi_tomasi(_p(img), img.shape[1], img.shape[0], img.shape[1], int(u), int(v)))


def quat_from_R(R):
    """Rotation matrix -> quaternion (x, y, z, w), w >= 0."""
    R = np.asarray(R, np.float64)
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    if w > 1e-6:
        q = np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
    else:   # 180 degree case: pick the largest diagonal
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = np.zeros(4)
        q[i] = s / 4
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    return q / np.linalg.norm(q)


def state_ikfom_from_frame(frame, P=None):
    """state_ikfom at the propagated prior of a synthetic frame (gravity along -z, |g| = 9.8090)."""
    s = StateIkfom()
    s.pos[:] = frame["p_prop"]
    s.rot[:] = quat_from_R(frame["R_prop"])
    s.offset_R_L_I[:] = quat_from_R(frame["R_LI"])
    s.offset_T_L_I[:] = frame["t_LI"]
    s.vel[:] = frame["vel"]
    s.bg[:] = frame["bg"]
    s.ba[:] = frame["ba"]
    s.grav[:] = [0.0, 0.0, -9.8090]
    if P is None:
        P = np.diag(np.concatenate([np.full(3, 1e-3), np.full(3, 1e-4), np.full(3, 1e-6), np.full(3, 1e-6),
                                    np.full(3, 1e-2), np.full(3, 1e-4), np.full(3, 1e-3), np.full(2, 1e-5)]))
    s.P[:] = np.asarray(P, np.float64).ravel()
    return s


def ikfom_params(frame, max_iteration, nthreads=4, limit=0.001):
    p = IkfomParams()
    p.laser_point_cov = frame["cfg"].laser_point_cov
    p.max_iteration = max_iteration
    p.limit[:] = [limit] * 23
    p.nthreads = nthreads
    return p


KNN_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int)


def build(force: bool = False) -> None:
    """Compile the checker and, whenever the reference tree is available, the reference ikd-Tree (see reference_dir)."""
    need = force or not os.path.exists(_LIB) or \
        os.path.getmtime(_LIB) < max(os.path.getmtime(os.path.join(_HERE, f)) for f in ("flo_oracle.cpp", "flo_ikfom.cpp", "flo_imu.cpp", "flo_vmap.cpp", "flo_oracle.h"))
    if need:
        subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    ref = reference_dir()
    if ref and (force or not os.path.exists(_REF)):
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref", f"REF={ref}"])


def reference_dir():
    """The FAST-LIVO checkout the reference ikd-Tree is compiled from: $FASTLIVO_REFERENCE, else a checkout named
    `reference` next to this repository; None when neither holds include/ikd-Tree (or it cannot be read)."""
    for d in (os.environ.get("FASTLIVO_REFERENCE", ""), os.path.join(os.path.dirname(_HERE), "..", "reference")):
        if d and os.path.isfile(os.path.join(d, "include", "ikd-Tree", "ikd_Tree.cpp")) \
                and os.access(os.path.join(d, "include", "ikd-Tree", "ikd_Tree.cpp"), os.R_OK):
            return os.path.abspath(d)
    return None


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        L.flo_knn_brute_ctx.restype = C.c_void_p
        L.flo_knn_brute_ctx.argtypes = [C.c_void_p, C.c_int]
        L.flo_free.argtypes = [C.c_void_p]
        L.flo_knn_brute.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        L.flo_esti_plane.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
        L.flo_lio_create.restype = C.c_void_p
        L.flo_lio_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.flo_lio_destroy.argtypes = [C.c_void_p]
        L.flo_lio_pass.restype = C.c_int
        L.flo_lio_pass.argtypes = [C.c_void_p, C.POINTER(LioParams), C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 15
        L.flo_lio_update.argtypes = [C.c_void_p, C.POINTER(LioParams), C.POINTER(State18), C.POINTER(State18),
                                     C.POINTER(LioReport)]
        L.flo_vio_create.restype = C.c_void_p
        L.flo_vio_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int, C.POINTER(Cam)]
        L.flo_vio_destroy.argtypes = [C.c_void_p]
        L.flo_vio_pass.restype = C.c_float
        L.flo_vio_pass.argtypes = [C.c_void_p, C.POINTER(VioParams), C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 7
        L.flo_vio_update.argtypes = [C.c_void_p, C.POINTER(VioParams), C.POINTER(State18), C.POINTER(State18),
                                     C.POINTER(VioReport)]
        L.flo_vio_errors.argtypes = [C.c_void_p, C.c_void_p]
        L.flo_vio_update_level.restype = C.c_float
        L.flo_vio_update_level.argtypes = [C.c_void_p, C.POINTER(VioParams), C.c_int, C.c_float, C.POINTER(State18), C.POINTER(State18),
                                           C.c_void_p, C.POINTER(VioReport)]
        vp = C.c_void_p
        L.flo_vmap_create.restype = vp
        L.flo_vmap_create.argtypes = [C.POINTER(Cam), C.c_int, C.c_double, C.c_int, C.c_double]
        L.flo_vmap_destroy.argtypes = [vp]
        L.flo_vmap_counts.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.flo_vmap_map_value.argtypes = [vp, vp]
        L.flo_vmap_select.argtypes = [vp, vp, vp, vp, vp, C.c_int]
        L.flo_vmap_selected.argtypes = [vp] * 7
        L.flo_vmap_grow.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int]
        L.flo_vmap_add_observations.argtypes = [vp, vp, vp, vp, C.c_int]
        L.flo_vmap_dump_points.argtypes = [vp] * 5
        L.flo_vmap_dump_features.argtypes = [vp] * 4
        L.flo_voxel_grid.argtypes = [vp, C.c_int, C.c_float, vp]
        L.flo_colorize.argtypes = [C.POINTER(Cam)] + [vp] * 4 + [C.c_int, vp, vp]
        L.flo_world2cam.argtypes = [C.POINTER(Cam), C.c_void_p, C.c_void_p]
        L.flo_exp3.argtypes = [C.c_void_p, C.c_void_p]
        L.flo_log3.argtypes = [C.c_void_p, C.c_void_p]
        L.flo_state_boxplus.argtypes = [C.POINTER(State18), C.c_void_p]
        L.flo_state_boxminus.argtypes = [C.POINTER(State18), C.POINTER(State18), C.c_void_p]
        L.flo_inverse.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        L.flo_lio_reset.argtypes = [C.c_void_p]
        L.flo_ikfom_boxplus.argtypes = [C.POINTER(StateIkfom), C.c_void_p]
        L.flo_ikfom_boxminus.argtypes = [C.POINTER(StateIkfom), C.POINTER(StateIkfom), C.c_void_p]
        L.flo_quat_to_R.argtypes = [C.c_void_p, C.c_void_p]
        L.flo_ikfom_update.argtypes = [C.c_void_p, C.POINTER(IkfomParams), C.POINTER(StateIkfom), C.POINTER(IkfomReport)]
        L.flo_shi_tomasi.restype = C.c_float
        L.flo_shi_tomasi.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.flo_visual_candidates.argtypes = [C.POINTER(Cam), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                            C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.flo_imu_undistort.argtypes = [C.POINTER(ImuParams), C.POINTER(ImuCarry), C.c_void_p, C.c_int, C.c_double, C.c_double,
                                        C.POINTER(State18), C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_void_p]
        _lib = L
    return _lib


def ref_lib():
    """The reference's own ikd-Tree (None if oracle/_ref was never built)."""
    global _ref
    if _ref is None:
        build()
        if not os.path.exists(_REF):
            return None
        R = C.CDLL(_REF)
        R.ikdref_build.restype = C.c_void_p
        R.ikdref_build.argtypes = [C.c_void_p, C.c_int, C.c_int]
        R.ikdref_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        R.ikdref_size.argtypes = [C.c_void_p]
        R.ikdref_add_points.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float]
        R.ikdref_delete_boxes.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        R.ikdref_flatten.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        _ref = R
    return _ref


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


# ------------------------------------------------------------------------------ kNN
def knn_brute(map_xyz, q, k=5, nthreads=8):
    L = lib()
    m, q = f32(map_xyz), f32(q)
    ctx = L.flo_knn_brute_ctx(_p(m), len(m))
    idx = np.empty((len(q), k), np.int32)
    d2 = np.empty((len(q), k), np.float32)
    L.flo_knn_brute(ctx, _p(q), len(q), k, _p(idx), _p(d2), nthreads)
    L.flo_free(ctx)
    return idx, d2


class IkdTreeRef:
    """The reference's KD_TREE (include/ikd-Tree/ikd_Tree.cpp), built once, never destroyed."""

    def __init__(self, map_xyz):
        R = ref_lib()
        if R is None:
            raise RuntimeError("oracle/_ref/libikdtree_ref.so missing (built only where the reference tree is available, see reference_dir)")
        self._R = R
        m = f32(map_xyz)
        # the reference's KD_TREE constructor printf()s "Multi thread started" (ikd_Tree.cpp:170); keep
        # the caller's stdout clean (bench.py prints exactly one JSON line)
        import sys
        sys.stdout.flush()
        saved = os.dup(1)
        devnull = os.open(os.devnull, os.O_WRONLY)
        try:
            os.dup2(devnull, 1)
            self.handle = R.ikdref_build(_p(m), len(m), 3)
            C.CDLL(None).fflush(None)
        finally:
            os.dup2(saved, 1)
            os.close(saved)
            os.close(devnull)

    def knn(self, q, k=5, nthreads=4):
        q = f32(q)
        idx = np.empty((len(q), k), np.int32)
        d2 = np.empty((len(q), k), np.float32)
        self._R.ikdref_knn(self.handle, _p(q), len(q), k, _p(idx), _p(d2), nthreads)
        return idx, d2

    def add_points(self, xyz, downsample_size):
        """ikdtree.Add_Points(points, true) with downsample_size = filter_size_map (laserMapping.cpp:692-706)."""
        a = f32(xyz)
        return self._R.ikdref_add_points(self.handle, _p(a), len(a), C.c_float(downsample_size))

    def delete_boxes(self, boxes):
        b = f32(boxes).reshape(-1, 6)
        return self._R.ikdref_delete_boxes(self.handle, _p(b), len(b))

    def points(self):
        n = self._R.ikdref_flatten(self.handle, None, 0)
        out = np.empty((n, 3), np.float32)
        self._R.ikdref_flatten(self.handle, _p(out), n)
        return out

    @property
    def fn_ptr(self):
        return C.cast(self._R.ikdref_knn, C.c_void_p)


def esti_plane(nb, threshold=0.1):
    nb = f32(nb).reshape(15)
    out = np.zeros(4, np.float32)
    ok = lib().flo_esti_plane(_p(nb), C.c_float(threshold), _p(out))
    return bool(ok), out


# ------------------------------------------------------------------------------ LIO
def lio_params(frame, max_iteration, nthreads=4, early_stop=True):
    p = LioParams()
    p.R_LI[:] = f64(frame["R_LI"]).ravel()
    p.t_LI[:] = f64(frame["t_LI"])
    p.laser_point_cov = frame["cfg"].laser_point_cov
    p.max_iteration = max_iteration
    p.conv_rot_deg = 0.01 if early_stop else 0.0
    p.conv_pos_cm = 0.015 if early_stop else 0.0
    p.nthreads = nthreads
    return p


class Lio:
    def __init__(self, map_xyz, scan_body, tree: IkdTreeRef | None = None):
        self.L = lib()
        self.map = f32(map_xyz)
        self.scan = f32(scan_body)
        self.N = len(self.scan)
        self.tree = tree
        fn = tree.fn_ptr if tree is not None else None
        ctx = tree.handle if tree is not None else None
        self.h = self.L.flo_lio_create(_p(self.map), len(self.map), _p(self.scan), self.N, fn, ctx)

    def __del__(self):
        try:
            self.L.flo_lio_destroy(self.h)
        except Exception:
            pass

    def run_pass(self, prm: LioParams, R, p, rematch: bool, rows12=False):
        N = self.N
        out = dict(world=np.zeros((N, 3), np.float32), nn_idx=np.zeros((N, 5), np.int32),
                   nn_d2=np.zeros((N, 5), np.float32), pabcd=np.zeros((N, 4), np.float32),
                   pd2=np.zeros(N, np.float32), selected=np.zeros(N, np.uint8),
                   Hsub=np.zeros((N, 6)), h_x=np.zeros((N, 12)) if rows12 else None, meas=np.zeros(N),
                   sel_idx=np.zeros(N, np.int32), HTH6=np.zeros((6, 6)), HTz6=np.zeros(6),
                   HTH12=np.zeros((12, 12)) if rows12 else None, HTh12=np.zeros(12) if rows12 else None)
        tot = np.zeros(1)
        R = f64(R)
        p = f64(p)
        n = self.L.flo_lio_pass(self.h, C.byref(prm), _p(R), _p(p), int(rematch), _p(out["world"]), _p(out["nn_idx"]),
                                _p(out["nn_d2"]), _p(out["pabcd"]), _p(out["pd2"]), _p(out["selected"]), _p(out["Hsub"]),
                                _p(out["h_x"]), _p(out["meas"]), _p(out["sel_idx"]), _p(out["HTH6"]), _p(out["HTz6"]),
                                _p(out["HTH12"]), _p(out["HTh12"]), _p(tot))
        out["n"] = n
        out["total_residual"] = float(tot[0])
        for k in ("Hsub", "h_x", "meas", "sel_idx"):
            if out[k] is not None:
                out[k] = out[k][:n]
        return out

    def update(self, prm: LioParams, x: State18, x_prop: State18):
        rep = LioReport()
        self.L.flo_lio_update(self.h, C.byref(prm), C.byref(x), C.byref(x_prop), C.byref(rep))
        return rep

    def update_ikfom(self, prm: "IkfomParams", x: "StateIkfom"):
        """esekfom update_iterated_dyn_share_modified on state_ikfom (oracle/flo_ikfom.cpp)."""
        rep = IkfomReport()
        rc = self.L.flo_ikfom_update(self.h, C.byref(prm), C.byref(x), C.byref(rep))
        if rc != 0:
            raise RuntimeError(f"flo_ikfom_update failed ({rc})")
        return rep


# ------------------------------------------------------------------------------ VIO
def make_cam(cam: dict) -> Cam:
    c = Cam()
    c.width, c.height = cam["width"], cam["height"]
    c.fx, c.fy, c.cx, c.cy = cam["fx"], cam["fy"], cam["cx"], cam["cy"]
    c.d[:] = cam["d"]
    return c


def vio_params(frame, max_iteration, early_stop=True, force_all_passes=False):
    p = VioParams()
    p.Rcl[:] = f64(frame["Rcl"]).ravel()
    p.Pcl[:] = f64(frame["Pcl"])
    p.R_LI[:] = f64(frame["R_LI"]).ravel()
    p.t_LI[:] = f64(frame["t_LI"])
    p.img_point_cov = frame["cfg"].img_point_cov
    p.max_iteration = max_iteration
    p.conv_rot_deg = 0.001 if early_stop else 0.0
    p.conv_pos_cm = 0.001 if early_stop else 0.0
    p.force_all_passes = int(force_all_passes)
    return p


class Vio:
    def __init__(self, image, patch_pos, patch_ref, patch_level, cam: dict):
        self.L = lib()
        self.img = np.ascontiguousarray(image, np.uint8)
        self.pos = f64(patch_pos)
        self.patch = f32(patch_ref).reshape(len(self.pos), 192)
        self.level = np.ascontiguousarray(patch_level, np.int32)
        self.Pn = len(self.pos)
        self.cam = make_cam(cam)
        h, w = self.img.shape
        self.h = self.L.flo_vio_create(_p(self.img), w, h, w, _p(self.pos), _p(self.patch), _p(self.level), self.Pn,
                                       C.byref(self.cam))

    def __del__(self):
        try:
            self.L.flo_vio_destroy(self.h)
        except Exception:
            pass

    def run_pass(self, prm: VioParams, R, p, level: int, rows=True):
        Pn = self.Pn
        z = np.zeros(Pn * 64) if rows else None
        H = np.zeros((Pn * 64, 6)) if rows else None
        err = np.zeros(Pn, np.float32)
        HTH, HTz = np.zeros((6, 6)), np.zeros(6)
        nm = np.zeros(1, np.int64)
        sk = np.zeros(1, np.int32)
        R, p = f64(R), f64(p)
        e = self.L.flo_vio_pass(self.h, C.byref(prm), _p(R), _p(p), level, _p(z), _p(H), _p(err), _p(HTH), _p(HTz),
                                _p(nm), _p(sk))
        return dict(error=np.float32(e), z=z, H_sub=H, errors=err, HTH6=HTH, HTz6=HTz, n_meas=int(nm[0]),
                    skipped=int(sk[0]))

    def update(self, prm: VioParams, x: State18, x_prop: State18):
        rep = VioReport()
        self.L.flo_vio_update(self.h, C.byref(prm), C.byref(x), C.byref(x_prop), C.byref(rep))
        return rep

    def update_level(self, prm: VioParams, level: int, total_residual: float, x: State18, x_prop: State18, G=None):
        """LidarSelector::UpdateState alone.  G (18x18, in/out) is the member G.  Returns (last_error, G, report)."""
        G = np.zeros((18, 18)) if G is None else np.ascontiguousarray(G, np.float64)
        rep = VioReport()
        e = self.L.flo_vio_update_level(self.h, C.byref(prm), int(level), C.c_float(total_residual), C.byref(x), C.byref(x_prop),
                                        _p(G), C.byref(rep))
        return e, G, rep

    def errors(self):
        """sub_sparse_map->errors as the last executed pass left them (lidar_selection.cpp:851)."""
        err = np.zeros(self.Pn, np.float32)
        self.L.flo_vio_errors(self.h, _p(err))
        return err


class VMap:
    """flo_vmap: the CPU restatement of the visual map (addFromSparseMap / addSparseMap / addObservation)."""

    def __init__(self, cam: dict, grid_size=40, outlier_threshold=100.0, ncc_en=0, ncc_thre=0.0):
        self.L = lib()
        self.cam = make_cam(cam)
        self.w, self.h_img = cam["width"], cam["height"]
        self.h = self.L.flo_vmap_create(C.byref(self.cam), int(grid_size), float(outlier_threshold), int(ncc_en), float(ncc_thre))

    def __del__(self):
        try:
            self.L.flo_vmap_destroy(self.h)
        except Exception:
            pass

    def counts(self):
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        length = self.L.flo_vmap_counts(self.h, C.byref(a), C.byref(b), C.byref(c))
        return dict(points=a.value, features=b.value, images=c.value, length=length)

    def map_value(self):
        out = np.zeros(self.counts()["length"], np.float32)
        self.L.flo_vmap_map_value(self.h, _p(out))
        return out

    def select(self, img, Rcw, Pcw, pg_down):
        img = np.ascontiguousarray(img, np.uint8)
        pg = f32(pg_down).reshape(-1, 3)
        Rcw, Pcw = f64(Rcw), f64(Pcw)
        n = self.L.flo_vmap_select(self.h, _p(img), _p(Rcw), _p(Pcw), _p(pg), len(pg))
        index, point, level = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        error, pos, patch = np.zeros(n, np.float32), np.zeros((n, 3)), np.zeros((n, 192), np.float32)
        self.L.flo_vmap_selected(self.h, _p(index), _p(point), _p(level), _p(error), _p(pos), _p(patch))
        return dict(index=index, point=point, search_level=level, error=error, pos=pos, patch=patch)

    def grow(self, img, Rcw, Pcw, pg, frame_id):
        img = np.ascontiguousarray(img, np.uint8)
        pg = f32(pg).reshape(-1, 3)
        Rcw, Pcw = f64(Rcw), f64(Pcw)
        return self.L.flo_vmap_grow(self.h, _p(img), _p(Rcw), _p(Pcw), _p(pg), len(pg), int(frame_id))

    def add_observations(self, img, Rcw, Pcw, frame_id):
        img = np.ascontiguousarray(img, np.uint8)
        Rcw, Pcw = f64(Rcw), f64(Pcw)
        return self.L.flo_vmap_add_observations(self.h, _p(img), _p(Rcw), _p(Pcw), int(frame_id))

    def dump(self):
        c = self.counts()
        n, m = c["points"], c["features"]
        pos, value, n_obs, obs = np.zeros((n, 3)), np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros((n, 20), np.int32)
        self.L.flo_vmap_dump_points(self.h, _p(pos), _p(value), _p(n_obs), _p(obs))
        geo, score, lii = np.zeros((m, 17)), np.zeros(m, np.float32), np.zeros((m, 3), np.int32)
        self.L.flo_vmap_dump_features(self.h, _p(geo), _p(score), _p(lii))
        return dict(pos=pos, value=value, n_obs=n_obs, obs=obs, ft_geo=geo, ft_score=score, ft_level_id_img=lii)


def voxel_grid(xyz, leaf):
    """flo_voxel_grid: pcl::VoxelGrid centroids, (m, 3) float32 in ascending leaf index."""
    a = f32(xyz).reshape(-1, 3)
    out = np.zeros((len(a), 3), np.float32)
    m = lib().flo_voxel_grid(_p(a), len(a), C.c_float(leaf), _p(out))
    return out[:m].copy()


def colorize(cam: dict, Rcw, Pcw, bgr, world_xyz):
    """flo_colorize: (rgb (n, 3) uint8, valid (n,) bool)."""
    c = make_cam(cam)
    img = np.ascontiguousarray(bgr, np.uint8)
    pts = f32(world_xyz).reshape(-1, 3)
    R, P = f64(Rcw), f64(Pcw)
    rgb = np.zeros((len(pts), 3), np.uint8)
    val = np.zeros(len(pts), np.uint8)
    lib().flo_colorize(C.byref(c), _p(R), _p(P), _p(img), _p(pts), len(pts), _p(rgb), _p(val))
    return rgb, val.astype(bool)


def world2cam(cam: dict, pf):
    c = make_cam(cam)
    pf = f64(pf)
    out = np.zeros(2)
    lib().flo_world2cam(C.byref(c), _p(pf), _p(out))
    return out


def state_from_frame(frame, prop=True) -> State18:
    R = frame["R_prop"] if prop else frame["R_true"]
    p = frame["p_prop"] if prop else frame["p_true"]
    return State18.make(R, p, frame["vel"], frame["bg"], frame["ba"], frame["grav"], frame["cov"])
