"""ctypes binding of libfastlivo_b200.so (include/fastlivo_b200.h).

No CPU fallback: if the library is missing it is built with nvcc; if there is no CUDA
device ``Handle()`` raises ``FlbError`` (FLB_ERR_NO_DEVICE).  Nothing here imports the
oracle.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfastlivo_b200.so")

FLB_OK = 0
ERRORS = {-1: "FLB_ERR_INVALID", -2: "FLB_ERR_CUDA", -3: "FLB_ERR_NO_DEVICE", -4: "FLB_ERR_STATE",
          -5: "FLB_ERR_NUMERIC", -6: "FLB_ERR_COMM", -7: "FLB_ERR_TIMEOUT"}


class FlbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"{ERRORS.get(code, code)}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("device", C.c_int), ("cell_size", C.c_double), ("knn_max_d2", C.c_double),
                ("plane_threshold", C.c_double), ("persistent", C.c_int), ("reserved", C.c_int * 7)]


class ImuParams(C.Structure):
    """flb_imu_params (include/fastlivo_b200.h)."""
    _fields_ = [("cov_gyr", C.c_double * 3), ("cov_acc", C.c_double * 3), ("cov_bias_gyr", C.c_double * 3),
                ("cov_bias_acc", C.c_double * 3), ("G_m_s2", C.c_double), ("mean_acc_norm", C.c_double),
                ("R_LI", C.c_double * 9), ("t_LI", C.c_double * 3)]


class ImuCarry(C.Structure):
    """flb_imu_carry: last_lidar_end_time_, acc_s_last, angvel_last of ImuProcess."""
    _fields_ = [("last_lidar_end_time", C.c_double), ("acc_s_last", C.c_double * 3), ("angvel_last", C.c_double * 3)]


class LidarFormat(C.Structure):
    """flb_lidar_format: where the fields of one driver record sit, and Preprocess's parameters."""
    _fields_ = [("kind", C.c_int), ("point_step", C.c_int), ("off_x", C.c_int), ("off_y", C.c_int), ("off_z", C.c_int),
                ("off_time", C.c_int), ("off_tag", C.c_int), ("off_line", C.c_int), ("n_scans", C.c_int),
                ("point_filter_num", C.c_int), ("blind", C.c_double)]


class VelodyneFormat(C.Structure):
    """flb_velodyne_format: where a Velodyne PointCloud2 record keeps x, y, z, time (-1: none) and ring, at any offset."""
    _fields_ = [("point_step", C.c_int), ("off_x", C.c_int), ("off_y", C.c_int), ("off_z", C.c_int), ("off_time", C.c_int),
                ("off_ring", C.c_int), ("n_scans", C.c_int), ("point_filter_num", C.c_int), ("blind", C.c_double)]


class State18(C.Structure):
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

    @classmethod
    def from_frame(cls, frame, prop=True):
        R = frame["R_prop"] if prop else frame["R_true"]
        p = frame["p_prop"] if prop else frame["p_true"]
        return cls.make(R, p, frame["vel"], frame["bg"], frame["ba"], frame["grav"], frame["cov"])

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
        return np.concatenate([self.rot[:], self.pos[:], self.vel[:], self.bg[:], self.ba[:], self.grav[:]])


class LioParams(C.Structure):
    _fields_ = [("R_LI", C.c_double * 9), ("t_LI", C.c_double * 3), ("laser_point_cov", C.c_double),
                ("max_iteration", C.c_int), ("conv_rot_deg", C.c_double), ("conv_pos_cm", C.c_double)]


class LioReport(C.Structure):
    _fields_ = [("passes", C.c_int), ("knn_passes", C.c_int), ("n_eff_last", C.c_int),
                ("res_mean_last", C.c_double), ("rows_total", C.c_int64), ("converged_last", C.c_int),
                ("status", C.c_int)]


class NormalEq(C.Structure):
    _fields_ = [("width", C.c_int), ("n_eff", C.c_int), ("sum_abs_res", C.c_double),
                ("HTH", C.c_double * 144), ("HTh", C.c_double * 12)]


class StateIkfom(C.Structure):
    """flb_state_ikfom == state_ikfom (reference include/use-ikfom.hpp:12-21); quaternions (x, y, z, w)."""
    _fields_ = [("pos", C.c_double * 3), ("rot", C.c_double * 4), ("offset_R_L_I", C.c_double * 4),
                ("offset_T_L_I", C.c_double * 3), ("vel", C.c_double * 3), ("bg", C.c_double * 3),
                ("ba", C.c_double * 3), ("grav", C.c_double * 3), ("P", C.c_double * 529)]

    def vector(self):
        return np.concatenate([self.pos[:], self.rot[:], self.offset_R_L_I[:], self.offset_T_L_I[:], self.vel[:],
                               self.bg[:], self.ba[:], self.grav[:]])

    @property
    def cov(self):
        return np.array(self.P[:]).reshape(23, 23)


class IkfomParams(C.Structure):
    _fields_ = [("laser_point_cov", C.c_double), ("max_iteration", C.c_int), ("limit", C.c_double * 23)]


class IkfomReport(C.Structure):
    _fields_ = [("passes", C.c_int), ("knn_passes", C.c_int), ("n_eff_last", C.c_int), ("converged_last", C.c_int),
                ("res_mean_last", C.c_double), ("rows_total", C.c_int64), ("status", C.c_int)]


class Camera(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_double), ("fy", C.c_double),
                ("cx", C.c_double), ("cy", C.c_double), ("d", C.c_double * 5)]


class VioParams(C.Structure):
    _fields_ = [("Rcl", C.c_double * 9), ("Pcl", C.c_double * 3), ("R_LI", C.c_double * 9),
                ("t_LI", C.c_double * 3), ("img_point_cov", C.c_double), ("max_iteration", C.c_int),
                ("conv_rot_deg", C.c_float), ("conv_pos_cm", C.c_float), ("force_all_passes", C.c_int)]


class VioReport(C.Structure):
    _fields_ = [("passes", C.c_int * 3), ("last_error", C.c_float * 3), ("rows_total", C.c_int64),
                ("skipped_last", C.c_int), ("cov_updated", C.c_int), ("status", C.c_int)]


class FrameInputs(C.Structure):
    """flb_frame_inputs (include/fastlivo_b200.h)."""
    _fields_ = [("scan_xyz", C.c_void_p), ("n_scan", C.c_int), ("scan_stride", C.c_int),
                ("gray", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("stride_bytes", C.c_int),
                ("patch_pos", C.c_void_p), ("patch", C.c_void_p), ("search_level", C.c_void_p), ("Pn", C.c_int),
                ("x", C.POINTER(State18)), ("x_prop", C.POINTER(State18))]


class VmapParams(C.Structure):
    """flb_vmap_params (include/fastlivo_b200.h)."""
    _fields_ = [("grid_size", C.c_int), ("ncc_en", C.c_int), ("outlier_threshold", C.c_double), ("ncc_thre", C.c_double),
                ("Rcl", C.c_double * 9), ("Pcl", C.c_double * 3), ("R_LI", C.c_double * 9), ("t_LI", C.c_double * 3)]


class VioEq(C.Structure):
    _fields_ = [("HTH", C.c_double * 36), ("HTz", C.c_double * 6), ("error", C.c_float),
                ("n_meas", C.c_int64), ("skipped", C.c_int)]


class FovParams(C.Structure):
    """flb_fov_params: cube_side_length, DET_RANGE, MOV_THRESHOLD of lasermap_fov_segment."""
    _fields_ = [("cube_len", C.c_double), ("det_range", C.c_float), ("mov_threshold", C.c_float)]


CLOUD_SCAN, CLOUD_UNDISTORTED = 0, 1       # flb_world_cloud sources (FLB_CLOUD_*)
# flb_rgb_cloud's 32-byte record, the layout of pcl::PointXYZRGB: x y z, w = data[3] (1.0), b g r a, 12 zero bytes
RGB_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<f4"), ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"),
                      ("pad", "u1", 12)])
# the 48-byte record of the intensity outputs (flb_lidar_download_points, flb_world_cloud_points,
# flb_effect_cloud_download_points, flb_lidar_save_download), the layout of pcl::PointXYZINormal: x y z, w = data[3] (1.0),
# normal and data_n (zero), intensity, curvature, 8 zero bytes
XYZINORMAL_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<f4"), ("normal", "<f4", 4), ("intensity", "<f4"),
                             ("curvature", "<f4"), ("pad", "<f4", 2)])
LIDAR_LIVOX, LIDAR_VELODYNE, LIDAR_OUSTER, LIDAR_XT32 = 1, 2, 3, 4    # flb_lidar_format.kind (FLB_LIDAR_*)
GRAY_CV4, GRAY_CV3 = 0, 1                  # flb_image_upload_bgr's cvtColor rules (FLB_GRAY_*)
# flb_image_upload_msg's encodings (FLB_ENC_*), keyed by sensor_msgs::Image's encoding string
ENCODINGS = {"bgr8": 0, "rgb8": 1, "mono8": 2, "bgra8": 3, "rgba8": 4,
             "bayer_rggb8": 5, "bayer_bggr8": 6, "bayer_gbrg8": 7, "bayer_grbg8": 8}
ENC_BYTES = {0: 3, 1: 3, 2: 1, 3: 4, 4: 4, 5: 1, 6: 1, 7: 1, 8: 1}       # bytes per pixel

# every symbol include/fastlivo_b200.h declares (checked by the CPU-only test tier)
SYMBOLS = ["flb_abi_version", "flb_create", "flb_destroy", "flb_last_error", "flb_set_stream", "flb_synchronize", "flb_host_alloc", "flb_host_free",
           "flb_map_upload", "flb_map_add_points", "flb_map_add_scan", "flb_map_delete_boxes", "flb_map_size", "flb_map_download", "flb_scan_upload", "flb_scan_from_undistorted", "flb_map_upload_scan", "flb_knn", "flb_lio_pass", "flb_lio_export", "flb_lio_update", "flb_lio_update_ikfom",
           "flb_image_upload", "flb_patches_upload", "flb_camera_set", "flb_vio_pass", "flb_vio_export",
           "flb_vio_update", "flb_state_upload", "flb_state_download", "flb_lio_update_enqueue",
           "flb_vio_update_enqueue", "flb_state_reset_enqueue", "flb_state_set_prior_enqueue", "flb_profile_start", "flb_profile_stop",
           "flb_launch_count", "flb_trace_enable", "flb_trace_download", "flb_comm_unique_id", "flb_comm_init", "flb_comm_destroy", "flb_p2p_export", "flb_p2p_attach", "flb_p2p_detach",
           "flb_imu_undistort", "flb_visual_candidates", "flb_vio_errors",
           "flb_vio_update_level", "flb_state_download_enqueue", "flb_state_download_wait", "flb_frame_enqueue",
           "flb_vmap_reset", "flb_vmap_select", "flb_vmap_selected", "flb_vmap_grow", "flb_vmap_add_observations", "flb_vmap_counts",
           "flb_vmap_map_value", "flb_vmap_dump", "flb_vmap_reclaim", "flb_vmap_usage", "flb_vmap_keyframe", "flb_colorize", "flb_voxel_grid",
           "flb_world_cloud", "flb_world_cloud_download", "flb_effect_cloud", "flb_effect_cloud_download", "flb_vmap_select_cloud", "flb_vmap_grow_cloud", "flb_colorize_cloud",
           "flb_rgb_cloud", "flb_rgb_cloud_download", "flb_rgb_save_begin", "flb_rgb_save_size", "flb_rgb_save_download", "flb_rgb_save_end",
           "flb_batch_begin", "flb_batch_set_frame", "flb_batch_state_reset_enqueue", "flb_batch_update_enqueue", "flb_batch_state_download",
           "flb_debug_set_packet_epoch", "flb_debug_block_stamps", "flb_debug_vio_stamps", "flb_debug_scan_order", "flb_debug_set_scan_sort",
           "flb_map_grid_info", "flb_debug_set_map_index", "flb_map_fov_segment", "flb_map_fov_reset",
           "flb_image_upload_bgr", "flb_image_download",
           "flb_lidar_upload", "flb_lidar_download", "flb_imu_undistort_lidar", "flb_lidar_upload_velodyne",
           "flb_lidar_upload_features", "flb_lidar_upload_velodyne_features", "flb_image_upload_msg",
           "flb_keypatch_image", "flb_lidar_upload_intensity", "flb_lidar_upload_velodyne_intensity", "flb_lidar_download_points",
           "flb_world_cloud_points", "flb_effect_cloud_download_points", "flb_lidar_save_begin", "flb_lidar_save_size",
           "flb_lidar_save_download", "flb_lidar_save_end"]


def lib_path() -> str:
    return _SO


def build(force: bool = False) -> str:
    """Compile libfastlivo_b200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    srcs = [os.path.join(_HERE, "csrc", f) for f in os.listdir(os.path.join(_HERE, "csrc"))]
    srcs.append(os.path.join(_HERE, "..", "include", "fastlivo_b200.h"))
    stale = (not os.path.exists(_SO)) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs)
    if force or stale:
        if not os.path.exists("/usr/local/cuda/bin/nvcc") and os.path.exists(_SO):
            return _SO  # a box without nvcc: use the prebuilt library that travelled with the repo
        subprocess.check_call(["bash", os.path.join(_HERE, "build.sh")])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        vp = C.c_void_p
        L.flb_abi_version.restype = C.c_int
        L.flb_last_error.restype = C.c_char_p
        L.flb_last_error.argtypes = [vp]
        L.flb_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
        L.flb_destroy.argtypes = [vp]
        L.flb_set_stream.argtypes = [vp, vp]
        L.flb_synchronize.argtypes = [vp]
        L.flb_host_alloc.argtypes = [vp, C.c_size_t, C.POINTER(vp)]
        L.flb_host_free.argtypes = [vp, vp]
        L.flb_map_upload.argtypes = [vp, vp, C.c_int, C.c_int]
        L.flb_scan_upload.argtypes = [vp, vp, C.c_int, C.c_int]
        L.flb_scan_from_undistorted.argtypes = [vp, C.c_float, C.POINTER(C.c_int)]
        L.flb_map_upload_scan.argtypes = [vp]
        L.flb_map_add_points.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float]
        L.flb_map_add_scan.argtypes = [vp, C.POINTER(LioParams), vp, vp, C.c_float]
        L.flb_map_delete_boxes.argtypes = [vp, vp, C.c_int]
        L.flb_map_fov_segment.argtypes = [vp, C.POINTER(FovParams), vp, C.POINTER(C.c_int), vp, vp, C.POINTER(C.c_int)]
        L.flb_map_fov_reset.argtypes = [vp]
        L.flb_map_size.argtypes = [vp]
        L.flb_map_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_knn.argtypes = [vp, vp, C.c_int, vp, vp]
        L.flb_lio_pass.argtypes = [vp, C.POINTER(LioParams), vp, vp, C.c_int, C.c_int, C.POINTER(NormalEq)]
        L.flb_lio_export.argtypes = [vp] + [vp] * 9 + [C.POINTER(C.c_int)]
        L.flb_lio_update.argtypes = [vp, C.POINTER(LioParams), C.POINTER(State18), C.POINTER(State18), C.POINTER(LioReport)]
        L.flb_lio_update_ikfom.argtypes = [vp, C.POINTER(IkfomParams), C.POINTER(StateIkfom), C.POINTER(IkfomReport)]
        L.flb_imu_undistort.argtypes = [vp, C.POINTER(ImuParams), C.POINTER(ImuCarry), vp, C.c_int, C.c_double, C.c_double,
                                        vp, C.c_int, C.c_int, C.c_int, vp, vp, C.POINTER(C.c_int)]
        L.flb_lidar_upload.argtypes = [vp, C.POINTER(LidarFormat), vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_float)]
        L.flb_lidar_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_lidar_upload_velodyne.argtypes = [vp, C.POINTER(VelodyneFormat), vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_float),
                                                C.POINTER(C.c_int)]
        L.flb_lidar_upload_features.argtypes = [vp, C.POINTER(LidarFormat), C.c_double, vp, C.c_int, C.POINTER(C.c_int),
                                                C.POINTER(C.c_float)]
        L.flb_lidar_upload_velodyne_features.argtypes = [vp, C.POINTER(VelodyneFormat), C.c_double, vp, C.c_int, C.POINTER(C.c_int),
                                                         C.POINTER(C.c_float), C.POINTER(C.c_int)]
        L.flb_lidar_upload_intensity.argtypes = [vp, C.POINTER(LidarFormat), C.c_int, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_float)]
        L.flb_lidar_upload_velodyne_intensity.argtypes = [vp, C.POINTER(VelodyneFormat), C.c_int, vp, C.c_int, C.POINTER(C.c_int),
                                                          C.POINTER(C.c_float), C.POINTER(C.c_int)]
        L.flb_lidar_download_points.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_world_cloud_points.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_effect_cloud_download_points.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_lidar_save_begin.argtypes = [vp, C.c_int64]
        L.flb_lidar_save_size.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.flb_lidar_save_download.argtypes = [vp, C.c_int64, C.c_int64, vp]
        L.flb_lidar_save_end.argtypes = [vp]
        L.flb_imu_undistort_lidar.argtypes = [vp, C.POINTER(ImuParams), C.POINTER(ImuCarry), vp, C.c_int, C.c_double, C.c_double,
                                              C.c_double, C.c_int, C.POINTER(C.c_int), vp, C.c_int, vp, C.POINTER(C.c_int)]
        L.flb_visual_candidates.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
        L.flb_image_upload.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_image_upload_bgr.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int]
        L.flb_image_upload_msg.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.flb_keypatch_image.argtypes = [vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_image_download.argtypes = [vp, vp, vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.flb_patches_upload.argtypes = [vp, vp, vp, vp, C.c_int]
        L.flb_camera_set.argtypes = [vp, C.POINTER(Camera)]
        L.flb_vio_pass.argtypes = [vp, C.POINTER(VioParams), vp, vp, C.c_int, C.POINTER(VioEq)]
        L.flb_vio_export.argtypes = [vp, vp, vp, vp]
        L.flb_vio_errors.argtypes = [vp, vp, C.c_int]
        L.flb_debug_scan_order.argtypes = [vp, vp, C.c_int]
        L.flb_debug_set_scan_sort.argtypes = [vp, C.c_int]
        L.flb_map_grid_info.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.flb_debug_set_map_index.argtypes = [vp, C.c_int]
        L.flb_vio_update_level.argtypes = [vp, C.POINTER(VioParams), C.c_int, C.c_float, C.POINTER(State18), C.POINTER(State18),
                                           C.POINTER(C.c_float), vp, C.POINTER(VioReport)]
        L.flb_batch_begin.argtypes = [vp, C.c_int, C.c_int]
        L.flb_batch_set_frame.argtypes = [vp, C.c_int, vp, C.c_int, C.c_int, C.POINTER(State18), C.POINTER(State18)]
        L.flb_batch_state_reset_enqueue.argtypes = [vp]
        L.flb_batch_update_enqueue.argtypes = [vp, C.POINTER(LioParams), C.POINTER(VioParams)]
        L.flb_batch_state_download.argtypes = [vp, C.c_int, C.POINTER(State18), C.POINTER(LioReport), C.POINTER(VioReport)]
        L.flb_voxel_grid.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_colorize.argtypes = [vp, vp, vp, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp]
        L.flb_world_cloud.argtypes = [vp, C.POINTER(LioParams), vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_world_cloud_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_effect_cloud.argtypes = [vp, C.POINTER(LioParams), vp, vp, C.POINTER(C.c_int)]
        L.flb_effect_cloud_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_vmap_select_cloud.argtypes = [vp, vp, vp, C.c_float, vp]
        L.flb_vmap_grow_cloud.argtypes = [vp, vp, vp, C.c_int]
        L.flb_colorize_cloud.argtypes = [vp, vp, vp, vp, C.c_int, vp, vp]
        L.flb_rgb_cloud.argtypes = [vp, vp, vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_rgb_cloud_download.argtypes = [vp, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_rgb_save_begin.argtypes = [vp, C.c_int64]
        L.flb_rgb_save_size.argtypes = [vp, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        L.flb_rgb_save_download.argtypes = [vp, C.c_int64, C.c_int64, vp]
        L.flb_rgb_save_end.argtypes = [vp]
        L.flb_vmap_reset.argtypes = [vp, C.POINTER(VmapParams)]
        L.flb_vmap_select.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, vp]
        L.flb_vmap_selected.argtypes = [vp, C.c_int, C.POINTER(C.c_int)] + [vp] * 6
        L.flb_vmap_grow.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, C.c_int]
        L.flb_vmap_add_observations.argtypes = [vp, vp, vp, C.c_int]
        L.flb_vmap_counts.argtypes = [vp] + [C.POINTER(C.c_int)] * 5
        L.flb_vmap_map_value.argtypes = [vp, vp, C.c_int]
        L.flb_vmap_dump.argtypes = [vp, C.c_int, C.c_int] + [vp] * 7
        L.flb_vmap_reclaim.argtypes = [vp]
        L.flb_vmap_usage.argtypes = [vp] + [C.POINTER(C.c_int)] * 7 + [C.POINTER(C.c_int64)]
        L.flb_vmap_keyframe.argtypes = [vp, C.c_int, vp, C.c_int]
        L.flb_vio_update.argtypes = [vp, C.POINTER(VioParams), C.POINTER(State18), C.POINTER(State18), C.POINTER(VioReport)]
        L.flb_state_upload.argtypes = [vp, C.POINTER(State18), C.POINTER(State18)]
        L.flb_state_download.argtypes = [vp, C.POINTER(State18), C.POINTER(LioReport), C.POINTER(VioReport)]
        L.flb_lio_update_enqueue.argtypes = [vp, C.POINTER(LioParams)]
        L.flb_frame_enqueue.argtypes = [vp, C.POINTER(FrameInputs), C.POINTER(LioParams), C.POINTER(VioParams), C.c_int]
        L.flb_state_download_enqueue.argtypes = [vp, C.c_int]
        L.flb_state_download_wait.argtypes = [vp, C.c_int, C.POINTER(State18), C.POINTER(LioReport), C.POINTER(VioReport)]
        L.flb_vio_update_enqueue.argtypes = [vp, C.POINTER(VioParams)]
        L.flb_state_reset_enqueue.argtypes = [vp]
        L.flb_state_set_prior_enqueue.argtypes = [vp]
        L.flb_profile_start.argtypes = [vp]
        L.flb_profile_stop.argtypes = [vp, vp, vp]
        L.flb_trace_enable.argtypes = [vp, C.c_int]
        L.flb_trace_download.argtypes = [vp, C.c_int, vp, C.c_int, C.POINTER(C.c_int)]
        L.flb_launch_count.restype = C.c_int64
        L.flb_launch_count.argtypes = [vp]
        L.flb_comm_unique_id.argtypes = [vp]
        L.flb_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
        L.flb_comm_destroy.argtypes = [vp]
        L.flb_p2p_export.argtypes = [vp, vp]
        L.flb_p2p_attach.argtypes = [vp, C.c_int, C.c_int, vp]
        L.flb_p2p_detach.argtypes = [vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def lio_params(frame, max_iteration, early_stop=True) -> LioParams:
    p = LioParams()
    p.R_LI[:] = np.asarray(frame["R_LI"], np.float64).ravel()
    p.t_LI[:] = np.asarray(frame["t_LI"], np.float64)
    p.laser_point_cov = frame["cfg"].laser_point_cov
    p.max_iteration = max_iteration
    p.conv_rot_deg = 0.01 if early_stop else 0.0
    p.conv_pos_cm = 0.015 if early_stop else 0.0
    return p


def vio_params(frame, max_iteration, early_stop=True, force_all_passes=False) -> VioParams:
    p = VioParams()
    p.Rcl[:] = np.asarray(frame["Rcl"], np.float64).ravel()
    p.Pcl[:] = np.asarray(frame["Pcl"], np.float64)
    p.R_LI[:] = np.asarray(frame["R_LI"], np.float64).ravel()
    p.t_LI[:] = np.asarray(frame["t_LI"], np.float64)
    p.img_point_cov = frame["cfg"].img_point_cov
    p.max_iteration = max_iteration
    p.conv_rot_deg = 0.001 if early_stop else 0.0
    p.conv_pos_cm = 0.001 if early_stop else 0.0
    p.force_all_passes = int(force_all_passes)
    return p


class Handle:
    """Owns one flb_handle.  Method names follow the C ABI."""

    def __init__(self, device=0, cell_size=0.6, knn_max_d2=5.0, plane_threshold=0.1, persistent=1):
        self.L = lib()
        cfg = Config()
        cfg.device, cfg.cell_size, cfg.knn_max_d2, cfg.plane_threshold, cfg.persistent = \
            device, cell_size, knn_max_d2, plane_threshold, persistent
        self.h = C.c_void_p()
        rc = self.L.flb_create(C.byref(cfg), C.byref(self.h))
        if rc != FLB_OK:
            raise FlbError(rc, self.L.flb_last_error(None).decode())
        self.N = self.M = self.Pn = 0
        self._wc_n = 0                  # points of the world cloud flb_world_cloud last built
        self._ef_n = 0                  # points of the effect cloud flb_effect_cloud last built
        self._rc_n = 0                  # records of the coloured cloud flb_rgb_cloud last built

    def close(self):
        if getattr(self, "h", None):
            self.L.flb_synchronize(self.h)
            for ptr in getattr(self, "_pinned", []):
                self.L.flb_host_free(self.h, ptr)
            self._pinned = []
            self.L.flb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != FLB_OK:
            raise FlbError(rc, self.L.flb_last_error(self.h).decode())

    # ---- uploads
    def map_upload(self, xyz):
        a = np.ascontiguousarray(xyz, np.float32)
        self._ck(self.L.flb_map_upload(self.h, _p(a), a.shape[0], a.shape[1]))
        self.M = a.shape[0]

    def map_add_points(self, world_xyz, downsample_size):
        a = np.ascontiguousarray(world_xyz, np.float32)
        self._ck(self.L.flb_map_add_points(self.h, _p(a), a.shape[0], a.shape[1], C.c_float(downsample_size)))
        self.M = self.L.flb_map_size(self.h)

    def map_add_scan(self, prm, downsample_size, R=None, p=None):
        """flb_map_add_scan: Add_Points of the uploaded scan at pose (R, p), or at the device state x when both are None."""
        R = None if R is None else np.ascontiguousarray(R, np.float64)
        p = None if p is None else np.ascontiguousarray(p, np.float64)
        self._ck(self.L.flb_map_add_scan(self.h, C.byref(prm) if prm is not None else None, _p(R), _p(p), C.c_float(downsample_size)))
        self.M = self.L.flb_map_size(self.h)

    def map_delete_boxes(self, boxes):
        b = np.ascontiguousarray(boxes, np.float32).reshape(-1, 6)
        self._ck(self.L.flb_map_delete_boxes(self.h, _p(b), len(b)))
        self.M = self.L.flb_map_size(self.h)

    def map_fov_segment(self, cube_len, det_range=300.0, mov_threshold=1.5, pos=None):
        """flb_map_fov_segment: lasermap_fov_segment + Delete_Point_Boxes at sensor position `pos`, or at the device state
        when None.  Returns (boxes (n, 6) float32, local_box (6,) float32, n_deleted)."""
        prm = FovParams(float(cube_len), float(det_range), float(mov_threshold))
        p = None if pos is None else np.ascontiguousarray(pos, np.float64).reshape(3)
        nb, nd = C.c_int(), C.c_int()
        boxes = np.zeros((3, 6), np.float32)
        local = np.zeros(6, np.float32)
        self._ck(self.L.flb_map_fov_segment(self.h, C.byref(prm), _p(p), C.byref(nb), _p(boxes), _p(local), C.byref(nd)))
        self.M = self.L.flb_map_size(self.h)
        return boxes[:nb.value].copy(), local, nd.value

    def map_fov_reset(self):
        """flb_map_fov_reset: the next flb_map_fov_segment only places the cube (Localmap_Initialized = false)."""
        self._ck(self.L.flb_map_fov_reset(self.h))

    def map_download(self):
        n = self.L.flb_map_size(self.h)
        out = np.empty((n, 3), np.float32)
        m = C.c_int()
        self._ck(self.L.flb_map_download(self.h, _p(out), n, C.byref(m)))
        return out

    def map_grid_info(self):
        """flb_map_grid_info: dict(cell_size, sparse, cells, index_bytes) of the map's kNN cell index."""
        cs, sp, nc, nb = C.c_double(), C.c_int(), C.c_int64(), C.c_int64()
        self._ck(self.L.flb_map_grid_info(self.h, C.byref(cs), C.byref(sp), C.byref(nc), C.byref(nb)))
        return dict(cell_size=cs.value, sparse=sp.value, cells=nc.value, index_bytes=nb.value)

    def voxel_grid(self, xyz, leaf):
        """flb_voxel_grid: pcl::VoxelGrid centroids (m, 3) float32."""
        a = np.ascontiguousarray(xyz, np.float32)
        out = np.zeros((len(a), 3), np.float32)
        n = C.c_int()
        self._ck(self.L.flb_voxel_grid(self.h, _p(a), len(a), a.shape[1] if a.ndim == 2 else 3, C.c_float(leaf), _p(out), len(a), C.byref(n)))
        return out[:n.value].copy()

    def scan_upload(self, body_xyz):
        a = np.ascontiguousarray(body_xyz, np.float32)
        self._ck(self.L.flb_scan_upload(self.h, _p(a), a.shape[0], a.shape[1] if a.ndim == 2 else 3))
        self.N = a.shape[0]

    def scan_from_undistorted(self, leaf):
        """flb_scan_from_undistorted: the scan = the voxel filter (leaf) of the last flb_imu_undistort output, on the
        device; returns feats_down_size."""
        n = C.c_int()
        self._ck(self.L.flb_scan_from_undistorted(self.h, C.c_float(leaf), C.byref(n)))
        self.N = n.value
        return n.value

    def map_upload_scan(self):
        """flb_map_upload_scan: the map = the current scan's points in the caller's order (the first frame's Build)."""
        self._ck(self.L.flb_map_upload_scan(self.h))
        self.M = self.L.flb_map_size(self.h)

    def debug_set_scan_sort(self, mode):
        """0 automatic, 1 one-block ordering kernel, 2 device-wide sort (test aid)."""
        self._ck(self.L.flb_debug_set_scan_sort(self.h, int(mode)))

    def debug_set_map_index(self, mode):
        """Cell index of the following map rebuilds: 0 automatic, 1 dense always, 2 sparse always (test aid)."""
        self._ck(self.L.flb_debug_set_map_index(self.h, int(mode)))

    def debug_scan_order(self):
        """Index in the caller's array of the point at each position of the uploaded (ordered) scan (test aid)."""
        out = np.zeros(max(self.N, 1), np.int32)
        self._ck(self.L.flb_debug_scan_order(self.h, _p(out), out.shape[0]))
        return out[:self.N]

    def image_upload(self, gray):
        a = np.ascontiguousarray(gray, np.uint8)
        self._ck(self.L.flb_image_upload(self.h, _p(a), a.shape[1], a.shape[0], a.shape[1]))

    def image_upload_bgr(self, bgr, gray_rule=GRAY_CV4):
        """flb_image_upload_bgr: a (height, width, 3) uint8 BGR frame at the camera's size or twice it.  A strided view
        (e.g. a column slice) is passed with its own row stride; its pixels must be contiguous within a row."""
        a = np.asarray(bgr)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.strides[1:] != (3, 1) or a.strides[0] < 0:
            a = np.ascontiguousarray(a, np.uint8)
        self._ck(self.L.flb_image_upload_bgr(self.h, _p(a), a.shape[1], a.shape[0], a.strides[0], int(gray_rule)))

    def image_upload_msg(self, img, encoding, gray_rule=GRAY_CV4):
        """flb_image_upload_msg: a camera message's pixels as a uint8 array, (height, width) for mono8 and Bayer or
        (height, width, bytes per pixel) for the others; encoding: a sensor_msgs::Image encoding string or FLB_ENC_*.
        A strided view (e.g. a column slice) is passed with its own row step; its pixels must be contiguous in a row."""
        enc = ENCODINGS[encoding] if isinstance(encoding, str) else int(encoding)
        bpp = ENC_BYTES.get(enc, 1)
        a = np.asarray(img)
        if a.ndim == 2:
            a = a[:, :, None]
        if a.dtype != np.uint8 or a.ndim != 3 or a.strides[1:] != (a.shape[2], 1) or a.strides[0] < 0:
            a = np.ascontiguousarray(a, np.uint8)
        if a.shape[2] != bpp:
            raise ValueError(f"image_upload_msg: encoding {encoding} has {bpp} bytes per pixel, the array {a.shape[2]}")
        self._ck(self.L.flb_image_upload_msg(self.h, _p(a), a.shape[1], a.shape[0], a.strides[0], enc, int(gray_rule)))

    def image_download(self, gray=True, bgr=True):
        """flb_image_download: (gray (H, W) uint8 or None, bgr (H, W, 3) uint8 or None) of the current image set."""
        w, hgt = C.c_int(), C.c_int()
        self._ck(self.L.flb_image_download(self.h, None, None, 0, C.byref(w), C.byref(hgt)))
        g = np.zeros((hgt.value, w.value), np.uint8) if gray else None
        c = np.zeros((hgt.value, w.value, 3), np.uint8) if bgr else None
        self._ck(self.L.flb_image_download(self.h, _p(g), _p(c), w.value * hgt.value, None, None))
        return g, c

    def patches_upload(self, pos, patch, level):
        pos = np.ascontiguousarray(pos, np.float64).reshape(-1, 3)
        patch = np.ascontiguousarray(patch, np.float32).reshape(len(pos), 192)
        level = np.ascontiguousarray(level, np.int32)
        self._ck(self.L.flb_patches_upload(self.h, _p(pos), _p(patch), _p(level), len(pos)))
        self.Pn = len(pos)

    def camera_set(self, cam: dict):
        c = Camera()
        c.width, c.height = cam["width"], cam["height"]
        c.fx, c.fy, c.cx, c.cy = cam["fx"], cam["fy"], cam["cx"], cam["cy"]
        c.d[:] = cam["d"]
        self._ck(self.L.flb_camera_set(self.h, C.byref(c)))
        self._cam_wh = (int(cam["width"]), int(cam["height"]))

    def load_frame(self, frame):
        """Upload everything a synthetic frame holds."""
        self.map_upload(frame["map_xyz"])
        self.scan_upload(frame["scan_body"])
        if len(frame["patch_pos"]):
            self.camera_set(frame["cam"])
            self.image_upload(frame["image"])
            self.patches_upload(frame["patch_pos"], frame["patch_ref"], frame["patch_level"])

    # ---- kNN
    def knn(self, q_world):
        q = np.ascontiguousarray(q_world, np.float32)
        idx = np.empty((len(q), 5), np.int32)
        d2 = np.empty((len(q), 5), np.float32)
        self._ck(self.L.flb_knn(self.h, _p(q), len(q), _p(idx), _p(d2)))
        return idx, d2

    # ---- LIO
    def lio_pass(self, prm: LioParams, R, p, rematch: bool, width=6, export=True):
        R = np.ascontiguousarray(R, np.float64)
        p = np.ascontiguousarray(p, np.float64)
        eq = NormalEq()
        self._ck(self.L.flb_lio_pass(self.h, C.byref(prm), _p(R), _p(p), int(rematch), width, C.byref(eq)))
        out = dict(n=eq.n_eff, total_residual=eq.sum_abs_res,
                   HTH=np.array(eq.HTH[:width * width]).reshape(width, width), HTh=np.array(eq.HTh[:width]))
        if export:
            N = self.N
            world = np.empty((N, 3), np.float32)
            nn_idx = np.empty((N, 5), np.int32)
            nn_d2 = np.empty((N, 5), np.float32)
            pabcd = np.empty((N, 4), np.float32)
            pd2 = np.empty(N, np.float32)
            sel = np.empty(N, np.uint8)
            rows = np.empty((N, width))
            meas = np.empty(N)
            sel_idx = np.empty(N, np.int32)
            n = C.c_int()
            self._ck(self.L.flb_lio_export(self.h, _p(world), _p(nn_idx), _p(nn_d2), _p(pabcd), _p(pd2), _p(sel), _p(rows),
                                           _p(meas), _p(sel_idx), C.byref(n)))
            out.update(world=world, nn_idx=nn_idx, nn_d2=nn_d2, pabcd=pabcd, pd2=pd2, rowmask=sel,
                       rows=rows[:n.value], meas=meas[:n.value], sel_idx=sel_idx[:n.value])
        return out

    def lio_update(self, prm: LioParams, x: State18, x_prop: State18) -> LioReport:
        rep = LioReport()
        self._ck(self.L.flb_lio_update(self.h, C.byref(prm), C.byref(x), C.byref(x_prop), C.byref(rep)))
        return rep

    def lio_update_ikfom(self, prm: IkfomParams, x: StateIkfom) -> IkfomReport:
        rep = IkfomReport()
        self._ck(self.L.flb_lio_update_ikfom(self.h, C.byref(prm), C.byref(x), C.byref(rep)))
        return rep

    # ---- VIO
    def vio_pass(self, prm: VioParams, R, p, level: int, export=True):
        R = np.ascontiguousarray(R, np.float64)
        p = np.ascontiguousarray(p, np.float64)
        eq = VioEq()
        self._ck(self.L.flb_vio_pass(self.h, C.byref(prm), _p(R), _p(p), level, C.byref(eq)))
        out = dict(error=np.float32(eq.error), n_meas=eq.n_meas, skipped=eq.skipped,
                   HTH6=np.array(eq.HTH[:]).reshape(6, 6), HTz6=np.array(eq.HTz[:]))
        if export:
            z = np.empty(self.Pn * 64)
            H = np.empty((self.Pn * 64, 6))
            err = np.empty(self.Pn, np.float32)
            self._ck(self.L.flb_vio_export(self.h, _p(z), _p(H), _p(err)))
            out.update(z=z, H_sub=H, errors=err)
        return out

    def vio_update_level(self, prm: VioParams, level: int, total_residual: float, x: State18, x_prop: State18):
        """flb_vio_update_level == LidarSelector::UpdateState.  Returns (last_error, G[18, 6], report)."""
        rep = VioReport()
        le = C.c_float()
        G = np.zeros((18, 6))
        self._ck(self.L.flb_vio_update_level(self.h, C.byref(prm), int(level), C.c_float(total_residual), C.byref(x), C.byref(x_prop),
                                             C.byref(le), _p(G), C.byref(rep)))
        return le.value, G, rep

    def vio_errors(self):
        """sub_sparse_map->errors as the last update's last pass left them (flb_vio_errors)."""
        err = np.zeros(self.Pn, np.float32)
        self._ck(self.L.flb_vio_errors(self.h, _p(err), self.Pn))
        return err

    def vio_update(self, prm: VioParams, x: State18, x_prop: State18) -> VioReport:
        rep = VioReport()
        self._ck(self.L.flb_vio_update(self.h, C.byref(prm), C.byref(x), C.byref(x_prop), C.byref(rep)))
        return rep

    # ---- visual-map growth: candidate scoring (row f4)
    def visual_candidates(self, Rcw, Pcw, world_xyz, grid_size, border, map_value):
        """flb_visual_candidates on the uploaded image / camera.  Returns (map_value_out, winner) per grid cell."""
        R = np.ascontiguousarray(Rcw, np.float64)
        P = np.ascontiguousarray(Pcw, np.float64)
        pts = np.ascontiguousarray(world_xyz, np.float32)
        mv = np.ascontiguousarray(map_value, np.float32).copy()
        win = np.zeros(len(mv), np.int32)
        self._ck(self.L.flb_visual_candidates(self.h, R.ctypes.data_as(C.c_void_p), P.ctypes.data_as(C.c_void_p),
                                              pts.ctypes.data_as(C.c_void_p), len(pts), pts.shape[1] if len(pts) else 3,
                                              int(grid_size), int(border), mv.ctypes.data_as(C.c_void_p),
                                              win.ctypes.data_as(C.c_void_p)))
        return mv, win

    # ---- batched frames
    def batch_begin(self, B, max_points):
        self._ck(self.L.flb_batch_begin(self.h, int(B), int(max_points)))

    def batch_set_frame(self, b, body_xyz, x: State18, x_prop: State18):
        a = np.ascontiguousarray(body_xyz, np.float32)
        self._ck(self.L.flb_batch_set_frame(self.h, int(b), _p(a), a.shape[0], a.shape[1], C.byref(x), C.byref(x_prop)))

    def batch_state_reset_enqueue(self):
        self._ck(self.L.flb_batch_state_reset_enqueue(self.h))

    def batch_update_enqueue(self, lprm, vprm=None):
        self._ck(self.L.flb_batch_update_enqueue(self.h, C.byref(lprm), C.byref(vprm) if vprm is not None else None))

    def batch_state_download(self, b):
        x, lr, vr = State18(), LioReport(), VioReport()
        self._ck(self.L.flb_batch_state_download(self.h, int(b), C.byref(x), C.byref(lr), C.byref(vr)))
        return x, lr, vr

    # ---- device-resident visual map (rows f2 / f4)
    def vmap_reset(self, seq_or_frame, grid_size=40, outlier_threshold=100.0, ncc_en=0, ncc_thre=0.0):
        """flb_vmap_reset; the extrinsics come from a synthetic frame / sequence dict (Rcl, Pcl, R_LI, t_LI)."""
        p = VmapParams()
        p.grid_size, p.ncc_en, p.outlier_threshold, p.ncc_thre = int(grid_size), int(ncc_en), float(outlier_threshold), float(ncc_thre)
        p.Rcl[:] = np.asarray(seq_or_frame["Rcl"], np.float64).ravel()
        p.Pcl[:] = np.asarray(seq_or_frame["Pcl"], np.float64)
        p.R_LI[:] = np.asarray(seq_or_frame["R_LI"], np.float64).ravel()
        p.t_LI[:] = np.asarray(seq_or_frame["t_LI"], np.float64)
        self._ck(self.L.flb_vmap_reset(self.h, C.byref(p)))

    @staticmethod
    def _pose(Rcw, Pcw):
        if Rcw is None:
            return None, None, None, None
        R = np.ascontiguousarray(Rcw, np.float64)
        P = np.ascontiguousarray(Pcw, np.float64)
        return R, P, R.ctypes.data_as(C.c_void_p), P.ctypes.data_as(C.c_void_p)

    def vmap_select(self, Rcw, Pcw, pg_down, blocking=True):
        """flb_vmap_select.  blocking: returns the number of selected patches; else enqueue-only (returns None)."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        pg = np.ascontiguousarray(pg_down, np.float32).reshape(-1, 3)
        n = C.c_int()
        self._ck(self.L.flb_vmap_select(self.h, pr, pp, _p(pg), len(pg), 3, C.byref(n) if blocking else None))
        if blocking:
            self.Pn = n.value
            return n.value
        return None

    def vmap_selected(self):
        n = C.c_int()
        self._ck(self.L.flb_vmap_selected(self.h, 0, C.byref(n), None, None, None, None, None, None))
        m = n.value
        o = dict(index=np.zeros(m, np.int32), point=np.zeros(m, np.int32), search_level=np.zeros(m, np.int32),
                 error=np.zeros(m, np.float32), pos=np.zeros((m, 3)), patch=np.zeros((m, 192), np.float32))
        if m:
            self._ck(self.L.flb_vmap_selected(self.h, m, C.byref(n), _p(o["index"]), _p(o["point"]), _p(o["search_level"]), _p(o["error"]),
                                              _p(o["pos"]), _p(o["patch"])))
        self.Pn = m
        return o

    def vmap_grow(self, Rcw, Pcw, pg, frame_id):
        R, P, pr, pp = self._pose(Rcw, Pcw)
        pg = np.ascontiguousarray(pg, np.float32).reshape(-1, 3)
        self._ck(self.L.flb_vmap_grow(self.h, pr, pp, _p(pg), len(pg), 3, int(frame_id)))

    def vmap_add_observations(self, Rcw, Pcw, frame_id):
        R, P, pr, pp = self._pose(Rcw, Pcw)
        self._ck(self.L.flb_vmap_add_observations(self.h, pr, pp, int(frame_id)))

    def colorize(self, Rcw, Pcw, bgr=None, world_xyz=None):
        """flb_colorize: (rgb (n, 3) uint8, valid (n,) bool).  bgr None: the current image set's colour frame."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        img = None if bgr is None else np.ascontiguousarray(bgr, np.uint8)
        pts = np.ascontiguousarray(world_xyz, np.float32).reshape(-1, 3)
        rgb = np.zeros((len(pts), 3), np.uint8)
        val = np.zeros(len(pts), np.uint8)
        self._ck(self.L.flb_colorize(self.h, pr, pp, _p(img), 0 if img is None else img.shape[1] * 3, _p(pts), len(pts), 3, _p(rgb),
                                     _p(val)))
        return rgb, val.astype(bool)

    # ---- the frame's world cloud (pcl_wait_pub) on the device
    def world_cloud(self, prm, source=CLOUD_UNDISTORTED, R=None, p=None):
        """flb_world_cloud: the source cloud (CLOUD_SCAN / CLOUD_UNDISTORTED) at pose (R, p), or at the device state x
        when both are None; returns its number of points."""
        R = None if R is None else np.ascontiguousarray(R, np.float64)
        p = None if p is None else np.ascontiguousarray(p, np.float64)
        n = C.c_int()
        self._wc_n = 0
        self._ck(self.L.flb_world_cloud(self.h, C.byref(prm) if prm is not None else None, _p(R), _p(p), int(source), C.byref(n)))
        self._wc_n = n.value
        return n.value

    def world_cloud_download(self):
        """flb_world_cloud_download: the world cloud (n, 3) float32."""
        out = np.zeros((self._wc_n, 3), np.float32)
        n = C.c_int()
        self._ck(self.L.flb_world_cloud_download(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def world_cloud_points(self, download=True):
        """flb_world_cloud_points: publish_frame_world's pcl_wait_pub, (n,) XYZINORMAL_POINT records (appended to an open
        LiDAR save).  download=False: points48 = NULL (only the save append); returns the point count."""
        n = C.c_int()
        if not download:
            self._ck(self.L.flb_world_cloud_points(self.h, None, 0, C.byref(n)))
            return n.value
        out = np.zeros(self._wc_n, XYZINORMAL_POINT)
        self._ck(self.L.flb_world_cloud_points(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def lidar_save_begin(self, max_points):
        self._ck(self.L.flb_lidar_save_begin(self.h, int(max_points)))

    def lidar_save_size(self):
        """flb_lidar_save_size: dict(n, dropped, device_bytes)."""
        n, d, b = C.c_int64(), C.c_int64(), C.c_int64()
        self._ck(self.L.flb_lidar_save_size(self.h, C.byref(n), C.byref(d), C.byref(b)))
        return dict(n=n.value, dropped=d.value, device_bytes=b.value)

    def lidar_save_download(self, first=0, count=None):
        """flb_lidar_save_download: records first .. first + count - 1 of the save (count None: to its end),
        XYZINORMAL_POINT."""
        if count is None:
            count = self.lidar_save_size()["n"] - first
        out = np.zeros(max(int(count), 0), XYZINORMAL_POINT)
        self._ck(self.L.flb_lidar_save_download(self.h, int(first), int(count), _p(out)))
        return out

    def lidar_save_end(self):
        self._ck(self.L.flb_lidar_save_end(self.h))

    # ---- the last LIO pass's effective points (publish_effect_world) on the device
    def effect_cloud(self, prm, R=None, p=None):
        """flb_effect_cloud: laserCloudOri of the last LIO pass at pose (R, p), or at the device state x when both are
        None; returns its number of points."""
        R = None if R is None else np.ascontiguousarray(R, np.float64)
        p = None if p is None else np.ascontiguousarray(p, np.float64)
        n = C.c_int()
        self._ef_n = 0
        self._ck(self.L.flb_effect_cloud(self.h, C.byref(prm) if prm is not None else None, _p(R), _p(p), C.byref(n)))
        self._ef_n = n.value
        return n.value

    def effect_cloud_download(self):
        """flb_effect_cloud_download: the effect cloud (n, 3) float32."""
        out = np.zeros((self._ef_n, 3), np.float32)
        n = C.c_int()
        self._ck(self.L.flb_effect_cloud_download(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def effect_cloud_download_points(self):
        """flb_effect_cloud_download_points: the effect cloud with its intensities, (n,) XYZINORMAL_POINT records."""
        out = np.zeros(self._ef_n, XYZINORMAL_POINT)
        n = C.c_int()
        self._ck(self.L.flb_effect_cloud_download_points(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def vmap_select_cloud(self, Rcw, Pcw, leaf=0.2, blocking=True):
        """flb_vmap_select_cloud: vmap_select of downSizeFilter(world cloud, leaf), all on the device."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        n = C.c_int()
        self._ck(self.L.flb_vmap_select_cloud(self.h, pr, pp, C.c_float(leaf), C.byref(n) if blocking else None))
        if blocking:
            self.Pn = n.value
            return n.value
        return None

    def vmap_grow_cloud(self, Rcw, Pcw, frame_id):
        R, P, pr, pp = self._pose(Rcw, Pcw)
        self._ck(self.L.flb_vmap_grow_cloud(self.h, pr, pp, int(frame_id)))

    def colorize_cloud(self, Rcw, Pcw, bgr=None):
        """flb_colorize_cloud: (rgb (n, 3) uint8, valid (n,) bool) of the world cloud.  bgr None: the current image
        set's colour frame."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        img = None if bgr is None else np.ascontiguousarray(bgr, np.uint8)
        rgb = np.zeros((self._wc_n, 3), np.uint8)
        val = np.zeros(self._wc_n, np.uint8)
        self._ck(self.L.flb_colorize_cloud(self.h, pr, pp, _p(img), 0 if img is None else img.shape[1] * 3, _p(rgb), _p(val)))
        return rgb, val.astype(bool)

    # ---- publish_frame_world_rgb's laserCloudWorldRGB and the run's pcl_wait_save on the device
    def rgb_cloud(self, Rcw=None, Pcw=None, bgr=None):
        """flb_rgb_cloud: the coloured points of the world cloud as records; returns their number.  bgr None: the
        current image set's colour frame; Rcw / Pcw None: the pose from the device state."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        img = None if bgr is None else np.ascontiguousarray(bgr, np.uint8)
        n = C.c_int()
        self._rc_n = 0
        self._ck(self.L.flb_rgb_cloud(self.h, pr, pp, _p(img), 0 if img is None else img.shape[1] * 3, C.byref(n)))
        self._rc_n = n.value
        return n.value

    def rgb_cloud_download(self):
        """flb_rgb_cloud_download: the coloured cloud, (n,) RGB_POINT records."""
        out = np.zeros(self._rc_n, RGB_POINT)
        n = C.c_int()
        self._ck(self.L.flb_rgb_cloud_download(self.h, _p(out), len(out), C.byref(n)))
        return out[:n.value]

    def rgb_save_begin(self, max_points):
        self._ck(self.L.flb_rgb_save_begin(self.h, int(max_points)))

    def rgb_save_size(self):
        """flb_rgb_save_size: dict(n, dropped, device_bytes)."""
        n, d, b = C.c_int64(), C.c_int64(), C.c_int64()
        self._ck(self.L.flb_rgb_save_size(self.h, C.byref(n), C.byref(d), C.byref(b)))
        return dict(n=n.value, dropped=d.value, device_bytes=b.value)

    def rgb_save_download(self, first=0, count=None):
        """flb_rgb_save_download: records first .. first + count - 1 of the save (count None: to its end), RGB_POINT."""
        if count is None:
            count = self.rgb_save_size()["n"] - first
        out = np.zeros(max(int(count), 0), RGB_POINT)
        self._ck(self.L.flb_rgb_save_download(self.h, int(first), int(count), _p(out)))
        return out

    def rgb_save_end(self):
        self._ck(self.L.flb_rgb_save_end(self.h))

    def keypatch_image(self, Rcw=None, Pcw=None, out=None):
        """flb_keypatch_image: (frame (H, W, 3) uint8, patch count) -- the current colour frame with display_keypatch's
        circles.  Rcw / Pcw None: the pose from the device state.  out: a (H, W, 3) uint8 array to write into (rows may
        be strided); a page-locked one (pinned_like) makes the call enqueue-only, its bytes valid after synchronize()."""
        R, P, pr, pp = self._pose(Rcw, Pcw)
        if out is None:
            W, H = getattr(self, "_cam_wh", (0, 0))
            out = np.zeros((H, W, 3), np.uint8)
        if out.dtype != np.uint8 or out.ndim != 3 or out.strides[1:] != (3, 1):
            raise ValueError("keypatch_image: out must be (H, W, 3) uint8 with packed pixels")
        n = C.c_int(-1)
        self._ck(self.L.flb_keypatch_image(self.h, pr, pp, _p(out), out.strides[0], C.byref(n)))
        return out, n.value

    def vmap_counts(self):
        v = [C.c_int() for _ in range(5)]
        self._ck(self.L.flb_vmap_counts(self.h, *[C.byref(x) for x in v]))
        return dict(points=v[0].value, features=v[1].value, images=v[2].value, selected=v[3].value, last_added=v[4].value)

    def vmap_map_value(self, length):
        out = np.zeros(length, np.float32)
        self._ck(self.L.flb_vmap_map_value(self.h, _p(out), length))
        return out

    def vmap_dump(self):
        c = self.vmap_counts()
        n, m = c["points"], c["features"]
        d = dict(pos=np.zeros((n, 3)), value=np.zeros(n, np.float32), n_obs=np.zeros(n, np.int32), obs=np.zeros((n, 20), np.int32),
                 ft_geo=np.zeros((m, 17)), ft_score=np.zeros(m, np.float32), ft_level_id_img=np.zeros((m, 3), np.int32))
        self._ck(self.L.flb_vmap_dump(self.h, n, m, _p(d["pos"]), _p(d["value"]), _p(d["n_obs"]), _p(d["obs"]), _p(d["ft_geo"]),
                                      _p(d["ft_score"]), _p(d["ft_level_id_img"])))
        return d

    def vmap_reclaim(self):
        """flb_vmap_reclaim (enqueue-only): drop evicted features, put unreferenced keyframe slots on the free-slot stack."""
        self._ck(self.L.flb_vmap_reclaim(self.h))

    def vmap_usage(self):
        """flb_vmap_usage (blocking): the visual map's sizes, capacities and device bytes."""
        v = [C.c_int() for _ in range(7)]
        b = C.c_int64()
        self._ck(self.L.flb_vmap_usage(self.h, *[C.byref(x) for x in v], C.byref(b)))
        keys = ("points", "features", "dead_features", "feature_capacity", "slots_in_use", "free_slots", "pool_slots")
        return dict(zip(keys, (x.value for x in v)), device_bytes=b.value)

    def vmap_keyframe(self, slot):
        """flb_vmap_keyframe: the keyframe image in pool slot `slot` (height, width) uint8."""
        w, hgt = self._cam_wh
        out = np.zeros((hgt, w), np.uint8)
        self._ck(self.L.flb_vmap_keyframe(self.h, int(slot), _p(out), out.size))
        return out

    # ---- IMU propagation + undistortion (row f3)
    def imu_undistort(self, prm: ImuParams, carry: ImuCarry, v_imu, pcl_beg_time, pcl_end_time, pts, offset_index=3, download=True):
        """flb_imu_undistort on the device state.  v_imu (K,7) [t, gyr, acc]; pts (n, stride) float32 with x,y,z
        first and the time offset (ms) at column offset_index.  Returns (xyz (n,3) float32, IMUpose (n_poses,22));
        carry is updated in place, the device state is propagated in place.  download=False: out_xyz = NULL (the points
        stay on the device for scan_from_undistorted / world_cloud) and xyz is None."""
        v = np.ascontiguousarray(v_imu, np.float64)
        pts = np.ascontiguousarray(pts, np.float32)
        n = pts.shape[0]
        out = np.zeros((n, 3), np.float32) if download else None
        poses = np.zeros((len(v), 22), np.float64)
        npo = C.c_int()
        self._ck(self.L.flb_imu_undistort(self.h, C.byref(prm), C.byref(carry), v.ctypes.data_as(C.c_void_p), len(v),
                                          float(pcl_beg_time), float(pcl_end_time), pts.ctypes.data_as(C.c_void_p),
                                          pts.shape[1] if n else 4, offset_index, n, _p(out),
                                          poses.ctypes.data_as(C.c_void_p), C.byref(npo)))
        return out, poses[:npo.value]

    # ---- the driver's LiDAR message (Preprocess::process, the time sort, UndistortPcl's window)
    def _lidar_upload(self, fn, fmt, records, n_records, *dis_b, yaw=False):
        """The four LiDAR uploads' shared binding: records = a uint8 array (or bytes) of n_records records of
        fmt.point_step bytes (default: all of them).  Returns (n_points, last_offset_ms), and yaw_times as a bool when
        `yaw`."""
        a = np.frombuffer(records, np.uint8) if isinstance(records, (bytes, bytearray)) else records
        if n_records is None:
            n_records = a.size // max(fmt.point_step, 1)
        n, last, yaw_times = C.c_int(), C.c_float(), C.c_int()
        outs = (C.byref(n), C.byref(last)) + ((C.byref(yaw_times),) if yaw else ())
        self._ck(fn(self.h, C.byref(fmt), *dis_b, _p(a) if a.size else None, int(n_records), *outs))
        self._lid_n = n.value
        return (n.value, np.float32(last.value)) + ((bool(yaw_times.value),) if yaw else ())

    def lidar_upload(self, fmt: LidarFormat, records, n_records=None):
        """flb_lidar_upload: records = a uint8 array (or bytes) of n_records records of fmt.point_step bytes.  Returns
        (pl_surf.size(), points.back().curvature after the sort)."""
        return self._lidar_upload(self.L.flb_lidar_upload, fmt, records, n_records)

    def lidar_upload_velodyne(self, fmt: VelodyneFormat, records, n_records=None):
        """flb_lidar_upload_velodyne: records = a uint8 array (or bytes) of n_records Velodyne records of fmt.point_step
        bytes.  Returns (pl_surf.size(), points.back().curvature after the sort, whether the times came from the yaw)."""
        return self._lidar_upload(self.L.flb_lidar_upload_velodyne, fmt, records, n_records, yaw=True)

    def lidar_upload_features(self, fmt: LidarFormat, records, dis_b=0.0, n_records=None):
        """flb_lidar_upload_features (feature_extract_enable: 1) for a Livox or Ouster message; fmt.off_line is the Livox
        line or the Ouster's u8 ring.  Returns (pl_surf.size(), points.back().curvature after the sort)."""
        return self._lidar_upload(self.L.flb_lidar_upload_features, fmt, records, n_records, float(dis_b))

    def lidar_upload_velodyne_features(self, fmt: VelodyneFormat, records, dis_b=0.0, n_records=None):
        """flb_lidar_upload_velodyne_features (feature_extract_enable: 1).  Returns (pl_surf.size(),
        points.back().curvature after the sort, whether the times came from the yaw)."""
        return self._lidar_upload(self.L.flb_lidar_upload_velodyne_features, fmt, records, n_records, float(dis_b), yaw=True)

    def lidar_upload_intensity(self, fmt: LidarFormat, records, off_intensity, n_records=None):
        """flb_lidar_upload_intensity: lidar_upload keeping each point's intensity; off_intensity = the field's byte offset
        (Livox reflectivity u8, others float32), or -1 (every point 0)."""
        return self._lidar_upload(self.L.flb_lidar_upload_intensity, fmt, records, n_records, int(off_intensity))

    def lidar_upload_velodyne_intensity(self, fmt: VelodyneFormat, records, off_intensity, n_records=None):
        """flb_lidar_upload_velodyne_intensity: lidar_upload_velodyne keeping each point's float32 intensity (any offset;
        -1: every point 0)."""
        return self._lidar_upload(self.L.flb_lidar_upload_velodyne_intensity, fmt, records, n_records, int(off_intensity), yaw=True)

    def lidar_download_points(self):
        """flb_lidar_download_points: the current cloud as pl_surf holds it, (n,) XYZINORMAL_POINT records."""
        n = C.c_int()
        self._ck(self.L.flb_lidar_download_points(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, XYZINORMAL_POINT)
        self._ck(self.L.flb_lidar_download_points(self.h, _p(out), n.value, None))
        return out

    def lidar_download(self):
        """flb_lidar_download: the decoded, time-sorted cloud, (n, 4) float32 x, y, z, curvature."""
        n = C.c_int()
        self._ck(self.L.flb_lidar_download(self.h, None, 0, C.byref(n)))
        out = np.zeros((n.value, 4), np.float32)
        self._ck(self.L.flb_lidar_download(self.h, _p(out), n.value, None))
        return out

    def imu_undistort_lidar(self, prm: ImuParams, carry: ImuCarry, v_imu, pcl_beg_time, pcl_end_time, pcl_offset_time,
                            is_lidar_end, download=True):
        """flb_imu_undistort_lidar: imu_undistort on the window of the device cloud.  Returns (n_taken, xyz (n_taken, 3)
        float32 or None, IMUpose)."""
        v = np.ascontiguousarray(v_imu, np.float64)
        cap = max(getattr(self, "_lid_n", 0), 1)
        out = np.zeros((cap, 3), np.float32) if download else None
        poses = np.zeros((len(v), 22), np.float64)
        npo, taken = C.c_int(), C.c_int()
        self._ck(self.L.flb_imu_undistort_lidar(self.h, C.byref(prm), C.byref(carry), v.ctypes.data_as(C.c_void_p), len(v),
                                                float(pcl_beg_time), float(pcl_end_time), float(pcl_offset_time),
                                                int(bool(is_lidar_end)), C.byref(taken), _p(out), cap,
                                                poses.ctypes.data_as(C.c_void_p), C.byref(npo)))
        return taken.value, (out[:taken.value] if download else None), poses[:npo.value]

    # ---- device-resident loop
    def state_upload(self, x: State18, x_prop: State18):
        self._ck(self.L.flb_state_upload(self.h, C.byref(x), C.byref(x_prop)))

    def state_download(self):
        x, lr, vr = State18(), LioReport(), VioReport()
        self._ck(self.L.flb_state_download(self.h, C.byref(x), C.byref(lr), C.byref(vr)))
        return x, lr, vr

    def frame_inputs(self, scan, x, x_prop, image=None, pos=None, patch=None, level=None):
        """A reusable flb_frame_inputs over caller-owned numpy arrays (keep them alive; pass page-locked arrays from
        pinned_like() to let the copy engine read them in place)."""
        fi = FrameInputs()
        fi._keep = (scan, image, pos, patch, level, x, x_prop)
        fi.scan_xyz, fi.n_scan, fi.scan_stride = scan.ctypes.data, scan.shape[0], scan.shape[1]
        if image is not None:
            fi.gray, fi.width, fi.height, fi.stride_bytes = image.ctypes.data, image.shape[1], image.shape[0], image.shape[1]
        if pos is not None:
            fi.patch_pos, fi.patch, fi.search_level, fi.Pn = pos.ctypes.data, patch.ctypes.data, level.ctypes.data, len(pos)
            self.Pn = len(pos)
        fi.x, fi.x_prop = C.pointer(x), C.pointer(x_prop)
        self.N = scan.shape[0]
        return fi

    def frame_enqueue(self, fi, lprm, vprm=None, slot=-1):
        self._ck(self.L.flb_frame_enqueue(self.h, C.byref(fi), C.byref(lprm), C.byref(vprm) if vprm is not None else None, int(slot)))

    def state_download_enqueue(self, slot):
        self._ck(self.L.flb_state_download_enqueue(self.h, int(slot)))

    def state_download_wait(self, slot):
        x, lr, vr = State18(), LioReport(), VioReport()
        self._ck(self.L.flb_state_download_wait(self.h, int(slot), C.byref(x), C.byref(lr), C.byref(vr)))
        return x, lr, vr

    def lio_update_enqueue(self, prm):
        self._ck(self.L.flb_lio_update_enqueue(self.h, C.byref(prm)))

    def vio_update_enqueue(self, prm):
        self._ck(self.L.flb_vio_update_enqueue(self.h, C.byref(prm)))

    def state_reset_enqueue(self):
        self._ck(self.L.flb_state_reset_enqueue(self.h))

    def state_set_prior_enqueue(self):
        self._ck(self.L.flb_state_set_prior_enqueue(self.h))

    def pinned_like(self, a):
        """A page-locked copy of numpy array `a` (flb_host_alloc); freed with the handle."""
        a = np.ascontiguousarray(a)
        ptr = C.c_void_p()
        self._ck(self.L.flb_host_alloc(self.h, max(a.nbytes, 1), C.byref(ptr)))
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append(ptr)
        buf = (C.c_ubyte * max(a.nbytes, 1)).from_address(ptr.value)
        out = np.frombuffer(buf, dtype=a.dtype, count=a.size).reshape(a.shape)
        out[...] = a
        return out

    def set_stream(self, stream_ptr):
        self._ck(self.L.flb_set_stream(self.h, C.c_void_p(stream_ptr)))

    def synchronize(self):
        self._ck(self.L.flb_synchronize(self.h))

    def launch_count(self) -> int:
        return int(self.L.flb_launch_count(self.h))

    def profile_start(self):
        self._ck(self.L.flb_profile_start(self.h))

    def profile_stop(self):
        ms = np.zeros(4)
        n = np.zeros(4, np.int64)
        self._ck(self.L.flb_profile_stop(self.h, _p(ms), _p(n)))
        return ms, n

    def trace_enable(self, on=True):
        self._ck(self.L.flb_trace_enable(self.h, int(on)))

    def trace_download(self, which):
        us = np.zeros(128)
        n = C.c_int()
        self._ck(self.L.flb_trace_download(self.h, which, _p(us), 128, C.byref(n)))
        return us[:n.value]

    # ---- multi-GPU
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        rc = lib().flb_comm_unique_id(buf)
        if rc != FLB_OK:
            raise FlbError(rc, lib().flb_last_error(None).decode())
        return buf.raw

    def p2p_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self.L.flb_p2p_export(self.h, buf))
        return buf.raw

    def p2p_attach(self, rank: int, world: int, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        buf = C.create_string_buffer(blob, len(blob))
        self._ck(self.L.flb_p2p_attach(self.h, rank, world, buf))

    def p2p_detach(self):
        self._ck(self.L.flb_p2p_detach(self.h))

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        buf = C.create_string_buffer(unique_id, 128)
        self._ck(self.L.flb_comm_init(self.h, buf, rank, world))
