// fastlivo_b200_adapters.hpp -- header-only C++ adapters from the reference's Eigen / PCL /
// OpenCV-typed call sites onto the C ABI (include/fastlivo_b200.h).
//
// The adapters are templates over the reference's own types so that this header needs NO
// Eigen / PCL / OpenCV include of its own: it compiles inside the reference tree against the
// real types (see INTEGRATION.md) and inside tests/adapters against small mock types.
//
//   flb::lio_update(h, prm, state, state_propagat)      replaces the loop body
//        src/laserMapping.cpp:1504-1733          (live 18-DoF path, StatesGroup)
//   flb::h_share_model(h, prm, s, ekfom_data, ...)      same contract as
//        void h_share_model(state_ikfom&, esekfom::dyn_share_datastruct<double>&)
//        src/laserMapping.cpp:960-1094           (IKFoM-typed callback; rows from the GPU)
//   flb::compute_j(h, prm, img, sub_sparse_map, state, state_propagat)   replaces
//        LidarSelector::ComputeJ(cv::Mat)  src/lidar_selection.cpp:967-983
//   flb::undistort_pcl(h, prm, carry, v_imu, pcl_beg_time, pcl_end_time, state_inout, pcl_out)   replaces
//        ImuProcess::UndistortPcl from src/IMU_Processing.cpp:655 on (propagation + undistortion)
//   flb::undistort_pcl_on_device(h, prm, carry, v_imu, pcl_beg_time, pcl_end_time, state_inout, pcl_in) +
//   flb::downsample_scan(h, filter_size_surf_min)   replace UndistortPcl + downSizeFilterSurf (src/laserMapping.cpp:
//        1398-1399) + upload_scan: feats_undistort stays on the device and becomes the scan there
//   flb::map_incremental(h, lio_prm, filter_size_map_min)  /  flb::map_incremental(h, lio_prm, R, p, filter_size_map_min)   replace
//        map_incremental()  src/laserMapping.cpp:692-706  (the uploaded scan into the map, no host transform)
//   flb::publish_effect_world(h, lio_prm, cloud)  /  flb::publish_effect_world(h, lio_prm, R, p, cloud)   fill the cloud of
//        publish_effect_world()  src/laserMapping.cpp:871-885  (the last LIO pass's laserCloudOri, transformed on the device)
//   flb::publish_frame_world(h, cloud)   fill pcl_wait_pub of publish_frame_world() src/laserMapping.cpp:780-813 (img_enable:
//        0; the world cloud with its intensities, one copy);  flb::save_intensity_map(h, cloud)   pcl_wait_save_lidar
//   flb::publish_frame_world_rgb(h, cloud)  /  (h, Rcw, Pcw, cloud)   fill laserCloudWorldRGB of publish_frame_world_rgb()
//        src/laserMapping.cpp:710-777 (the world cloud coloured on the device, one copy);  flb::save_rgb_map(h, cloud)
//        fills pcl_wait_save from the device's save for the PCD written at exit (:1839-1846)
//   flb::lasermap_fov_segment(h, cube_len, &kdtree_delete_counter)  /  (h, cube_len, pos_lid, &kdtree_delete_counter)
//        replace lasermap_fov_segment()  src/laserMapping.cpp:363-421  (local-map cube + box delete on the device)
//   flb::upload_camera_frame(h, bgr, gray_rule)   replaces the resize / img_rgb / cvtColor lines of
//        LidarSelector::detect  src/lidar_selection.cpp:1029-1037  (one BGR upload; the gray image is made on the device)
//   flb::upload_camera_msg(h, msg, gray_rule)   the same from the sensor_msgs::Image itself, replacing getImageFromMsg
//        (src/laserMapping.cpp:490-493): mono8, rgb8, bgra8, rgba8 and Bayer frames are converted on the device
//   flb::display_keypatch(h, img_cp, time)   replaces LidarSelector::display_keypatch (src/lidar_selection.cpp:985-1005):
//        the circles are drawn on the device into img_cp, only the "N HZ" text on the host
//   flb::preprocess(h, livox_msg, n_scans, blind, point_filter_num)  /  flb::preprocess(h, pc2_msg, kind, n_scans, blind,
//        point_filter_num)   replace p_pre->process (src/preprocess.cpp:43-70) and the sort of sync_packages
//        (src/laserMapping.cpp:551): the driver's records go up as they are; the cloud is decoded and sorted on the device
//   flb::preprocess_velodyne(h, pc2_msg, n_scans, blind, point_filter_num)   the same for a Velodyne in any field layout,
//        with the times derived from the yaw angle on the device when the cloud has none (src/preprocess.cpp:376-428)
//   flb::preprocess_features(h, livox_msg, n_scans, blind, point_filter_num)  /  flb::preprocess_features(h, pc2_msg,
//        FLB_LIDAR_OUSTER or FLB_LIDAR_VELODYNE, n_scans, blind, point_filter_num)   the same with feature_extract_enable = 1:
//        the handlers' feature branches and give_feature (src/preprocess.cpp:94-135, :174-227, :299-373, :466-936)
//   flb::undistort_pcl_from_lidar(h, prm, carry, v_imu, lidar_meas, state_inout)   replaces UndistortPcl from :621 on
//        with that device cloud as lidar_meas.lidar (the window, the LidarMeasureGroup bookkeeping, the propagation)
//
// Type requirements (all met by the reference's types):
//   Mat3  : operator()(i,j) read/write (Eigen::Matrix3d)          Vec3 : operator()(i) / [i]
//   Cov   : operator()(i,j), 18x18 (Eigen::Matrix<double,18,18>)
//   StatesGroup : .rot_end .pos_end .vel_end .bias_g .bias_a .gravity .cov  (include/common_lib.h:296-381)
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/fastlivo_b200.h"

namespace flb {

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
inline void check(flb_handle* h, int rc) {
    if (rc != FLB_OK) throw Error(rc, flb_last_error(h));
}

// ---- StatesGroup <-> flb_state18 (Eigen is column-major; the ABI is row-major) ------------
template <class StatesGroup>
inline void to_abi(const StatesGroup& s, flb_state18& o) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) o.rot[3 * i + j] = s.rot_end(i, j);
        o.pos[i] = s.pos_end(i);
        o.vel[i] = s.vel_end(i);
        o.bg[i] = s.bias_g(i);
        o.ba[i] = s.bias_a(i);
        o.grav[i] = s.gravity(i);
    }
    for (int i = 0; i < 18; ++i)
        for (int j = 0; j < 18; ++j) o.cov[18 * i + j] = s.cov(i, j);
}
template <class StatesGroup>
inline void from_abi(const flb_state18& o, StatesGroup& s) {
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) s.rot_end(i, j) = o.rot[3 * i + j];
        s.pos_end(i) = o.pos[i];
        s.vel_end(i) = o.vel[i];
        s.bias_g(i) = o.bg[i];
        s.bias_a(i) = o.ba[i];
        s.gravity(i) = o.grav[i];
    }
    for (int i = 0; i < 18; ++i)
        for (int j = 0; j < 18; ++j) s.cov(i, j) = o.cov[18 * i + j];
}

template <class Mat3, class Vec3>
inline flb_lio_params make_lio_params(const Mat3& Lidar_rot_to_IMU, const Vec3& Lidar_offset_to_IMU, double laser_point_cov,
                                      int max_iteration) {
    flb_lio_params p{};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) p.R_LI[3 * i + j] = Lidar_rot_to_IMU(i, j);
        p.t_LI[i] = Lidar_offset_to_IMU(i);
    }
    p.laser_point_cov = laser_point_cov;
    p.max_iteration = max_iteration;
    p.conv_rot_deg = 0.01;    // src/laserMapping.cpp:1688
    p.conv_pos_cm = 0.015;
    return p;
}

// ---- scan / map upload from PCL clouds ---------------------------------------------------
// PointCloud: .points (vector of pcl::PointXYZINormal, 48 bytes, x,y,z first) -- stride 12 floats.
template <class PointCloud>
inline void upload_scan(flb_handle* h, const PointCloud& feats_down_body) {
    static_assert(sizeof(feats_down_body.points[0]) % sizeof(float) == 0, "point type must be float-packed");
    const int stride = (int)(sizeof(feats_down_body.points[0]) / sizeof(float));
    check(h, flb_scan_upload(h, feats_down_body.points.empty() ? nullptr : &feats_down_body.points[0].x,
                             (int)feats_down_body.points.size(), stride));
}
// PointVector = ikd-Tree's flattened storage (KD_TREE::flatten, include/ikd-Tree/ikd_Tree.cpp:1247-1273)
template <class PointVector>
inline void upload_map(flb_handle* h, const PointVector& map_points) {
    const int stride = (int)(sizeof(map_points[0]) / sizeof(float));
    check(h, flb_map_upload(h, &map_points[0].x, (int)map_points.size(), stride));
}

// ---- live LIO: the whole iterated update (src/laserMapping.cpp:1504-1733) -------------------
// On return `state` holds the updated state and covariance; the report carries effct_feat_num,
// res_mean_last and the pass counts the reference prints (:1784-1805).
template <class StatesGroup>
inline flb_lio_report lio_update(flb_handle* h, const flb_lio_params& prm, StatesGroup& state, const StatesGroup& state_propagat) {
    flb_state18 x, xp;
    to_abi(state, x);
    to_abi(state_propagat, xp);
    flb_lio_report rep{};
    check(h, flb_lio_update(h, &prm, &x, &xp, &rep));
    from_abi(x, state);
    return rep;
}

// ---- map_incremental (src/laserMapping.cpp:692-706) from the uploaded scan ---------------------
// Replaces the pointBodyToWorld loop over feats_down_body and ikdtree.Add_Points(feats_down_world, true) with
// downsample_size = filter_size_map_min: the scan uploaded for this frame (upload_scan) is transformed on the device.
// 18-DoF path: at the device state the LIO update just left (call it right after lio_update).
inline void map_incremental(flb_handle* h, const flb_lio_params& lio_prm, float filter_size_map_min) {
    check(h, flb_map_add_scan(h, &lio_prm, nullptr, nullptr, filter_size_map_min));
}
// Explicit pose (R: Mat3 with operator()(i, j), p: Vec3) with lio_prm's extrinsic.  IKFoM callers (RGBpointBodyToWorld
// under USE_IKFOM): R = s.rot.toRotationMatrix(), p = s.pos, and lio_prm.R_LI / t_LI from s.offset_R_L_I.toRotationMatrix()
// / s.offset_T_L_I (make_lio_params).
template <class Mat3, class Vec3>
inline void map_incremental(flb_handle* h, const flb_lio_params& lio_prm, const Mat3& R, const Vec3& p, float filter_size_map_min) {
    double Rm[9], pv[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rm[3 * i + j] = R(i, j);
        pv[i] = p(i);
    }
    check(h, flb_map_add_scan(h, &lio_prm, Rm, pv, filter_size_map_min));
}

// ---- publish_effect_world (src/laserMapping.cpp:871-885) from the last LIO pass on the device -----------------
// Fills `laserCloudWorld` (a PCL cloud: resize(n) and .points with x, y, z) with laserCloudOri of the last LIO pass
// (:1588-1600) transformed by RGBpointBodyToWorld; the caller converts and publishes it as before.  x, y, z are written,
// and the intensity too when the scan carries one (flb::preprocess -> undistort_pcl_on_device -> downsample_scan);
// with a host-uploaded scan the points' other fields are left as they were.  18-DoF path: at the device state the LIO
// update left.
template <class PointCloud>
inline int effect_cloud_fill(flb_handle* h, int n, PointCloud& cloud) {
    std::vector<float> rec((size_t)n * 12);
    int m = 0;
    const int rc = flb_effect_cloud_download_points(h, rec.data(), n, &m);
    const bool with_intensity = rc == FLB_OK;
    if (!with_intensity) {
        if (rc != FLB_ERR_STATE) check(h, rc);
        check(h, flb_effect_cloud_download(h, rec.data(), n, &m));   // no intensity: packed x, y, z
    }
    cloud.resize((size_t)n);
    const size_t w = with_intensity ? 12 : 3;
    for (int i = 0; i < n; ++i) {
        cloud.points[i].x = rec[w * (size_t)i];
        cloud.points[i].y = rec[w * (size_t)i + 1];
        cloud.points[i].z = rec[w * (size_t)i + 2];
        if (with_intensity) cloud.points[i].intensity = rec[w * (size_t)i + 8];
    }
    return n;
}
template <class PointCloud>
inline int publish_effect_world(flb_handle* h, const flb_lio_params& lio_prm, PointCloud& laserCloudWorld) {
    int n = 0;
    check(h, flb_effect_cloud(h, &lio_prm, nullptr, nullptr, &n));
    return effect_cloud_fill(h, n, laserCloudWorld);
}
// IKFoM callers: R = state_point.rot.toRotationMatrix(), p = state_point.pos, and lio_prm.R_LI / t_LI from
// state_point.offset_R_L_I.toRotationMatrix() / offset_T_L_I (make_lio_params), as for map_incremental.
template <class Mat3, class Vec3, class PointCloud>
inline int publish_effect_world(flb_handle* h, const flb_lio_params& lio_prm, const Mat3& R, const Vec3& p, PointCloud& laserCloudWorld) {
    double Rm[9], pv[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rm[3 * i + j] = R(i, j);
        pv[i] = p(i);
    }
    int n = 0;
    check(h, flb_effect_cloud(h, &lio_prm, Rm, pv, &n));
    return effect_cloud_fill(h, n, laserCloudWorld);
}

// ---- publish_frame_world (src/laserMapping.cpp:780-813, img_enable: 0) and its pcd_save_en map from the device --------
// The intensity records are pcl::PointXYZINormal's layout: x y z data[3] | normal data_n | intensity curvature 0 0.  P
// (PointType) must be that type, and its default constructor must leave data[3] = 1 and the rest zero, because the
// records carry those bytes (RGBpointBodyToWorld writes into a fresh PointCloudXYZI(size, 1)).
template <class P>
inline void xyzi_point_check() {
    static_assert(sizeof(P) == 48, "PointType must be pcl::PointXYZINormal's 48 bytes");
    static_assert(offsetof(P, intensity) == 32 && offsetof(P, curvature) == 36,
                  "PointType's intensity and curvature must sit at bytes 32 and 36");
    static const bool defaults_ok = [] {
        const P p{};
        return p.data[3] == 1.0f && p.normal_x == 0.f && p.normal_y == 0.f && p.normal_z == 0.f && p.intensity == 0.f &&
               p.curvature == 0.f;
    }();
    if (!defaults_ok)
        throw Error(FLB_ERR_INVALID, "flb: PointType() does not construct data[3] = 1 and zero normal / intensity / curvature "
                                     "(the intensity records do)");
}
// Fills the published cloud of publish_frame_world (pcl_wait_pub) from the world cloud (flb_world_cloud of a source that
// carries intensity: flb::preprocess, undistort_pcl_on_device and, for dense_map_en = 0, downsample_scan), one copy and
// no host loop.  With pcd_save_en, flb_lidar_save_begin at start-up makes it append to the device's save too (:812).
template <class PointCloud>
inline int publish_frame_world(flb_handle* h, PointCloud& pcl_wait_pub) {
    xyzi_point_check<typename std::decay<decltype(pcl_wait_pub.points[0])>::type>();
    int n = 0;
    check(h, flb_world_cloud_download(h, nullptr, 0, &n));       // the count only
    pcl_wait_pub.resize((size_t)n);
    check(h, flb_world_cloud_points(h, n > 0 ? &pcl_wait_pub.points[0] : nullptr, n, &n));   // one copy, and the save's append
    return n;
}
// pcl_wait_save_lidar at exit (intensity_sacn_all.pcd, :1848-1853): the whole device save, filled slice by slice.
// Throws flb::Error when frames were dropped at flb_lidar_save_begin's cap: a map with holes is not written silently.
template <class PointCloud>
inline int64_t save_intensity_map(flb_handle* h, PointCloud& pcl_wait_save_lidar) {
    xyzi_point_check<typename std::decay<decltype(pcl_wait_save_lidar.points[0])>::type>();
    int64_t n = 0, dropped = 0;
    check(h, flb_lidar_save_size(h, &n, &dropped, nullptr));
    if (dropped > 0)
        throw Error(FLB_ERR_STATE, "flb::save_intensity_map: " + std::to_string((long long)dropped) +
                                       " points were dropped at flb_lidar_save_begin's max_points");
    pcl_wait_save_lidar.resize((size_t)n);
    const int64_t kSlice = (int64_t)1 << 22;
    for (int64_t first = 0; first < n; first += kSlice)
        check(h, flb_lidar_save_download(h, first, n - first < kSlice ? n - first : kSlice, &pcl_wait_save_lidar.points[(size_t)first]));
    return n;
}

// ---- publish_frame_world_rgb (src/laserMapping.cpp:710-777) and the pcd_save_en map from the device ---------------
// flb_rgb_cloud's records are pcl::PointXYZRGB's layout: x y z data[3] | b g r a | 12 zero bytes.  P (PointTypeRGB) must
// be that type, and its default constructor must leave data[3] = 1 and a = 255 (PCL 1.8 and later), because the records
// carry those bytes: a PCL with other defaults is refused at the first use instead of saving other bytes.
template <class P>
inline void rgb_point_check() {
    static_assert(sizeof(P) == 32, "PointTypeRGB must be pcl::PointXYZRGB's 32 bytes");
    static_assert(offsetof(P, b) == 16 && offsetof(P, g) == 17 && offsetof(P, r) == 18 && offsetof(P, a) == 19,
                  "PointTypeRGB's colour must sit at bytes 16..19 (b, g, r, a)");
    static const bool defaults_ok = [] {
        const P p{};
        return p.data[3] == 1.0f && p.a == 255;
    }();
    if (!defaults_ok)
        throw Error(FLB_ERR_INVALID, "flb: PointTypeRGB() does not construct data[3] = 1 and a = 255 (flb_rgb_cloud's records do)");
}
template <class PointCloud>
inline int rgb_cloud_fill(flb_handle* h, int n, PointCloud& cloud) {
    cloud.resize((size_t)n);
    int m = 0;
    if (n > 0) check(h, flb_rgb_cloud_download(h, &cloud.points[0], n, &m));
    return n;
}
// Fills laserCloudWorldRGB (:726-747, one copy, no host loop) from the world cloud (flb_world_cloud) coloured with the
// current image set's colour frame (flb::upload_camera_frame / upload_camera_msg), at the device state's camera pose
// (after flb_vmap_reset).  With pcd_save_en, flb_rgb_save_begin at start-up makes it append to the device's save too.
template <class PointCloud>
inline int publish_frame_world_rgb(flb_handle* h, PointCloud& laserCloudWorldRGB) {
    rgb_point_check<typename std::decay<decltype(laserCloudWorldRGB.points[0])>::type>();
    int n = 0;
    check(h, flb_rgb_cloud(h, nullptr, nullptr, nullptr, 0, &n));
    return rgb_cloud_fill(h, n, laserCloudWorldRGB);
}
// The same at an explicit camera pose: Rcw = new_frame_->T_f_w_.rotation_matrix(), Pcw = its translation().
template <class Mat3, class Vec3, class PointCloud>
inline int publish_frame_world_rgb(flb_handle* h, const Mat3& Rcw, const Vec3& Pcw, PointCloud& laserCloudWorldRGB) {
    rgb_point_check<typename std::decay<decltype(laserCloudWorldRGB.points[0])>::type>();
    double Rm[9], pv[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) Rm[3 * i + j] = Rcw(i, j);
        pv[i] = Pcw(i);
    }
    int n = 0;
    check(h, flb_rgb_cloud(h, Rm, pv, nullptr, 0, &n));
    return rgb_cloud_fill(h, n, laserCloudWorldRGB);
}
// pcl_wait_save at exit (:1839-1846): the whole device save, filled slice by slice, for pcd_writer.writeBinary.  Throws
// flb::Error when frames were dropped at flb_rgb_save_begin's cap: a map with holes is not written silently.
template <class PointCloud>
inline int64_t save_rgb_map(flb_handle* h, PointCloud& pcl_wait_save) {
    rgb_point_check<typename std::decay<decltype(pcl_wait_save.points[0])>::type>();
    int64_t n = 0, dropped = 0;
    check(h, flb_rgb_save_size(h, &n, &dropped, nullptr));
    if (dropped > 0)
        throw Error(FLB_ERR_STATE, "flb::save_rgb_map: " + std::to_string((long long)dropped) +
                                       " points were dropped at flb_rgb_save_begin's max_points");
    pcl_wait_save.resize((size_t)n);
    const int64_t kSlice = (int64_t)1 << 22;
    for (int64_t first = 0; first < n; first += kSlice)
        check(h, flb_rgb_save_download(h, first, n - first < kSlice ? n - first : kSlice, &pcl_wait_save.points[(size_t)first]));
    return n;
}

// ---- lasermap_fov_segment (src/laserMapping.cpp:363-421) with the cube on the device ---------------
// Replaces lasermap_fov_segment() and its ikdtree.Delete_Point_Boxes(cub_needrm): the cube steps at the device state's
// position (state.pos_end; call it where the reference does, :1395, after the propagation) and the points in its boxes
// leave the device map.  kdtree_delete_counter receives the number of deleted points (:417).  DET_RANGE and
// MOV_THRESHOLD default to the reference's constants (:83, :90).
inline void lasermap_fov_segment(flb_handle* h, double cube_len, int* kdtree_delete_counter = nullptr, float det_range = 300.0f,
                                 float mov_threshold = 1.5f) {
    const flb_fov_params prm{cube_len, det_range, mov_threshold};
    check(h, flb_map_fov_segment(h, &prm, nullptr, nullptr, nullptr, nullptr, kdtree_delete_counter));
}
// IKFoM callers: pos_LiD = pos_lid (Vec3 with operator()(i), :1289).  Not a pointer: lasermap_fov_segment(h, cube_len,
// nullptr) is the overload above with no counter.
template <class Vec3, class = typename std::enable_if<!std::is_pointer<typename std::decay<Vec3>::type>::value &&
                                                      !std::is_same<typename std::decay<Vec3>::type, std::nullptr_t>::value>::type>
inline void lasermap_fov_segment(flb_handle* h, double cube_len, const Vec3& pos_lid, int* kdtree_delete_counter = nullptr,
                                 float det_range = 300.0f, float mov_threshold = 1.5f) {
    const flb_fov_params prm{cube_len, det_range, mov_threshold};
    const double p[3] = {pos_lid(0), pos_lid(1), pos_lid(2)};
    check(h, flb_map_fov_segment(h, &prm, p, nullptr, nullptr, nullptr, kdtree_delete_counter));
}

// ---- IKFoM-typed measurement callback (src/laserMapping.cpp:960-1094) ------------------------
// StateIkfom: .pos (vect3), .rot / .offset_R_L_I (MTK SO3, Eigen quaternion: toRotationMatrix()),
//             .offset_T_L_I (vect3)                     (include/use-ikfom.hpp:12-21)
// DynShare  : esekfom::dyn_share_datastruct<double>: .valid .converge .h_x (MatrixXd) .h (VectorXd)
//             (include/IKFoM_toolkit/esekfom/esekfom.hpp:79-89)
// The scan must have been uploaded (upload_scan) before kf.update_iterated_dyn_share_modified().
// Side effects mirrored for the caller: effct_feat_num, res_mean_last, and the scan indices of the
// effective rows (laserCloudOri order) for publish_effect_world (:871-885).
template <class StateIkfom, class DynShare>
inline void h_share_model(flb_handle* h, double laser_point_cov, StateIkfom& s, DynShare& ekfom_data, int& effct_feat_num,
                          double& res_mean_last, std::vector<int>* effective_scan_idx = nullptr) {
    flb_lio_params prm{};
    const auto R_LI = s.offset_R_L_I.toRotationMatrix();
    const auto R = s.rot.toRotationMatrix();
    double Rm[9], pv[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) { prm.R_LI[3 * i + j] = R_LI(i, j); Rm[3 * i + j] = R(i, j); }
        prm.t_LI[i] = s.offset_T_L_I(i);
        pv[i] = s.pos(i);
    }
    prm.laser_point_cov = laser_point_cov;
    flb_normal_eq eq{};
    check(h, flb_lio_pass(h, &prm, Rm, pv, ekfom_data.converge ? 1 : 0, 12, &eq));   // :994 converge => redo kNN
    const int n = eq.n_eff;
    std::vector<double> rows((size_t)n * 12 + 1), meas((size_t)n + 1);
    std::vector<int> idx((size_t)n + 1);
    int n_rows = 0;
    check(h, flb_lio_export(h, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, rows.data(), meas.data(), idx.data(), &n_rows));
    effct_feat_num = n_rows;                                      // :1039-1052
    res_mean_last = eq.sum_abs_res / n_rows;                      // :1054
    ekfom_data.h_x.resize(n_rows, 12);                            // :1059  (MatrixXd::Zero(effct_feat_num, 12))
    ekfom_data.h.resize(n_rows);                                  // :1060
    for (int r = 0; r < n_rows; ++r) {
        for (int c = 0; c < 12; ++c) ekfom_data.h_x(r, c) = rows[(size_t)r * 12 + c];   // :1082
        ekfom_data.h(r) = meas[r];                                                      // :1088
    }
    if (effective_scan_idx) effective_scan_idx->assign(idx.begin(), idx.begin() + n_rows);
}

// ---- VIO: ComputeJ (src/lidar_selection.cpp:967-983) -------------------------------------------
// Image : cv::Mat-like: .data (uint8*), .cols, .rows, .step (bytes per row)
// SubMap: SubSparseMap (include/common_lib.h:263-292): .voxel_points[i]->pos_ (Vector3d, may be nullptr),
//         .patch[i] (vector<float>, 3*64), .search_levels[i], .errors[i]
// Patches with a null voxel point are dropped (the reference `continue`s over them, :798).
template <class Mat3, class Vec3>
inline flb_vio_params make_vio_params(const Mat3& Rcl, const Vec3& Pcl, const Mat3& Lidar_rot_to_IMU,
                                      const Vec3& Lidar_offset_to_IMU, double img_point_cov, int max_iteration) {
    flb_vio_params p{};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) { p.Rcl[3 * i + j] = Rcl(i, j); p.R_LI[3 * i + j] = Lidar_rot_to_IMU(i, j); }
        p.Pcl[i] = Pcl(i);
        p.t_LI[i] = Lidar_offset_to_IMU(i);
    }
    p.img_point_cov = img_point_cov;
    p.max_iteration = max_iteration;
    p.conv_rot_deg = 0.001f;   // src/lidar_selection.cpp:883
    p.conv_pos_cm = 0.001f;
    p.force_all_passes = 0;
    return p;
}

// ---- the camera frame (LidarSelector::detect, src/lidar_selection.cpp:1029-1037) --------------------------------
// Image: cv::Mat-like BGR8 frame (.data, .cols, .rows, .step) as getImageFromMsg(..., "bgr8") delivers it, at the
// camera's size or twice it.  The device halves it when needed, keeps the colour frame for flb_colorize(_cloud) with
// bgr = nullptr and makes the gray image every VIO / visual-map call reads.  gray_rule: FLB_GRAY_CV4 or FLB_GRAY_CV3,
// the cvtColor of the OpenCV the caller links (CV_VERSION_MAJOR).
template <class Image>
inline void upload_camera_frame(flb_handle* h, const Image& bgr, int gray_rule) {
    check(h, flb_image_upload_bgr(h, bgr.data, bgr.cols, bgr.rows, (int)bgr.step, gray_rule));
}

// The FLB_ENC_* of a sensor_msgs::Image encoding string (sensor_msgs/image_encodings.h); any other string throws
// flb::Error (FLB_ERR_INVALID) before anything is uploaded, so the caller can fall back to cv_bridge.
inline int camera_encoding(const std::string& encoding) {
    static const struct { const char* name; int enc; } table[] = {
        {"bgr8", FLB_ENC_BGR8},   {"rgb8", FLB_ENC_RGB8},   {"mono8", FLB_ENC_MONO8},
        {"bgra8", FLB_ENC_BGRA8}, {"rgba8", FLB_ENC_RGBA8}, {"bayer_rggb8", FLB_ENC_BAYER_RGGB8},
        {"bayer_bggr8", FLB_ENC_BAYER_BGGR8}, {"bayer_gbrg8", FLB_ENC_BAYER_GBRG8}, {"bayer_grbg8", FLB_ENC_BAYER_GRBG8}};
    for (const auto& e : table)
        if (encoding == e.name) return e.enc;
    throw Error(FLB_ERR_INVALID, "flb::camera_encoding: encoding '" + encoding + "' is not taken on the device");
}
// ImageMsg: sensor_msgs::Image-like (.encoding, .width, .height, .step, .data with .data()), the message img_cbk
// receives (src/laserMapping.cpp:490-493).  Replaces getImageFromMsg + upload_camera_frame: the message's own bytes go
// up and the device converts, demosaics and resizes them as cv_bridge::toCvCopy(msg, "bgr8") and detect() would.
template <class ImageMsg>
inline void upload_camera_msg(flb_handle* h, const ImageMsg& msg, int gray_rule) {
    const int enc = camera_encoding(msg.encoding);
    check(h, flb_image_upload_msg(h, msg.data.data(), (int)msg.width, (int)msg.height, (int)msg.step, enc, gray_rule));
}

// ---- display_keypatch (src/lidar_selection.cpp:985-1005) on the device ---------------------------------------------
// Mat: cv::Mat-like camera-size CV_8UC3 (.data, .cols, .rows, .step), img_cp.  The device draws the circles of the current
// patch list into it (flb_keypatch_image, the pose the VIO update left on the device); a page-locked img_cp (its data
// from flb_host_alloc) is filled by the copy engine in place.  When there are patches, put_text(img_cp, text, x, y)
// draws the rate as :1000-1004 do (text = to_string(int(1 / time)) + " HZ" at (20, 20)); with none, display_keypatch
// returns before its text and so does this.  Returns the patch count.
template <class Mat, class PutText>
inline int display_keypatch(flb_handle* h, Mat& img_cp, double time, PutText put_text) {
    int n = 0;
    check(h, flb_keypatch_image(h, nullptr, nullptr, img_cp.data, (int)img_cp.step, &n));
    check(h, flb_synchronize(h));                     // the bytes of a page-locked img_cp land with the stream
    if (n == 0) return 0;                             // :987-988
    put_text(img_cp, std::to_string(int(1 / time)) + " HZ", 20.0f, 20.0f);
    return n;
}
#if defined(CV_VERSION_MAJOR)
// With OpenCV included first: the reference's own putText (:1003).
inline int display_keypatch(flb_handle* h, cv::Mat& img_cp, double time) {
    return display_keypatch(h, img_cp, time, [](cv::Mat& img, const std::string& text, float x, float y) {
        cv::putText(img, text, cv::Point2f(x, y), cv::FONT_HERSHEY_COMPLEX, 0.6, cv::Scalar(255, 255, 255), 1, 8, 0);
    });
}
#endif

template <class Image, class SubMap, class StatesGroup>
inline flb_vio_report compute_j(flb_handle* h, const flb_vio_params& prm, const Image& img, SubMap& sub_sparse_map,
                                StatesGroup& state, const StatesGroup& state_propagat) {
    const int total = (int)sub_sparse_map.index.size();
    flb_vio_report rep{};
    if (total == 0) return rep;                                    // :969-970
    std::vector<double> pos;
    std::vector<float> patch;
    std::vector<int> level, src;
    pos.reserve((size_t)total * 3);
    patch.reserve((size_t)total * 192);
    for (int i = 0; i < total; ++i) {
        const auto& pt = sub_sparse_map.voxel_points[i];
        if (pt == nullptr) continue;                               // :798
        for (int k = 0; k < 3; ++k) pos.push_back(pt->pos_(k));
        patch.insert(patch.end(), sub_sparse_map.patch[i].begin(), sub_sparse_map.patch[i].begin() + 192);
        level.push_back(sub_sparse_map.search_levels[i]);
        src.push_back(i);
    }
    check(h, flb_image_upload(h, img.data, img.cols, img.rows, (int)img.step));
    check(h, flb_patches_upload(h, pos.data(), patch.data(), level.data(), (int)level.size()));
    flb_state18 x, xp;
    to_abi(state, x);
    to_abi(state_propagat, xp);
    check(h, flb_vio_update(h, &prm, &x, &xp, &rep));
    from_abi(x, state);
    // sub_sparse_map->errors[i] = patch_error of the last executed pass (:851; display_keypatch reads it, :995)
    std::vector<float> err(level.size());
    check(h, flb_vio_errors(h, err.data(), (int)err.size()));
    for (size_t k = 0; k < src.size(); ++k) sub_sparse_map.errors[src[k]] = err[k];
    return rep;
}

// ---- VIO: one pyramid level, float LidarSelector::UpdateState(cv::Mat img, float total_residual, int level)
// (include/lidar_selection.h:72, src/lidar_selection.cpp:743-902).  The caller keeps its own ComputeJ loop (:974-981):
//     for (level = 2; level >= 0; level--) now_error = flb::update_state(h, prm, img, *sub_sparse_map, *state, *state_propagat, error, level, G);
//     if (now_error < error) state->cov -= G * state->cov;
// G: the caller's 18 x 18 member (anything with operator()(i, j)); its first six columns are rewritten whenever a pass
// of this call was accepted, exactly as :874 does.  The image / patch upload happens on the first level only
// (level == 2) unless `upload` says otherwise.
template <class Image, class SubMap, class StatesGroup, class Mat18>
inline float update_state(flb_handle* h, const flb_vio_params& prm, const Image& img, SubMap& sub_sparse_map, StatesGroup& state,
                          const StatesGroup& state_propagat, float total_residual, int level, Mat18& G, int upload = -1) {
    const int total = (int)sub_sparse_map.index.size();
    if (total == 0) return 0.f;                                    // :746
    std::vector<int> src;
    for (int i = 0; i < total; ++i)
        if (sub_sparse_map.voxel_points[i] != nullptr) src.push_back(i);
    if (upload > 0 || (upload < 0 && level == 2)) {
        std::vector<double> pos;
        std::vector<float> patch;
        std::vector<int> lv;
        for (int i : src) {
            for (int k = 0; k < 3; ++k) pos.push_back(sub_sparse_map.voxel_points[i]->pos_(k));
            patch.insert(patch.end(), sub_sparse_map.patch[i].begin(), sub_sparse_map.patch[i].begin() + 192);
            lv.push_back(sub_sparse_map.search_levels[i]);
        }
        check(h, flb_image_upload(h, img.data, img.cols, img.rows, (int)img.step));
        check(h, flb_patches_upload(h, pos.data(), patch.data(), lv.data(), (int)lv.size()));
    }
    flb_state18 x, xp;
    to_abi(state, x);
    to_abi(state_propagat, xp);
    float last_error = 0.f;
    double Gc[108];
    flb_vio_report rep{};
    check(h, flb_vio_update_level(h, &prm, level, total_residual, &x, &xp, &last_error, Gc, &rep));
    from_abi(x, state);
    if (rep.passes[level] > 0 && last_error < total_residual)     // at least one pass was accepted: G was rewritten (:874)
        for (int i = 0; i < 18; ++i)
            for (int j = 0; j < 6; ++j) G(i, j) = Gc[6 * i + j];
    std::vector<float> err(src.size());
    check(h, flb_vio_errors(h, err.data(), (int)err.size()));
    for (size_t k = 0; k < src.size(); ++k) sub_sparse_map.errors[src[k]] = err[k];
    return last_error;
}

// ---- IMU forward propagation + backward undistortion (src/IMU_Processing.cpp:655-808) ----------------
// ImuDeque  : the reference's `v_imu` (std::deque<sensor_msgs::Imu::ConstPtr>, last_imu_ pushed to the front,
//             :617-618): elements dereference to .header.stamp.toSec(), .angular_velocity.{x,y,z},
//             .linear_acceleration.{x,y,z}
// PointCloud: pcl_out (:623-639), already cut to this update's points, in time order; compensated in place.
// `carry` holds ImuProcess::last_lidar_end_time_, acc_s_last, angvel_last (the caller keeps `last_imu_ =
// v_imu.back()` itself, :760).  On return state_inout is the propagated state (rot/pos/vel_end, cov).
template <class Mat3, class Vec3>
inline flb_imu_params make_imu_params(const Vec3& cov_gyr, const Vec3& cov_acc, const Vec3& cov_bias_gyr, const Vec3& cov_bias_acc,
                                      double G_m_s2, double mean_acc_norm, const Mat3& Lid_rot_to_IMU, const Vec3& Lid_offset_to_IMU) {
    flb_imu_params p{};
    for (int i = 0; i < 3; ++i) {
        p.cov_gyr[i] = cov_gyr(i); p.cov_acc[i] = cov_acc(i); p.cov_bias_gyr[i] = cov_bias_gyr(i); p.cov_bias_acc[i] = cov_bias_acc(i);
        p.t_LI[i] = Lid_offset_to_IMU(i);
        for (int j = 0; j < 3; ++j) p.R_LI[3 * i + j] = Lid_rot_to_IMU(i, j);
    }
    p.G_m_s2 = G_m_s2;
    p.mean_acc_norm = mean_acc_norm;
    return p;
}

namespace detail {
// out == nullptr: the compensated points stay on the device
template <class ImuDeque, class StatesGroup, class PointCloud>
inline void undistort(flb_handle* h, const flb_imu_params& prm, flb_imu_carry& carry, const ImuDeque& v_imu, double pcl_beg_time,
                      double pcl_end_time, StatesGroup& state_inout, const PointCloud& pcl, float* out) {
    std::vector<flb_imu_sample> s;
    s.reserve(v_imu.size());
    for (const auto& m : v_imu) {
        flb_imu_sample e;
        e.t = m->header.stamp.toSec();
        e.gyr[0] = m->angular_velocity.x; e.gyr[1] = m->angular_velocity.y; e.gyr[2] = m->angular_velocity.z;
        e.acc[0] = m->linear_acceleration.x; e.acc[1] = m->linear_acceleration.y; e.acc[2] = m->linear_acceleration.z;
        s.push_back(e);
    }
    flb_state18 x{};
    to_abi(state_inout, x);
    check(h, flb_state_upload(h, &x, &x));
    static_assert(sizeof(pcl.points[0]) % sizeof(float) == 0, "point type must be float-packed");
    const int stride = (int)(sizeof(pcl.points[0]) / sizeof(float));
    const int n = (int)pcl.points.size();
    const int off = n ? (int)(&pcl.points[0].curvature - &pcl.points[0].x) : 3;
    check(h, flb_imu_undistort(h, &prm, &carry, s.data(), (int)s.size(), pcl_beg_time, pcl_end_time,
                               n ? &pcl.points[0].x : nullptr, n ? stride : 4, off, n, out, nullptr, nullptr));
    check(h, flb_state_download(h, &x, nullptr, nullptr));
    from_abi(x, state_inout);
}
}  // namespace detail

template <class ImuDeque, class StatesGroup, class PointCloud>
inline void undistort_pcl(flb_handle* h, const flb_imu_params& prm, flb_imu_carry& carry, const ImuDeque& v_imu,
                          double pcl_beg_time, double pcl_end_time, StatesGroup& state_inout, PointCloud& pcl_out) {
    const int n = (int)pcl_out.points.size();
    std::vector<float> out((size_t)n * 3 + 1);
    detail::undistort(h, prm, carry, v_imu, pcl_beg_time, pcl_end_time, state_inout, pcl_out, out.data());
    for (int i = 0; i < n; ++i) {
        pcl_out.points[i].x = out[3 * (size_t)i];
        pcl_out.points[i].y = out[3 * (size_t)i + 1];
        pcl_out.points[i].z = out[3 * (size_t)i + 2];
    }
}

// The same propagation and undistortion, with pcl_in left as it is: feats_undistort exists only on the device, where
// downsample_scan turns it into this frame's scan (and flb_world_cloud(FLB_CLOUD_UNDISTORTED) reads it).
template <class ImuDeque, class StatesGroup, class PointCloud>
inline void undistort_pcl_on_device(flb_handle* h, const flb_imu_params& prm, flb_imu_carry& carry, const ImuDeque& v_imu,
                                    double pcl_beg_time, double pcl_end_time, StatesGroup& state_inout, const PointCloud& pcl_in) {
    detail::undistort(h, prm, carry, v_imu, pcl_beg_time, pcl_end_time, state_inout, pcl_in, nullptr);
}

// downSizeFilterSurf.setInputCloud(feats_undistort); downSizeFilterSurf.filter(*feats_down_body); then upload_scan
// (src/laserMapping.cpp:1398-1399), all on the device.  Returns feats_down_size (:1400).
inline int downsample_scan(flb_handle* h, float filter_size_surf_min) {
    int n = 0;
    check(h, flb_scan_from_undistorted(h, filter_size_surf_min, &n));
    return n;
}

// ---- the driver's LiDAR message (Preprocess::process, src/preprocess.cpp:43-70, with feature_extract_enable = 0) ----
struct LidarInfo {
    int n_points;            // pl_surf.size(): sync_packages skips the message when it is <= 1 (src/laserMapping.cpp:538)
    float last_offset_ms;    // points.back().curvature after the sort, for lidar_end_time (:553)
};

// livox_ros_driver::CustomMsg (.points, .point_num): avia_handler.  CustomPoint is offset_time, x, y, z, reflectivity,
// tag, line; the offsets are taken from the type itself.
template <class LivoxMsg>
inline LidarInfo preprocess(flb_handle* h, const LivoxMsg& msg, int n_scans, double blind, int point_filter_num) {
    flb_lidar_format f{};
    f.kind = FLB_LIDAR_LIVOX;
    f.point_step = (int)sizeof(msg.points[0]);
    LidarInfo r{};
    const int n = (int)msg.point_num;
    if (n > 0) {
        const char* p0 = reinterpret_cast<const char*>(&msg.points[0]);
        f.off_time = (int)(reinterpret_cast<const char*>(&msg.points[0].offset_time) - p0);
        f.off_x = (int)(reinterpret_cast<const char*>(&msg.points[0].x) - p0);
        f.off_y = (int)(reinterpret_cast<const char*>(&msg.points[0].y) - p0);
        f.off_z = (int)(reinterpret_cast<const char*>(&msg.points[0].z) - p0);
        f.off_tag = (int)(reinterpret_cast<const char*>(&msg.points[0].tag) - p0);
        f.off_line = (int)(reinterpret_cast<const char*>(&msg.points[0].line) - p0);
    } else {
        f.off_x = 4, f.off_y = 8, f.off_z = 12, f.off_tag = 17, f.off_line = 18;
    }
    const int off_intensity = (int)offsetof(typename std::decay<decltype(msg.points[0])>::type, reflectivity);
    f.n_scans = n_scans;
    f.point_filter_num = point_filter_num;
    f.blind = blind;
    check(h, flb_lidar_upload_intensity(h, &f, off_intensity, n > 0 ? &msg.points[0] : nullptr, n, &r.n_points, &r.last_offset_ms));
    return r;
}

// The PointCloud2's `intensity` field when it is FLOAT32, else -1: pcl::fromROSMsg maps a field into the typed cloud only
// when name and datatype match, so any other intensity leaves every point's at 0.
template <class PointCloud2>
inline int intensity_field(const PointCloud2& msg) {
    enum { kFloat32 = 7 };                               // sensor_msgs::PointField::FLOAT32
    for (const auto& fld : msg.fields)
        if (fld.name == "intensity" && (int)fld.datatype == kFloat32) return (int)fld.offset;
    return -1;
}

// sensor_msgs::PointCloud2 (.fields[].name / .offset, .point_step, .width, .height, .data): oust64_handler,
// velodyne_handler (clouds with per-point times) or xt32_handler by `kind` (FLB_LIDAR_*).  The time field is the one
// the handler's point type names: t (Ouster), time (Velodyne), timestamp (XT32).  The intensity is kept (intensity_field).
template <class PointCloud2>
inline LidarInfo preprocess(flb_handle* h, const PointCloud2& msg, int kind, int n_scans, double blind, int point_filter_num) {
    flb_lidar_format f{};
    f.kind = kind;
    f.point_step = (int)msg.point_step;
    f.off_x = f.off_y = f.off_z = f.off_time = -1;
    const char* time_name = kind == FLB_LIDAR_OUSTER ? "t" : (kind == FLB_LIDAR_VELODYNE ? "time" : "timestamp");
    for (const auto& fld : msg.fields) {
        if (fld.name == "x") f.off_x = (int)fld.offset;
        else if (fld.name == "y") f.off_y = (int)fld.offset;
        else if (fld.name == "z") f.off_z = (int)fld.offset;
        else if (fld.name == time_name) f.off_time = (int)fld.offset;
    }
    f.n_scans = n_scans;
    f.point_filter_num = point_filter_num;
    f.blind = blind;
    LidarInfo r{};
    const int n = (int)((size_t)msg.width * msg.height);
    check(h, flb_lidar_upload_intensity(h, &f, intensity_field(msg), n > 0 ? msg.data.data() : nullptr, n, &r.n_points,
                                        &r.last_offset_ms));
    return r;
}

// sensor_msgs::PointCloud2 of any Velodyne driver: velodyne_handler with or without per-point times, fields at any
// offset.  x, y, z (FLOAT32) and ring (UINT16) are looked up by name, time (FLOAT32) when the cloud has one; a missing
// field or another datatype throws.  The intensity is kept (intensity_field).  yaw_times = the times came from the yaw angle (!given_offset_time, src/preprocess.cpp:279).
struct VelodyneInfo : LidarInfo {
    bool yaw_times;
};
template <class PointCloud2>
inline VelodyneInfo preprocess_velodyne(flb_handle* h, const PointCloud2& msg, int n_scans, double blind, int point_filter_num) {
    enum { kUint16 = 4, kFloat32 = 7 };                  // sensor_msgs::PointField datatypes
    flb_velodyne_format f{};
    f.point_step = (int)msg.point_step;
    f.off_x = f.off_y = f.off_z = f.off_time = f.off_ring = -1;
    for (const auto& fld : msg.fields) {
        int* off = fld.name == "x" ? &f.off_x : fld.name == "y" ? &f.off_y : fld.name == "z" ? &f.off_z
                 : fld.name == "time" ? &f.off_time : fld.name == "ring" ? &f.off_ring : nullptr;
        if (!off) continue;
        if ((int)fld.datatype != (off == &f.off_ring ? kUint16 : kFloat32))
            throw Error(FLB_ERR_INVALID, ("preprocess_velodyne: field " + std::string(fld.name) + " has the wrong datatype").c_str());
        *off = (int)fld.offset;
    }
    if (f.off_x < 0 || f.off_y < 0 || f.off_z < 0 || f.off_ring < 0)
        throw Error(FLB_ERR_INVALID, "preprocess_velodyne: the cloud lacks one of the fields x, y, z, ring");
    f.n_scans = n_scans;
    f.point_filter_num = point_filter_num;
    f.blind = blind;
    VelodyneInfo r{};
    int yaw = 0;
    const int n = (int)((size_t)msg.width * msg.height);
    check(h, flb_lidar_upload_velodyne_intensity(h, &f, intensity_field(msg), n > 0 ? msg.data.data() : nullptr, n, &r.n_points,
                                                 &r.last_offset_ms, &yaw));
    r.yaw_times = yaw != 0;
    return r;
}

// ---- feature_extract_enable = 1: the feature branches and give_feature, pl_surf on the device --------------------
// Preprocess::disB is never assigned by the reference's constructor (src/preprocess.cpp:12-13 assign disA twice), so a
// node runs with whatever its heap held.  p_pre is allocated once during static initialisation (src/laserMapping.cpp:208),
// from memory the process has not used before, which the OS hands out zeroed: 0 is the value such a node sees, and
// the adapters pass it.  A caller who wants another value calls flb_lidar_upload_features directly.
constexpr double kFeatureDisB = 0.0;

// livox_ros_driver::CustomMsg: avia_handler's feature branch (:94-135).  Offsets from the type, as flb::preprocess.
template <class LivoxMsg>
inline LidarInfo preprocess_features(flb_handle* h, const LivoxMsg& msg, int n_scans, double blind, int point_filter_num) {
    flb_lidar_format f{};
    f.kind = FLB_LIDAR_LIVOX;
    f.point_step = (int)sizeof(msg.points[0]);
    LidarInfo r{};
    const int n = (int)msg.point_num;
    if (n > 0) {
        const char* p0 = reinterpret_cast<const char*>(&msg.points[0]);
        f.off_time = (int)(reinterpret_cast<const char*>(&msg.points[0].offset_time) - p0);
        f.off_x = (int)(reinterpret_cast<const char*>(&msg.points[0].x) - p0);
        f.off_y = (int)(reinterpret_cast<const char*>(&msg.points[0].y) - p0);
        f.off_z = (int)(reinterpret_cast<const char*>(&msg.points[0].z) - p0);
        f.off_tag = (int)(reinterpret_cast<const char*>(&msg.points[0].tag) - p0);
        f.off_line = (int)(reinterpret_cast<const char*>(&msg.points[0].line) - p0);
    } else {
        f.off_x = 4, f.off_y = 8, f.off_z = 12, f.off_tag = 17, f.off_line = 18;
    }
    f.n_scans = n_scans;
    f.point_filter_num = point_filter_num;
    f.blind = blind;
    check(h, flb_lidar_upload_features(h, &f, kFeatureDisB, n > 0 ? &msg.points[0] : nullptr, n, &r.n_points, &r.last_offset_ms));
    return r;
}

// sensor_msgs::PointCloud2 of an Ouster (kind FLB_LIDAR_OUSTER: oust64_handler's feature branch, :174-227) or a Velodyne
// (FLB_LIDAR_VELODYNE: velodyne_handler's, :299-373, with or without per-point times).  Fields are looked up by name and
// their datatypes checked: x, y, z FLOAT32 and, for the Ouster, t UINT32 and ring UINT8; for the Velodyne ring UINT16 and
// time FLOAT32 when the cloud has one.  A missing field, another datatype or another kind throws before any upload.
template <class PointCloud2>
inline VelodyneInfo preprocess_features(flb_handle* h, const PointCloud2& msg, int kind, int n_scans, double blind,
                                        int point_filter_num) {
    enum { kUint8 = 2, kUint16 = 4, kUint32 = 6, kFloat32 = 7 };          // sensor_msgs::PointField datatypes
    if (kind != FLB_LIDAR_OUSTER && kind != FLB_LIDAR_VELODYNE)
        throw Error(FLB_ERR_INVALID, "preprocess_features: kind must be FLB_LIDAR_OUSTER or FLB_LIDAR_VELODYNE (the XT32 has no "
                                     "feature branch: flb::preprocess serves it)");
    const bool ouster = kind == FLB_LIDAR_OUSTER;
    int off_x = -1, off_y = -1, off_z = -1, off_time = -1, off_ring = -1;
    for (const auto& fld : msg.fields) {
        int* off = fld.name == "x" ? &off_x : fld.name == "y" ? &off_y : fld.name == "z" ? &off_z
                 : fld.name == (ouster ? "t" : "time") ? &off_time : fld.name == "ring" ? &off_ring : nullptr;
        if (!off) continue;
        const int want = off == &off_ring ? (ouster ? kUint8 : kUint16) : (off == &off_time && ouster) ? kUint32 : kFloat32;
        if ((int)fld.datatype != want)
            throw Error(FLB_ERR_INVALID, ("preprocess_features: field " + std::string(fld.name) + " has the wrong datatype").c_str());
        *off = (int)fld.offset;
    }
    if (off_x < 0 || off_y < 0 || off_z < 0 || off_ring < 0 || (ouster && off_time < 0))
        throw Error(FLB_ERR_INVALID, ouster ? "preprocess_features: the cloud lacks one of the fields x, y, z, t, ring"
                                            : "preprocess_features: the cloud lacks one of the fields x, y, z, ring");
    VelodyneInfo r{};
    const int n = (int)((size_t)msg.width * msg.height);
    const void* data = n > 0 ? msg.data.data() : nullptr;
    if (ouster) {
        flb_lidar_format f{};
        f.kind = FLB_LIDAR_OUSTER;
        f.point_step = (int)msg.point_step;
        f.off_x = off_x, f.off_y = off_y, f.off_z = off_z, f.off_time = off_time, f.off_line = off_ring;
        f.n_scans = n_scans;
        f.point_filter_num = point_filter_num;
        f.blind = blind;
        check(h, flb_lidar_upload_features(h, &f, kFeatureDisB, data, n, &r.n_points, &r.last_offset_ms));
        r.yaw_times = false;
    } else {
        flb_velodyne_format f{};
        f.point_step = (int)msg.point_step;
        f.off_x = off_x, f.off_y = off_y, f.off_z = off_z, f.off_time = off_time, f.off_ring = off_ring;
        f.n_scans = n_scans;
        f.point_filter_num = point_filter_num;
        f.blind = blind;
        int yaw = 0;
        check(h, flb_lidar_upload_velodyne_features(h, &f, kFeatureDisB, data, n, &r.n_points, &r.last_offset_ms, &yaw));
        r.yaw_times = yaw != 0;
    }
    return r;
}

// ImuProcess::UndistortPcl from :621 on, with the cloud of flb::preprocess as lidar_meas.lidar.  lidar_meas needs
// .lidar_beg_time, .last_update_time, .is_lidar_end, .lidar_scan_index_now and .measures.back().img_offset_time
// (include/common_lib.h's LidarMeasureGroup); last_offset_ms is LidarInfo's.  Returns pcl_out.size(); the undistorted
// points stay on the device for flb::downsample_scan / flb_world_cloud(FLB_CLOUD_UNDISTORTED).
template <class ImuDeque, class LidarMeasureGroup, class StatesGroup>
inline int undistort_pcl_from_lidar(flb_handle* h, const flb_imu_params& prm, flb_imu_carry& carry, const ImuDeque& v_imu,
                                    LidarMeasureGroup& lidar_meas, float last_offset_ms, StatesGroup& state_inout) {
    const double pcl_beg_time = lidar_meas.lidar_beg_time > lidar_meas.last_update_time ? lidar_meas.lidar_beg_time
                                                                                        : lidar_meas.last_update_time;   // :621
    const double pcl_end_time = lidar_meas.is_lidar_end ? lidar_meas.lidar_beg_time + last_offset_ms / double(1000)
                                                        : lidar_meas.lidar_beg_time + lidar_meas.measures.back().img_offset_time;   // :628-630
    const double pcl_offset_time = lidar_meas.is_lidar_end ? (pcl_end_time - lidar_meas.lidar_beg_time) * double(1000) : 0.0;   // :631-633
    std::vector<flb_imu_sample> s;
    s.reserve(v_imu.size());
    for (const auto& m : v_imu) {
        flb_imu_sample e;
        e.t = m->header.stamp.toSec();
        e.gyr[0] = m->angular_velocity.x; e.gyr[1] = m->angular_velocity.y; e.gyr[2] = m->angular_velocity.z;
        e.acc[0] = m->linear_acceleration.x; e.acc[1] = m->linear_acceleration.y; e.acc[2] = m->linear_acceleration.z;
        s.push_back(e);
    }
    flb_state18 x{};
    to_abi(state_inout, x);
    check(h, flb_state_upload(h, &x, &x));
    int n_taken = 0;
    check(h, flb_imu_undistort_lidar(h, &prm, &carry, s.data(), (int)s.size(), pcl_beg_time, pcl_end_time, pcl_offset_time,
                                     lidar_meas.is_lidar_end ? 1 : 0, &n_taken, nullptr, 0, nullptr, nullptr));
    check(h, flb_state_download(h, &x, nullptr, nullptr));
    from_abi(x, state_inout);
    lidar_meas.last_update_time = pcl_end_time;                                                   // :642
    lidar_meas.lidar_scan_index_now = lidar_meas.is_lidar_end ? 0 : lidar_meas.lidar_scan_index_now + n_taken;   // :638, :643-646
    return n_taken;
}

}  // namespace flb
