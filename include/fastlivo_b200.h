/* fastlivo_b200 -- C ABI of the H100-native FAST-LIVO measurement/ESKF hot path.
 *
 * Plain C, plain pointers and sizes, no torch / Eigen / PCL types.  Every entry
 * point cites the reference code it replaces (paths relative to the reference
 * tree hku-mars/FAST-LIVO @ dcebf84).  INTEGRATION.md shows the bindings a
 * maintainer of the reference adds on its side.
 *
 * Conventions
 *   - all pointers are HOST pointers owned by the caller for the duration of
 *     the call only; the library copies.  The opaque handle owns all device
 *     memory, one CUDA stream and (optionally) one NCCL communicator.
 *   - matrices are row-major doubles; rotations are 3x3 row-major.
 *   - every function returns an int status: FLB_OK (0) or a negative FLB_ERR_*;
 *     nothing throws or aborts.  flb_last_error() gives a message.
 *   - a handle is single-caller; distinct handles are independent.
 *   - there is NO CPU fallback: without a CUDA device flb_create() fails with
 *     FLB_ERR_NO_DEVICE.
 */
#ifndef FASTLIVO_B200_H
#define FASTLIVO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FLB_OK             0
#define FLB_ERR_INVALID   -1  /* bad argument */
#define FLB_ERR_CUDA      -2  /* CUDA runtime error (see flb_last_error) */
#define FLB_ERR_NO_DEVICE -3  /* no usable CUDA device: the product path refuses to run */
#define FLB_ERR_STATE     -4  /* call order: map / scan / image / patches not uploaded */
#define FLB_ERR_NUMERIC   -5  /* singular normal matrix or non-finite state */
#define FLB_ERR_COMM      -6  /* NCCL not available / communicator error */
#define FLB_ERR_TIMEOUT   -7  /* device-side barrier watchdog tripped */

#define FLB_ABI_VERSION 1

typedef struct flb_handle flb_handle;

typedef struct flb_config {
    int    device;           /* CUDA ordinal */
    double cell_size;        /* uniform-grid cell for the device map; <=0 -> 0.6 (2 x filter_size_map) */
    double knn_max_d2;       /* neighbours farther than this never select a point: 5.0,
                                src/laserMapping.cpp:1549; <=0 -> 5.0 */
    double plane_threshold;  /* esti_plane threshold 0.1f, src/laserMapping.cpp:1571; <=0 -> 0.1 */
    int    persistent;       /* 1: one persistent kernel per update (default); 0: kernel-per-pass */
    int    reserved[7];
} flb_config;

/* 18-DoF state == StatesGroup, include/common_lib.h:296-381.
 * cov order [rot, pos, vel, bias_g, bias_a, gravity]. */
typedef struct flb_state18 {
    double rot[9];
    double pos[3];
    double vel[3];
    double bg[3];
    double ba[3];
    double grav[3];
    double cov[324];
} flb_state18;

/* ---- lifetime ------------------------------------------------------------------ */
int         flb_abi_version(void);
int         flb_create(const flb_config* cfg, flb_handle** out);
int         flb_destroy(flb_handle* h);
const char* flb_last_error(const flb_handle* h);   /* h may be NULL: last create error */
/* Run all subsequent work of this handle on an existing CUDA stream (cudaStream_t
 * passed as void*), e.g. torch's current stream.  NULL restores the handle's own. */
int         flb_set_stream(flb_handle* h, void* cuda_stream);
int         flb_synchronize(flb_handle* h);
/* Optional page-locked host buffers.  Upload calls detect page-locked sources (these, cudaHostAlloc or
 * cudaHostRegister memory) and let the copy engine read them directly instead of staging through the
 * handle's own pinned area; such a buffer must then stay unmodified until the next blocking call on the
 * handle (flb_*_update, flb_*_pass, flb_synchronize; for a pipelined frame: the flb_state_download_wait that
 * collects THAT frame's result) returns.  Pageable buffers keep the plain contract: free to reuse as soon as the
 * upload call returns.
 * Uploads never wait for the update that is running: scan, image and patch list each have two device sets, an
 * upload fills the idle one on its own stream and the handle switches sets for everything enqueued afterwards. */
int         flb_host_alloc(flb_handle* h, size_t bytes, void** out);
int         flb_host_free(flb_handle* h, void* p);

/* ---- map: the query half of ikd-Tree -------------------------------------------
 * Replaces KD_TREE::Build (include/ikd-Tree/ikd_Tree.cpp:337-348, called at
 * src/laserMapping.cpp:1411-1419): uploads M map points (float xyz, stride in
 * floats: 3 for packed, 4 for float4, 12 for pcl::PointXYZINormal) and builds the
 * device-resident sorted uniform grid the kNN kernel walks. */
int flb_map_upload(flb_handle* h, const float* xyz, int M, int stride_floats);

/* Device-resident map maintenance (SURVEY.md section 8 row f1): the map follows the reference's ikd-Tree
 * without a per-frame re-upload.
 *   flb_map_add_points  == ikdtree.Add_Points(PointToAdd, true) with downsample_size = filter_size_map
 *                          (map_incremental, src/laserMapping.cpp:692-706; ikd_Tree.cpp:382-457): per
 *                          downsample voxel touched by a new point, only the point closest to the voxel
 *                          centre survives (existing or new); untouched voxels are left alone.
 *   flb_map_delete_boxes == ikdtree.Delete_Point_Boxes(cub_needrm) (lasermap_fov_segment,
 *                          src/laserMapping.cpp:363-421; ikd_Tree.cpp:501-521): boxes nb x 6 floats
 *                          (min xyz, max xyz), half-open containment min <= p < max.
 * After either call map indices (flb_knn / flb_lio_export nn_idx) refer to the order flb_map_download
 * returns.  |coordinate / downsample_size| must stay below 2^20. */
int flb_map_add_points(flb_handle* h, const float* world_xyz, int n, int stride_floats, float downsample_size);
/* map_incremental (src/laserMapping.cpp:692-706) from what is on the device: every point of the scan most recently
 * uploaded (flb_scan_upload / flb_frame_enqueue / flb_batch_set_frame), in the caller's original order, transformed by
 * pointBodyToWorld (:272-286; double math, float store) at pose (R, p) with prm->R_LI / prm->t_LI, then
 * Add_Points(..., downsample_size) exactly as flb_map_add_points: the same map bytes, order and grid as that call on the
 * host-transformed scan.  R == p == NULL: the device state x as it stands in stream order (call it right after the LIO
 * update for the reference's order).  IKFoM callers pass R = rot, p = pos and offset_R_L_I / offset_T_L_I as the
 * extrinsic (RGBpointBodyToWorld under USE_IKFOM).  Blocking, like flb_map_add_points.  Single GPU.
 * Errors, all leaving the map unchanged: FLB_ERR_STATE without a map, without a scan, after flb_voxel_grid used the scan
 * slot as scratch, without a device state for R == NULL, and after flb_comm_init / flb_p2p_attach (each rank holds only
 * its shard of the scan); FLB_ERR_INVALID for prm == NULL, exactly one of R / p NULL, downsample_size <= 0, and a
 * transformed point that is not finite or beyond flb_map_add_points' limits. */
struct flb_lio_params;
int flb_map_add_scan(flb_handle* h, const struct flb_lio_params* prm, const double R[9], const double p[3], float downsample_size);
int flb_map_delete_boxes(flb_handle* h, const float* boxes, int nb);
/* lasermap_fov_segment (src/laserMapping.cpp:363-421) + ikdtree.Delete_Point_Boxes(cub_needrm) in one call.  The local-
 * map cube (LocalMap_Points, Localmap_Initialized: :361-362) lives on the device in the handle and survives map uploads.
 *   cube_len = cube_side_length (:1118), det_range = DET_RANGE (:83, 300 in the reference), mov_threshold =
 *   MOV_THRESHOLD (:90, 1.5).  pos = pos_LiD (:368-373): NULL = state.pos_end of the device state x as it stands in
 *   stream order (after flb_imu_undistort that is the propagated prior, as at :1395); IKFoM callers pass pos_lid.
 * The cube steps exactly as the reference's (float vertices, double pose; the first call after flb_create or
 * flb_map_fov_reset only places the cube: *n_boxes = 0).  The points inside the boxes (half-open, as
 * flb_map_delete_boxes) are removed from the live sorted map without rebuilding it: survivors keep their order, the grid
 * box is kept.  When no point is inside, the map, its grid and its download bytes are unchanged.  Map indices still
 * refer to flb_map_download's array.  Blocking (one small read).  Runs before any map exists (M = 0: the cube moves,
 * nothing is deleted).  Outputs (each may be NULL): *n_boxes (0..3) = cub_needrm.size(), boxes[18] = the boxes
 * (min xyz, max xyz; unused slots all zero), local_box[6] = the cube after the call (min xyz, max xyz), *n_deleted =
 * kdtree_delete_counter (:417).  Bitwise the same on every rank, so multi-GPU handles may call it too.
 *   FLB_ERR_INVALID: prm NULL, or cube_len / det_range / mov_threshold not finite or not > 0.
 *   FLB_ERR_STATE: pos NULL without a device state; boxes that hold every map point (map and cube unchanged).
 * flb_map_fov_reset: Localmap_Initialized = false. */
typedef struct flb_fov_params {
    double cube_len;       /* cube_side_length (src/laserMapping.cpp:1118) */
    float det_range;       /* DET_RANGE (:83) */
    float mov_threshold;   /* MOV_THRESHOLD (:90) */
} flb_fov_params;
int flb_map_fov_segment(flb_handle* h, const flb_fov_params* prm, const double pos[3], int* n_boxes, float boxes[18],
                        float local_box[6], int* n_deleted);
int flb_map_fov_reset(flb_handle* h);
int flb_map_size(const flb_handle* h);
int flb_map_download(flb_handle* h, float* xyz, int capacity_points, int* M_out);
/* flb_map_grid_info: the kNN cell geometry in use.  The map's cells are indexed by a dense table over the map's box
 * (plus a margin); where that would need more than 2^25 cells of flb_config.cell_size the cell is enlarged until it
 * fits (cell_size reports the enlarged cell).  sparse = 1: a sparse hash index of the occupied cells at the configured
 * cell (flb_debug_set_map_index).  cells: dense table cells, or occupied cells when sparse; index_bytes: device bytes of
 * the index.  Any output pointer may be NULL. */
int flb_map_grid_info(flb_handle* h, double* cell_size, int* sparse, int64_t* cells, int64_t* index_bytes);

/* ---- IMU forward propagation + backward undistortion (SURVEY.md section 8 row f3) ----------------------
 * Replaces ImuProcess::UndistortPcl from src/IMU_Processing.cpp:655 on (called by Process2, :811-849, at
 * src/laserMapping.cpp:1353): per IMU interval the mid-point propagation of attitude / velocity / position
 * and of the 18x18 covariance (cov = F_x cov F_x^T + cov_w, :699-720), the frame-end prediction (:743-758),
 * and the per-point backward motion compensation to the frame end (:778-808).  The LidarMeasureGroup
 * bookkeeping of :613-652 (which points belong to this update, pcl_beg_time, pcl_end_time) stays with the
 * caller.
 *   The device state (flb_state_upload) is state_inout: it is propagated in place (rot_end, pos_end, vel_end,
 *   cov; biases and gravity unchanged), so x_prop and P are on the device for the update that follows
 *   (flb_state_set_prior_enqueue makes it state_propagat, src/laserMapping.cpp:1354).
 *   v_imu: last_imu_ followed by meas.imu (:617-618), times non-decreasing.  carry: the ImuProcess members
 *   that survive from frame to frame (last_lidar_end_time_, acc_s_last, angvel_last), in/out.
 *   pts: n_points lidar-frame points in time order, stride_floats floats apart, x,y,z at [0..2] and the time
 *   offset in ms (PointType::curvature) at [offset_index] (pcl::PointXYZINormal: stride 12, offset_index 9).
 *   out_xyz: n_points x 3 compensated coordinates, or NULL: the compensated points stay on the device only (no copy
 *   back), for flb_scan_from_undistorted / flb_world_cloud; everything else is the same as with a buffer.
 *   poses_out (optional, capacity n_imu entries of 22 doubles: offset_time, acc, gyr, vel, pos, rot) receives
 *   IMUpose; n_poses_out its length. */
typedef struct flb_imu_sample { double t; double gyr[3]; double acc[3]; } flb_imu_sample;   /* sensor_msgs::Imu */
typedef struct flb_imu_params {
    double cov_gyr[3], cov_acc[3], cov_bias_gyr[3], cov_bias_acc[3];   /* src/IMU_Processing.cpp:15-20, :58-83 */
    double G_m_s2, mean_acc_norm;                                      /* acc * G_m_s2 / mean_acc.norm(), :688 */
    double R_LI[9], t_LI[3];                                           /* Lid_rot_to_IMU, Lid_offset_to_IMU */
} flb_imu_params;
typedef struct flb_imu_carry { double last_lidar_end_time; double acc_s_last[3]; double angvel_last[3]; } flb_imu_carry;
int flb_imu_undistort(flb_handle* h, const flb_imu_params* prm, flb_imu_carry* carry, const flb_imu_sample* v_imu, int n_imu,
                      double pcl_beg_time, double pcl_end_time, const float* pts, int stride_floats, int offset_index,
                      int n_points, float* out_xyz, double* poses_out, int* n_poses_out);

/* ---- the driver's LiDAR message on the device ------------------------------------------------------------
 * Preprocess::process (src/preprocess.cpp:43-70) with feature_extract_enable = 0 (every shipped config), the time sort
 * of sync_packages (src/laserMapping.cpp:551) and the window at the top of UndistortPcl
 * (src/IMU_Processing.cpp:621-646), from the raw records of one driver message.  Each handler's arithmetic and quirks
 * are kept bit for bit:
 *   FLB_LIDAR_LIVOX (avia_handler, :138-160; Avia, Mid360): the loop starts at record 1, so record 0 is never kept
 *     (:138).  A record is valid when line < n_scans and (tag & 0x30) is 0x10 or 0x00 (:140); valid_num counts the valid
 *     records and a record is taken when valid_num % point_filter_num == 0 (:142-143).  curvature = offset_time /
 *     float(1000000) (:149).  It is kept when some |coordinate - pl_full[i-1]'s| > 1e-7 and x*x + y*y + z*z (float) >
 *     blind * blind (:151-154); pl_full[i-1] holds record i-1 only when that record was taken itself, otherwise the
 *     (0, 0, 0) of pl_full.resize (:83), so a repeated point that follows a record which was not taken is compared with
 *     zero and kept.
 *   FLB_LIDAR_OUSTER (oust64_handler, :233-252): i % point_filter_num == 0 (:235); skipped when the float sum of squares,
 *     widened to double, is < blind * blind (:237-239); curvature = t * 1.e-6f (:250).
 *   FLB_LIDAR_VELODYNE (velodyne_handler, :376-428): only clouds with per-point times, i.e. the last record's time > 0
 *     (given_offset_time, :279).  curvature = time * 1.e-3f (:387); i % point_filter_num == 0 (:421); kept when the
 *     float sum of squares > blind * blind (:423).  Without times the reference derives them from the yaw angle with a
 *     sequential per-ring state (:389-419); that stays with the host and the call returns FLB_ERR_INVALID.
 *   FLB_LIDAR_XT32 (xt32_handler, :441-461): curvature = float((timestamp - timestamp[0]) * 1000.f), computed in double
 *     (:454); i % point_filter_num == 0 (:456); kept when the float sum of squares > blind, not its square (:458).
 * The kept points are then sorted by curvature (time_list).  std::sort leaves the order of equal times unspecified; here
 * it is the stable order (equal times keep record order).  Ties are real: the lines of a Livox fire together.
 * The cloud stays on the device as {x, y, z, curvature}; intensity is not kept (no device cloud carries it).
 *
 * flb_lidar_upload: records = n_records records of fmt->point_step bytes (CustomMsg::points, or PointCloud2::data).
 * *n_points = pl_surf.size(), *last_offset_ms = points.back().curvature after the sort (0 for an empty cloud); either
 * may be NULL.  The records fill the idle one of two device sets on the copy stream and never wait for an update that is
 * running; a page-locked source (flb_host_alloc) is read in place, a pageable one is free on return.  Blocking (one
 * 16-byte read, a second one when the times had to be sorted).  n_records 0 or 1, or everything filtered, gives an empty
 * cloud (sync_packages skips points.size() <= 1 itself, src/laserMapping.cpp:538).  A successful call resets the cursor
 * (lidar_scan_index_now) to 0.  On any error the previous cloud and its cursor stay current and unchanged:
 *   FLB_ERR_INVALID: fmt NULL, records NULL with n_records > 0, n_records < 0, an unknown kind, point_filter_num < 1,
 *   n_scans < 1, blind not finite, a field that does not fit in point_step or is not aligned to its type, a Velodyne
 *   cloud without times, a kept coordinate or time that is not finite. */
#define FLB_LIDAR_LIVOX    1
#define FLB_LIDAR_VELODYNE 2
#define FLB_LIDAR_OUSTER   3
#define FLB_LIDAR_XT32     4
typedef struct flb_lidar_format {
    int    kind;               /* FLB_LIDAR_* (LID_TYPE, include/preprocess.h:13) */
    int    point_step;         /* bytes per record: sizeof(livox_ros_driver::CustomPoint) (20) or PointCloud2::point_step */
    int    off_x, off_y, off_z;/* float32 fields; Livox: 4, 8, 12 */
    int    off_time;           /* Livox offset_time (u32, 0); Ouster t (u32); Velodyne time (f32); XT32 timestamp (f64) */
    int    off_tag, off_line;  /* Livox only (u8 at 17 and 18); ignored otherwise */
    int    n_scans;            /* N_SCANS (scan_line); read by the Livox handler only */
    int    point_filter_num;   /* >= 1 */
    double blind;              /* Preprocess::blind, used per handler as above */
} flb_lidar_format;
int flb_lidar_upload(flb_handle* h, const flb_lidar_format* fmt, const void* records, int n_records, int* n_points,
                     float* last_offset_ms);
/* The current cloud, x, y, z, curvature per point, for tests and for a node that publishes the raw cloud.  *n_out (may
 * be NULL) = its size; xyzt may be NULL.  Blocking.  FLB_ERR_STATE without a cloud, FLB_ERR_INVALID when
 * capacity_points is below its size. */
int flb_lidar_download(flb_handle* h, float* xyzt, int capacity_points, int* n_out);
/* UndistortPcl from :621 on with the device cloud as lidar_meas.lidar.  The window (:634-639): the points from the
 * handle's cursor on while (double)curvature <= pcl_offset_time, read in place; *n_taken (may be NULL) = pcl_out.size().
 * Then everything flb_imu_undistort does on those points, with the same outputs (out_xyz may be NULL; its capacity is
 * capacity_points) and the same effect on flb_scan_from_undistorted / flb_world_cloud(FLB_CLOUD_UNDISTORTED).  The cursor
 * advances by *n_taken, or returns to 0 when is_lidar_end (:643-646).  pcl_offset_time is the caller's (:631-633): 0.0
 * for a camera update, (pcl_end_time - lidar_beg_time) * 1000 at the scan end.  That product can round below
 * points.back().curvature; the last points are then left out, as in the reference, and dropped by the cursor's reset.
 *   FLB_ERR_STATE: no cloud; no device state.  FLB_ERR_INVALID: as flb_imu_undistort, a NaN pcl_offset_time, or
 *   capacity_points < *n_taken with out_xyz given.  On an error the cursor does not move. */
int flb_imu_undistort_lidar(flb_handle* h, const flb_imu_params* prm, flb_imu_carry* carry, const flb_imu_sample* v_imu,
                            int n_imu, double pcl_beg_time, double pcl_end_time, double pcl_offset_time, int is_lidar_end,
                            int* n_taken, float* out_xyz, int capacity_points, double* poses_out, int* n_poses_out);

/* ---- a Velodyne message in any field layout, with or without per-point times ------------------------------
 * velodyne_handler (src/preprocess.cpp:259-297, and its non-feature branch :376-428) on the PointCloud2 data of any
 * Velodyne driver: XYZIRT, XYZIR without a time field, a time of 0 everywhere, and float fields at any byte offset
 * (a packed 22-byte record puts the time at 18).  The result goes where flb_lidar_upload's goes, so flb_lidar_download
 * and flb_imu_undistort_lidar work on it unchanged.
 *   With times (the last record's time > 0, given_offset_time, :279): exactly flb_lidar_upload(FLB_LIDAR_VELODYNE) on
 *     the same records wherever that call accepts the layout; the ring is not read.  *yaw_times = 0.
 *   Without times: the times come from the yaw angle, per ring (layer = ring, :391), in record order:
 *     yaw = atan2(y, x) * 57.2957 (:392).  The reference's arguments are floats, so its atan2 is the float overload of
 *       the libm it links; here the yaw is defined as (float)atan2((double)y, (double)x), widened to double before the
 *       multiply.  The two agree except near float rounding midpoints; DESIGN §2 gives the effect (a few 1e-6 ms).
 *     The first record of a ring sets yaw_fp = yaw and time_last = 0 and is never kept (the `continue` of :403), whatever
 *       i % point_filter_num is; it still uses up its index i.
 *     Every later record: base = float((yaw_fp - yaw) / omega_l) when yaw <= yaw_fp, else float((yaw_fp - yaw + 360.0)
 *       / omega_l), with omega_l = 0.361 * 10 (:272, :406-413); t = float(base + 360.0 / omega_l) when base < time_last,
 *       else base (:415); time_last = t.  A NaN yaw (a no-return record) gives a NaN time_last, so the next record of
 *       the ring cannot wrap.  *yaw_times = 1.
 *     A record is kept when i % point_filter_num == 0 and the float x*x + y*y + z*z > blind * blind (:421-423).
 *   The kept points are then sorted by time, stably, as by flb_lidar_upload.  The rings are walked as one parallel scan
 *   (DESIGN §4.9), not a loop.  n_records 0 gives an empty cloud and *yaw_times = 0.
 * fmt: off_x, off_y, off_z float32 and off_ring uint16 at any byte offset within point_step; off_time float32 seconds at
 * any offset, or -1 for a cloud without a time field (the reference then reads 0: the yaw route).  n_points,
 * last_offset_ms and yaw_times may be NULL.  Everything else is flb_lidar_upload's: the idle set on the copy stream, a
 * page-locked source read in place, the swap on success only, the cursor reset to 0.  On any error the previous cloud
 * and its cursor stay current and unchanged:
 *   FLB_ERR_INVALID: fmt NULL, records NULL with n_records > 0, n_records < 0, point_filter_num < 1, n_scans < 1, blind
 *   not finite, a field that does not fit in point_step, a ring >= n_scans on the yaw route (the reference indexes past
 *   its per-ring vectors there; the message names the ring and the record), a kept coordinate or time that is not
 *   finite (a ring whose first record has no return makes every time of that ring NaN). */
typedef struct flb_velodyne_format {
    int    point_step;         /* PointCloud2::point_step */
    int    off_x, off_y, off_z;/* float32, any alignment */
    int    off_time;           /* float32 seconds, any alignment; -1: no time field */
    int    off_ring;           /* uint16, any alignment */
    int    n_scans;            /* N_SCANS (scan_line) */
    int    point_filter_num;   /* >= 1 */
    double blind;              /* Preprocess::blind */
} flb_velodyne_format;
int flb_lidar_upload_velodyne(flb_handle* h, const flb_velodyne_format* fmt, const void* records, int n_records, int* n_points,
                              float* last_offset_ms, int* yaw_times);

/* ---- surface features (feature_extract_enable: 1) ------------------------------------------------------------------
 * The feature branches of Preprocess: avia_handler :94-135, oust64_handler :174-227 and velodyne_handler :299-373,
 * each bucketing its points by line and running give_feature (:466-775) per line.  The result is pl_surf (the only
 * cloud FAST-LIVO reads, :43-70), sorted by time stably on pl_surf's line-major order, and it goes exactly where
 * flb_lidar_upload's goes: the idle set on the copy stream, a page-locked source read in place, the swap on success
 * only, the cursor reset to 0; on any error the previous cloud and cursor stay current and unchanged.  So
 * flb_lidar_download, flb_imu_undistort_lidar, flb_scan_from_undistorted and flb_world_cloud work on it unchanged.
 *   dis_b: Preprocess::disB.  The reference's constructor assigns disA twice (:12-13) and never disB, so its value there
 *     is whatever the heap held; the caller states it.  The other constants are the constructor's (group_size 8,
 *     disA 0.1, p2l_ratio 225, ...), and its four cos() thresholds are computed with the host's std::cos.
 *   point_filter_num: the chunk length of the surface output (:728-774), not an input decimation.
 *   Per handler: Livox (FLB_LIDAR_LIVOX): from record 1, a record is dropped when |dx|, |dy| or |dz| against the raw
 *     previous record is below 1e-8, x*x + y*y < blind, line > n_scans or (tag & 0x30) != 0x10; line == n_scans is
 *     dropped too (its buffer is never processed); lines of <= 5 points are skipped; range = x*x + y*y.  Ouster
 *     (FLB_LIDAR_OUSTER): off_line names the u8 ring (26 in ouster_ros::Point); the float x*x + y*y + z*z < blind *
 *     blind drops a point, and ring < n_scans is required; an empty ring is skipped (the reference indexes types[-1]).
 *     Velodyne: no blind filter at input; a ring >= n_scans is dropped; on the yaw route (no per-point times, as
 *     flb_lidar_upload_velodyne) each ring's first record is not kept; lines of < 2 points are skipped.
 *   Defined where the reference is not (DESIGN §2): a line's last dista is 0.0; a plane step's write past the line's
 *   end is dropped; a line entirely within blind yields nothing; Eigen's reductions are left to right.
 *   FLB_ERR_INVALID: fmt NULL, records NULL with n_records > 0, n_records < 0, dis_b not finite, point_filter_num < 1,
 *   n_scans outside 1..128 (pl_buff[128]), blind not finite, a field that does not fit or is misaligned, a point of
 *   pl_surf or its time that is not finite; flb_lidar_upload_features with FLB_LIDAR_VELODYNE or FLB_LIDAR_XT32 (the
 *   XT32 has no feature branch, :432-464: flb_lidar_upload serves it with either setting). */
int flb_lidar_upload_features(flb_handle* h, const flb_lidar_format* fmt, double dis_b, const void* records, int n_records,
                              int* n_points, float* last_offset_ms);
int flb_lidar_upload_velodyne_features(flb_handle* h, const flb_velodyne_format* fmt, double dis_b, const void* records,
                                       int n_records, int* n_points, float* last_offset_ms, int* yaw_times);

/* ---- scan ------------------------------------------------------------------------
 * feats_down_body (src/laserMapping.cpp:1398-1399): N already-downsampled points in
 * the LiDAR body frame. */
int flb_scan_upload(flb_handle* h, const float* body_xyz, int N, int stride_floats);
/* downSizeFilterSurf.setInputCloud(feats_undistort); downSizeFilterSurf.filter(*feats_down_body)
 * (src/laserMapping.cpp:1398-1399) followed by flb_scan_upload, with the cloud never leaving the device.  The source is
 * the output of the last successful flb_imu_undistort (out_xyz may be NULL there), in its point order.  The scan is
 * then exactly what flb_scan_upload(flb_voxel_grid(out_xyz, leaf)) gives: the same points, order and per-point state,
 * so every call that reads the scan works unchanged.  *n_out (may be NULL) = feats_down_size.  Blocking (one 96-byte
 * read).  On any error the previous scan stays current and unchanged.
 *   FLB_ERR_STATE: no flb_imu_undistort output (none yet, or the last call failed); after flb_comm_init /
 *   flb_p2p_attach (each rank holds only its shard of the scan).
 *   FLB_ERR_INVALID: !(leaf > 0), a non-finite point, a leaf too small for the cloud's extent (PCL's index-overflow
 *   case, as in flb_voxel_grid).  Zero points give an empty scan, as flb_scan_upload(h, ..., 0, ...) does. */
int flb_scan_from_undistorted(flb_handle* h, float leaf, int* n_out);
/* ikdtree.Build(feats_down_body->points) of the first frame (src/laserMapping.cpp:1411-1419) from the scan on the
 * device: replaces the map with the current scan's points in the caller's order, byte-identical to flb_map_upload of
 * the same points.  Blocking.  FLB_ERR_STATE: no scan (or flb_voxel_grid used its slot as scratch), and after
 * flb_comm_init / flb_p2p_attach; FLB_ERR_INVALID: an empty scan (as flb_map_upload refuses M < 1). */
int flb_map_upload_scan(flb_handle* h);

/* Exact 5-NN of nq WORLD-frame float queries, KD_TREE::Nearest_Search semantics
 * (include/ikd-Tree/ikd_Tree.cpp:350-380, 843-986, 1291-1295): float32
 * (dx*dx+dy*dy)+dz*dz, ascending order.  idx: nq x 5 indices into the uploaded map,
 * d2: nq x 5.  A query whose 5th neighbour is farther than knn_max_d2 gets
 * idx = -1 / d2 = +inf for the entries beyond knn_max_d2 (the reference rejects such
 * points at src/laserMapping.cpp:1549, so the bounded search is behaviourally identical). */
int flb_knn(flb_handle* h, const float* q_world, int nq, int* idx, float* d2);

/* ---- LIO -------------------------------------------------------------------------- */
typedef struct flb_lio_params {
    double R_LI[9];          /* Lidar_rot_to_IMU     src/laserMapping.cpp:104-105 */
    double t_LI[3];          /* Lidar_offset_to_IMU */
    double laser_point_cov;  /* LASER_POINT_COV      src/laserMapping.cpp:1109 */
    int    max_iteration;    /* NUM_MAX_ITERATIONS: the loop runs iterCount = -1..T-1 (:1506) */
    double conv_rot_deg;     /* 0.01  (:1688); 0 disables the convergence test */
    double conv_pos_cm;      /* 0.015 (:1688) */
} flb_lio_params;

typedef struct flb_lio_report {
    int     passes;
    int     knn_passes;
    int     n_eff_last;      /* effct_feat_num */
    double  res_mean_last;   /* src/laserMapping.cpp:1602 */
    int64_t rows_total;      /* point-to-plane rows assembled over all passes */
    int     converged_last;
    int     status;          /* FLB_OK or FLB_ERR_NUMERIC / FLB_ERR_TIMEOUT raised on device */
} flb_lio_report;

/* Packed normal equations of one pass.  width = 6: live layout [rot, pos]
 * (Hsub, src/laserMapping.cpp:1608-1629); width = 12: IKFoM layout
 * [pos, rot, offset_R_L_I, offset_T_L_I] (h_x, src/laserMapping.cpp:1059-1089). */
typedef struct flb_normal_eq {
    int    width;
    int    n_eff;
    double sum_abs_res;      /* total_residual, :1597 */
    double HTH[144];         /* width x width row-major in the leading entries */
    double HTh[12];
} flb_normal_eq;

/* One pass of the matching loop body src/laserMapping.cpp:1508-1630 at pose (R,p):
 * pointBodyToWorld (:272-286), [kNN (:1543) + esti_plane (common_lib.h:448-493) when
 * rematch], residual + gates (:1573-1584), compaction (:1588-1602), rows (:1608-1629),
 * H^T H / H^T z (:1664-1666).  Also the measurement half of h_share_model (:960-1094)
 * when width = 12 (rematch == ekfom_data.converge, :994). */
int flb_lio_pass(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3],
                 int rematch, int width, flb_normal_eq* out);

/* Per-point / per-row products of the LAST flb_lio_pass (any pointer may be NULL):
 *   world_xyz N x 3 float (feats_down_world); nn_idx N x 5 (Nearest_Points as map
 *   indices, -1 = none); nn_d2 N x 5; pabcd N x 4 (cached plane); pd2 N;
 *   selected N (point_selected_surf && res_last<=2, i.e. the row mask);
 *   rows n x width doubles row-major (Hsub or h_x); meas n (meas_vec / h);
 *   sel_idx n (scan index of each compacted row, the order of laserCloudOri). */
int flb_lio_export(flb_handle* h, float* world_xyz, int* nn_idx, float* nn_d2, float* pabcd, float* pd2,
                   uint8_t* selected, double* rows, double* meas, int* sel_idx, int* n_rows);

/* The whole iterated update src/laserMapping.cpp:1504-1733 (control flow: SURVEY.md
 * Appendix A), run on the device without a host round trip per pass.  x: in = state
 * before the update (normally == x_prop), out = updated state and covariance. */
int flb_lio_update(flb_handle* h, const flb_lio_params* prm, flb_state18* x, const flb_state18* x_prop,
                   flb_lio_report* rep);

/* ---- IKFoM-typed LIO update (the `#define USE_IKFOM` estimator) -------------------------
 * state_ikfom (include/use-ikfom.hpp:12-21): pos, rot, offset_R_L_I, offset_T_L_I, vel, bg, ba, grav(S2,
 * |g| = 9.8090).  Quaternions are (x, y, z, w) like Eigen's coeffs(); P is the 23x23 covariance, row-major,
 * in the sub-manifold order above (DOF 23). */
typedef struct flb_state_ikfom {
    double pos[3];
    double rot[4];
    double offset_R_L_I[4];
    double offset_T_L_I[3];
    double vel[3], bg[3], ba[3];
    double grav[3];
    double P[529];
} flb_state_ikfom;

typedef struct flb_ikfom_params {
    double laser_point_cov;  /* R in kf.update_iterated_dyn_share_modified(LASER_POINT_COV, ...), laserMapping.cpp:1484 */
    int    max_iteration;    /* maximum_iter of kf.init_dyn_share(..., NUM_MAX_ITERATIONS, epsi), :1235 */
    double limit[23];        /* epsi (0.001 each, :1233-1234) */
} flb_ikfom_params;

typedef struct flb_ikfom_report {
    int     passes, knn_passes, n_eff_last, converged_last;
    double  res_mean_last;
    int64_t rows_total;
    int     status;
} flb_ikfom_report;

/* esekfom::esekf<state_ikfom,12,input_ikfom>::update_iterated_dyn_share_modified
 * (include/IKFoM_toolkit/esekfom/esekfom.hpp:1619-1928) with h_dyn_share = h_share_model
 * (src/laserMapping.cpp:960-1094), i.e. the block src/laserMapping.cpp:1482-1494, in one device launch:
 * per pass the 12-column rows [n, A, B, C] and h_x^T h_x / h_x^T h, the SO3/S2 re-projection of P, the
 * information-form gain, x [+] dx, the per-component convergence test and, on the last pass, the
 * covariance update.  x: in = x_ (== the propagated state) and P_; out = updated.  Needs the map and the
 * scan uploaded; single GPU, persistent mode. */
int flb_lio_update_ikfom(flb_handle* h, const flb_ikfom_params* prm, flb_state_ikfom* x, flb_ikfom_report* rep);

/* ---- VIO --------------------------------------------------------------------------- */
typedef struct flb_camera {
    int    width, height;
    double fx, fy, cx, cy;   /* vikit PinholeCamera (config/camera_pinhole.yaml) */
    double d[5];             /* radtan; enabled iff |d0| > 1e-7 */
} flb_camera;

typedef struct flb_vio_params {
    double Rcl[9], Pcl[3];   /* camera<-lidar extrinsic, src/laserMapping.cpp:1206 (set_camera2lidar) */
    double R_LI[9], t_LI[3]; /* LidarSelector::set_extrinsic, src/lidar_selection.cpp:35-39 */
    double img_point_cov;    /* src/lidar_selection.cpp:873 */
    int    max_iteration;    /* LidarSelector::NUM_MAX_ITERATIONS */
    float  conv_rot_deg;     /* 0.001f (:883); 0 disables */
    float  conv_pos_cm;      /* 0.001f */
    int    force_all_passes; /* benchmark mode: fixed pass count (no error test, no EKF_end) */
} flb_vio_params;

typedef struct flb_vio_report {
    int     passes[3];       /* index = pyramid level */
    float   last_error[3];
    int64_t rows_total;      /* photometric rows (pixels) assembled over all passes */
    int     skipped_last;    /* patches dropped by the bounds / depth guard in the last pass */
    int     cov_updated;
    int     status;
} flb_vio_report;

typedef struct flb_vio_eq {
    double  HTH[36];
    double  HTz[6];
    float   error;           /* mean squared photometric error, :857 */
    int64_t n_meas;
    int     skipped;
} flb_vio_eq;

/* cv::Mat img of LidarSelector::detect (src/lidar_selection.cpp:1027-1037): gray uint8.  The image set it makes current
 * holds no colour frame (flb_colorize / flb_colorize_cloud with bgr == NULL refuse it). */
int flb_image_upload(flb_handle* h, const uint8_t* gray, int width, int height, int stride_bytes);
/* The first lines of LidarSelector::detect (src/lidar_selection.cpp:1029-1037) on the device: the camera frame as the
 * driver delivers it (getImageFromMsg(..., "bgr8"), src/laserMapping.cpp:490-493), halved by cv::resize(0.5,
 * INTER_LINEAR) when its size differs from the camera's, kept as img_rgb and converted by cv::cvtColor(CV_BGR2GRAY).
 * The current image set then holds the camera-size gray image, byte-identical to flb_image_upload of OpenCV's
 * cvtColor(resize(bgr)), so every reader of the image works unchanged, and the camera-size BGR frame, which
 * flb_colorize / flb_colorize_cloud read with bgr == NULL (publish_frame_world_rgb, :727-744).
 *   (width, height) = the camera's (no resize), or exactly twice it (each output channel is OpenCV's 2x2 area mean
 *   (a + b + c + d + 2) >> 2, what cv::resize does for an even-sized frame at scale 0.5).  stride_bytes >= 3 * width.
 *   gray_rule: the fixed-point cvtColor of the OpenCV the caller links (the reference asks for OpenCV >= 3.2).
 * The same rules as flb_image_upload: the frame fills the idle one of two device sets on the copy stream and never
 * waits for the update that is running; a page-locked source is read in place (keep it until the next synchronise), a
 * pageable one is free on return.  Needs flb_camera_set (FLB_ERR_STATE).  FLB_ERR_INVALID: bgr NULL, any other size,
 * stride_bytes < 3 * width, an unknown gray_rule.  On any error the previous image set stays current and unchanged.
 * Odd-sized frames (OpenCV's general bilinear path) and encodings other than BGR8 are not handled. */
#define FLB_GRAY_CV4 0   /* (3735 B + 19235 G + 9798 R + 2^14) >> 15: OpenCV 4.x */
#define FLB_GRAY_CV3 1   /* (1868 B + 9617 G + 4899 R + 2^13) >> 14: OpenCV 3.x  */
int flb_image_upload_bgr(flb_handle* h, const uint8_t* bgr, int width, int height, int stride_bytes, int gray_rule);
/* The camera message as the driver delivers it (sensor_msgs::Image: data, width, height, step, encoding): what
 * flb_image_upload_bgr does with cv_bridge::toCvCopy(msg, "bgr8")->image (getImageFromMsg, src/laserMapping.cpp:
 * 490-493), with the colour conversion on the device, so the host neither converts nor demosaics the frame and the
 * upload carries the message's own bytes per pixel.  The current image set then holds the camera-size colour frame
 * (img_rgb) and its gray image exactly as after flb_image_upload_bgr, and every reader works unchanged.
 *   encoding: FLB_ENC_*.  Packed encodings are byte permutations to BGR (mono8 repeats its byte, the alpha byte is
 *   dropped).  Bayer encodings are cv_bridge's bilinear demosaic (the OpenCV code beside each).
 *   (width, height): the size rule of detect()'s cv::resize(Size(cols * 0.5, rows * 0.5), INTER_LINEAR):
 *     the camera's size: no resize;  exactly twice it: the 2x2 area mean of flb_image_upload_bgr;
 *     2W or 2W + 1 by 2H or 2H + 1 with an odd side: OpenCV 4's fixed-point linear resize, 11-bit weights.  That rule
 *     is defined for FLB_GRAY_CV4 only: OpenCV 3's rounding there depends on its SIMD path, so FLB_GRAY_CV3 refuses it.
 *   step_bytes >= width * the encoding's bytes per pixel.
 * FLB_ENC_BGR8 at the camera's size or twice it is flb_image_upload_bgr, byte for byte.  Copy semantics, streams and
 * FLB_ERR_STATE as flb_image_upload_bgr.  FLB_ERR_INVALID: data NULL, an unknown encoding or gray_rule, any other size,
 * step_bytes too small, FLB_GRAY_CV3 with an odd side.  On any error the previous image set stays current and
 * unchanged.
 * Not handled: 16-bit encodings, YUV 4:2:2 and sensor_msgs::CompressedImage (JPEG / PNG).  display_keypatch's circles
 * on img_cp are drawn on the device too (flb_keypatch_image); only its "N HZ" text stays on the host. */
#define FLB_ENC_BGR8        0
#define FLB_ENC_RGB8        1
#define FLB_ENC_MONO8       2
#define FLB_ENC_BGRA8       3
#define FLB_ENC_RGBA8       4
#define FLB_ENC_BAYER_RGGB8 5   /* cv_bridge: COLOR_BayerBG2BGR */
#define FLB_ENC_BAYER_BGGR8 6   /* COLOR_BayerRG2BGR */
#define FLB_ENC_BAYER_GBRG8 7   /* COLOR_BayerGR2BGR */
#define FLB_ENC_BAYER_GRBG8 8   /* COLOR_BayerGB2BGR */
int flb_image_upload_msg(flb_handle* h, const uint8_t* data, int width, int height, int step_bytes, int encoding, int gray_rule);
/* test / debugging aid (blocking): the current image set's gray (W*H) and colour (W*H*3) frames; either pointer may be
 * NULL.  capacity_pixels >= W*H when either is given.  *width / *height (may be NULL) = W, H.  FLB_ERR_STATE: no image
 * yet, or bgr != NULL for an image from flb_image_upload. */
int flb_image_download(flb_handle* h, uint8_t* gray, uint8_t* bgr, int capacity_pixels, int* width, int* height);
/* SubSparseMap (include/common_lib.h:263-292) flattened: pos Pn x 3 (Point::pos_),
 * patch Pn x 3 x 64 floats (warpAffine layout, src/lidar_selection.cpp:279-295),
 * search_level Pn. */
int flb_patches_upload(flb_handle* h, const double* pos, const float* patch, const int* search_level, int Pn);
int flb_camera_set(flb_handle* h, const flb_camera* cam);

/* ---- visual-map growth: candidate scoring (SURVEY.md section 8 row f4) -----------------------------------
 * Replaces the first loop of LidarSelector::addSparseMap (src/lidar_selection.cpp:150-168): every point of pg
 * (world frame) is projected into the new frame (T_f_w = [Rcw | Pcw], include/frame.h:89), kept when it lies
 * inside the image with the `border` margin ((patch_size_half+1)*8, :154), scored with vk::shiTomasiScore
 * on the uploaded image (flb_image_upload + flb_camera_set) and takes its grid cell
 * (int(u/grid_size)*grid_n_height + int(v/grid_size), :156) when the score is STRICTLY above the cell's value.
 *   map_value (grid_n_width*grid_n_height floats, grid_n_* = image size / grid_size, :55-56): in = the values
 *   addFromSparseMap left there (:447-455), out = updated.  winner: per cell the index into world_xyz of the
 *   point that took the cell in this call (the reference's add_voxel_points_[cell] / TYPE_POINTCLOUD), -1
 *   otherwise.  Creating the Point / Feature objects for the winners (:174-195) stays with the caller.
 *   FLB_ERR_STATE: no camera or no image, or a camera whose size differs from the uploaded image's. */
int flb_visual_candidates(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* world_xyz, int n,
                          int stride_floats, int grid_size, int border, float* map_value, int* winner);

/* pcl::VoxelGrid<PointType>::filter on x, y, z (src/laserMapping.cpp:1398-1399 downSizeFilterSurf; src/lidar_selection.cpp:7,
 * :351-352 downSizeFilter): one centroid per occupied leaf, leaves indexed and ordered as PCL does (min_b from the cloud's
 * minimum, idx = ijk . divb_mul, output in ascending idx).  The points of a leaf are summed in float in their INPUT order:
 * PCL's own within-leaf order is that of an unstable std::sort, i.e. unspecified, so this is a defined member of the family
 * of results PCL can produce, not a bit-level reproduction of one PCL build.  out_xyz: up to `capacity` x 3 floats;
 * *n_out = number of occupied leaves.  Uses the handle's scan slot as scratch (upload the scan afterwards).  Blocking. */
int flb_voxel_grid(flb_handle* h, const float* xyz, int n, int stride_floats, float leaf, float* out_xyz, int capacity, int* n_out);

/* ---- device-resident visual map (SURVEY.md section 8 rows f2 and f4) ---------------------------------------
 * The sparse visual map of LidarSelector -- feat_map (unordered_map<VOXEL_KEY, VOXEL_POINTS*>), its Points
 * (include/point.h) with their observation lists of Features (include/feature.h) and the keyframe images those
 * reference -- lives on the device.  Ids (points, features, images) are creation order.  The three calls are the
 * three visual-map steps of LidarSelector::detect (src/lidar_selection.cpp:1027-1080); ComputeJ between them is
 * flb_vio_update / flb_vio_update_enqueue, which consumes the patch list IN PLACE (no host round trip, no
 * flb_patches_upload).  Rcw / Pcw = new_frame_->T_f_w_ (updateFrameState, :905-911); pass NULL for both to take
 * it from the device state with the extrinsics given to flb_vmap_reset.  Single GPU.
 * Needs flb_camera_set and the current frame uploaded with flb_image_upload. */
typedef struct flb_vmap_params {
    int    grid_size;          /* LidarSelector::grid_size (laserMapping.cpp:1198); one patch per grid cell */
    int    ncc_en;             /* :549 */
    double outlier_threshold;  /* :560 */
    double ncc_thre;           /* :552 */
    double Rcl[9], Pcl[3];     /* sparse_map->Rcl / Pcl */
    double R_LI[9], t_LI[3];   /* set_extrinsic(transl, rot), :35-39 */
} flb_vmap_params;
/* clears the map (LidarSelector::init, :41-79), the free-slot stack of flb_vmap_reclaim included */
int flb_vmap_reset(flb_handle* h, const flb_vmap_params* p);
/* LidarSelector::addFromSparseMap (:346-587).  pg_down: the scan in the world frame after the caller's
 * pcl::VoxelGrid (0.2 m, :7, :351-352), n x stride floats.  Builds sub_sparse_map on the device: positions, warped
 * 3-level reference patches and search levels become the inputs of the next VIO update.  n_selected == NULL:
 * enqueue-only (the count stays on the device); otherwise blocks and returns sub_sparse_map->index.size(). */
int flb_vmap_select(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* pg_down, int n, int stride_floats,
                    int* n_selected);
/* sub_sparse_map of the last flb_vmap_select (blocking; any pointer may be NULL): index (grid cell), point (id),
 * search_levels, propa_errors, voxel_points[i]->pos_, patch (3 x 64 floats each). */
int flb_vmap_selected(flb_handle* h, int capacity, int* n, int* index, int* point, int* search_level, float* error, double* pos,
                      float* patch);
/* LidarSelector::addSparseMap (:142-202): Shi-Tomasi candidate per grid cell over pg (world frame, unfiltered scan),
 * then one new Point + Feature per won cell (AddPoint, :204-230).  Enqueue-only. */
int flb_vmap_grow(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* pg, int n, int stride_floats, int frame_id);
/* LidarSelector::addObservation (:913-965) for the patches of the last flb_vmap_select, with the frame pose AFTER
 * ComputeJ (NULL, NULL = the device state).  Enqueue-only. */
int flb_vmap_add_observations(flb_handle* h, const double Rcw[9], const double Pcw[3], int frame_id);
/* publish_frame_world_rgb (src/laserMapping.cpp:710-745): colour every world point that projects into the current
 * frame with the bilinear BGR sample of LidarSelector::getpixel (src/lidar_selection.cpp:1007-1025).  bgr: the
 * colour frame (img_rgb), 3 bytes per pixel, uploaded by the call; or NULL: the colour frame of the current image set
 * (flb_image_upload_bgr), read on the device with no host copy and no upload (FLB_ERR_STATE when the current image came
 * from flb_image_upload or does not match the camera's size); rgb: n x 3 bytes (r, g, b as the reference stores them); valid[i] = 1
 * for the points the reference pushes into laserCloudWorldRGB (in front of the camera, inside the image), whose order
 * is the input order.  Rcw / Pcw NULL: from the device state (after flb_vmap_reset).  Blocking. */
int flb_colorize(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, const float* world_xyz, int n,
                 int stride_floats, uint8_t* rgb, uint8_t* valid);

/* ---- the frame's world cloud on the device (pcl_wait_pub) -------------------------------------------------------
 * pcl_wait_pub (src/laserMapping.cpp:1763-1772) is the source cloud in the world frame; its three readers are the visual
 * map's select and grow (LidarSelector::detect(img, pcl_wait_pub), :1345) and publish_frame_world_rgb (:710-745).
 * flb_world_cloud builds it on the device and the *_cloud calls read it there: no read-back of the state, no host
 * transform, no host voxel filter and no upload of the cloud. */
#define FLB_CLOUD_SCAN        0   /* feats_down_body: the scan last uploaded (dense_map_en = 0) */
#define FLB_CLOUD_UNDISTORTED 1   /* feats_undistort: the output of the last flb_imu_undistort (dense_map_en = 1) */
/* The source cloud, in the caller's original order, transformed by RGBpointBodyToWorld (:303-315, pointBodyToWorld's op
 * order; double math, float store) at (R, p) with prm->R_LI / prm->t_LI, or at the device state x when R == p == NULL
 * (stream order: call it after the LIO update, after flb_map_add_scan).  IKFoM callers pass R = rot, p = pos and the
 * offset_R_L_I / offset_T_L_I extrinsic.  The library keeps the cloud until the next call; it is a copy, so later scan
 * uploads and flb_imu_undistort calls do not change it.  Blocking (one 32-byte read).  *n_out (may be NULL) = points.
 * On any error no cloud is held, and every *_cloud call returns FLB_ERR_STATE until the next successful call.
 *   FLB_ERR_STATE: no source (no scan, the scan slot used as scratch by flb_voxel_grid, no flb_imu_undistort since
 *   creation or since a failed one), no pose given and no device state, FLB_CLOUD_SCAN after flb_comm_init /
 *   flb_p2p_attach (each rank holds only its shard of the scan).
 *   FLB_ERR_INVALID: prm == NULL, a bad source, exactly one of R / p NULL, a transformed point that is not finite or
 *   whose |coordinate| exceeds 5e5 (the visual map's limit, as flb_vmap_select / flb_vmap_grow / flb_colorize check). */
int flb_world_cloud(flb_handle* h, const struct flb_lio_params* prm, const double R[9], const double p[3], int source, int* n_out);
/* publish_frame_world / the PCD save: up to `capacity` points of the world cloud, xyz floats (blocking). */
int flb_world_cloud_download(flb_handle* h, float* xyz, int capacity, int* n_out);

/* ---- the effective points of the last LIO pass on the device (publish_effect_world) ------------------------------
 * publish_effect_world (src/laserMapping.cpp:871-885, called at :1776) publishes laserCloudOri -- the body points of the
 * effective rows point_selected_surf[i] && res_last[i] <= 2.0 of the last iteration the LIO loop ran (:1588-1600) --
 * transformed by RGBpointBodyToWorld at the state after the update.  Every LIO pass keeps its row mask on the device,
 * so the cloud costs no extra pass and no read-back of the scan.
 *   The effect cloud is the rows of the last LIO pass executed on the handle (stream order), in scan-index order
 * (laserCloudOri's), body x, y, z, transformed at (R, p) with prm->R_LI / prm->t_LI, or at the device state x when
 * R == p == NULL.  The passes that count: the stop pass of flb_lio_update, flb_lio_update_enqueue and flb_frame_enqueue;
 * the last h_share_model evaluation of flb_lio_update_ikfom; the pass of flb_lio_pass.  Batched frames (flb_batch_*) do
 * not touch it.  IKFoM callers pass R = rot, p = pos and the offset_R_L_I / offset_T_L_I extrinsic, as for
 * flb_world_cloud.
 *   The first call after a pass captures that pass's rows; with no pass since, the rows captured last are transformed
 * at the new pose (the reference republishes its stale laserCloudOri when the loop does not run: before flg_EKF_inited,
 * :1506, or with lidar_en off).  No pass ever: 0 points.  The scan, its row mask and its plane cache are double-buffered
 * together, so a pass's rows can be captured until the second scan upload after it (or an flb_voxel_grid, which uses
 * the scan slot as scratch); after that the call returns FLB_ERR_STATE until the next pass.  Intensity is not carried.
 * Blocking.  *n_out (may be NULL) = points.  On any error no effect cloud is held.
 *   FLB_ERR_STATE: the pass's rows were replaced before capture, no pose given and no device state, after flb_comm_init
 *   / flb_p2p_attach (each rank holds only its shard of the scan).
 *   FLB_ERR_INVALID: prm == NULL, exactly one of R / p NULL, a transformed point that is not finite. */
int flb_effect_cloud(flb_handle* h, const struct flb_lio_params* prm, const double R[9], const double p[3], int* n_out);
/* pubLaserCloudEffect's points: up to `capacity` points of the effect cloud, xyz floats (blocking, as
 * flb_world_cloud_download).  FLB_ERR_INVALID for a bad capacity or buffer, FLB_ERR_STATE when no effect cloud is held. */
int flb_effect_cloud_download(flb_handle* h, float* xyz, int capacity, int* n_out);
/* flb_vmap_select / flb_vmap_grow / flb_colorize with pg = the world cloud: the same pose, enqueue and blocking rules and
 * byte-identical results to those calls on the host-transformed cloud.  flb_vmap_select_cloud applies downSizeFilter
 * (pcl::VoxelGrid with `leaf`, 0.2 in the reference: src/lidar_selection.cpp:7, :351-353; flb_voxel_grid's result) on
 * the device first, in buffers of its own (the scan slot is untouched); the leaf count stays on the device, so with
 * n_selected == NULL it is enqueue-only.  FLB_ERR_INVALID for a leaf too small for the cloud's extent (PCL's
 * index-overflow case, as in flb_voxel_grid).  flb_colorize_cloud writes world-cloud-size entries to rgb (x 3) / valid. */
int flb_vmap_select_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], float leaf, int* n_selected);
int flb_vmap_grow_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], int frame_id);
int flb_colorize_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, uint8_t* rgb,
                       uint8_t* valid);
/* publish_frame_world_rgb's laserCloudWorldRGB (src/laserMapping.cpp:726-747) built on the device as records: the world
 * cloud's points that flb_colorize_cloud marks valid, in world-cloud order, with its r, g, b bytes (its clamp for pc in
 * (-1, 0) and for the last row and column included).  Pose, bgr and stride rules, and the FLB_ERR_STATE cases (no
 * camera, no world cloud, bgr == NULL without a colour frame of the camera's size, no pose and no flb_vmap_reset), are
 * flb_colorize_cloud's; a world cloud of 0 points gives 0 records (and needs no pose).  One 32-byte record per point, the
 * layout of pcl::PointXYZRGB:
 *   float x, y, z at bytes 0 / 4 / 8; float 1.0f at 12 (data[3]); uint8 b, g, r, a at 16..19 with a = 255; bytes 20..31 zero.
 * Blocking: reading the record count back (4 bytes) is its one synchronise.  *n_out (may be NULL) = records.  The LIO
 * export (flb_lio_export) stays valid.  With a save open (flb_rgb_save_begin) the records are appended to it as well.
 * On any error no coloured cloud is held.  FLB_ERR_INVALID: bgr with stride_bytes < 3 * width. */
int flb_rgb_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, int* n_out);
/* Up to `capacity` records of the last flb_rgb_cloud, 32 bytes each, into points32 (blocking); *n_out = records held.
 * FLB_ERR_INVALID for a bad capacity or buffer, FLB_ERR_STATE when no coloured cloud is held. */
int flb_rgb_cloud_download(flb_handle* h, void* points32, int capacity, int* n_out);
/* pcl_wait_save with pcd_save_en (`*pcl_wait_save += *laserCloudWorldRGB`, :777; written as rgb_scan_all.pcd at exit,
 * :1839-1846) on the device.  After flb_rgb_save_begin every successful flb_rgb_cloud appends its records, so the save
 * is the frames' clouds concatenated in call order.  It is held as 16-byte records {x, y, z, bgra} in device chunks of
 * 2^20 records, allocated as frames need them and never copied.  max_points (>= 1) caps it: a frame whose records would
 * pass the cap is not appended at all and its record count is added to `dropped` (so is a frame for which no chunk can be
 * allocated); its own cloud is still built and flb_rgb_cloud returns FLB_OK.  One save per handle.
 *   flb_rgb_save_begin: FLB_ERR_INVALID for max_points < 1, FLB_ERR_STATE when a save is open.
 *   flb_rgb_save_size: records held, records dropped, device bytes the save holds (any pointer may be NULL).
 *   flb_rgb_save_download: records first .. first + count - 1 as 32-byte records (flb_rgb_cloud's layout), expanded on
 *   the device through a bounded staging buffer (blocking); FLB_ERR_INVALID for a range outside the save.
 *   flb_rgb_save_end: frees the save (no save open: nothing to do).
 *   Size and download return FLB_ERR_STATE when no save is open. */
int flb_rgb_save_begin(flb_handle* h, int64_t max_points);
int flb_rgb_save_size(flb_handle* h, int64_t* n, int64_t* dropped, int64_t* device_bytes);
int flb_rgb_save_download(flb_handle* h, int64_t first, int64_t count, void* points32);
int flb_rgb_save_end(flb_handle* h);
/* LidarSelector::display_keypatch (src/lidar_selection.cpp:985-1005) without its putText: the current image set's
 * camera-size colour frame (img_cp = img_rgb, :1035-1036) with one filled circle per patch of the current patch list,
 * written to bgr_out (W x H x 3 BGR8, stride_bytes a row).  The image set's colour frame itself is not modified, so
 * flb_colorize(_cloud) still read the undrawn img_rgb.  For patch i, in list order:
 *   centre: cvRound of cv::Point2f(world2cam(Rcw * pos_i + Pcw)) -- the double projection rounded to float, then to
 *     int half to even; a non-finite coordinate, or one that rounds beyond +-2^30, draws nothing (a definition: OpenCV's
 *     clipping overflows there);
 *   shape: cv::circle(img, c, 6, colour, FILLED, LINE_8), the fixed 113-pixel disk, clipped to the image;
 *   colour: errors[i] < 8000 (float) green (0, 255, 0), otherwise (NaN included) blue (255, 0, 0);
 *   overlaps: the highest patch index wins, as drawing in list order leaves it.
 * errors[i] = sub_sparse_map->errors[i] at :995: the errors of the last VIO pass executed on this patch list
 * (flb_vio_errors' values), or, when no pass has run since a visual-map selection, that selection's errors
 * (flb_vmap_selected's, :576); zero after flb_patches_upload until a pass runs.
 * Rcw / Pcw: new_frame_->T_f_w_; NULL for both = from the device state in stream order (after flb_vmap_reset), which
 * after flb_vio_update_enqueue is the pose ComputeJ leaves (:982).  *n_patches (may be NULL) = the list's length; 0
 * leaves the frame unchanged (display_keypatch returns before its text).
 * Completion: bgr_out page-locked (flb_host_alloc): enqueue-only, the bytes are valid after the next synchronising call
 * (flb_synchronize, flb_state_download); *n_patches too when it is page-locked or the count is on the host (a count an
 * enqueue-only flb_vmap_select* left on the device is copied into pageable memory before the call returns).  Pageable
 * bgr_out: blocking.
 *   FLB_ERR_INVALID: bgr_out NULL, stride_bytes < 3 W, exactly one of Rcw / Pcw NULL.
 *   FLB_ERR_STATE: no camera; no colour frame of the camera's size (no image, or one from flb_image_upload); after
 *   flb_comm_init / flb_p2p_attach (each rank holds only its shard of the patch list); no patch list; no pose given and
 *   no flb_vmap_reset or no device state.
 * On any error nothing is written. */
int flb_keypatch_image(flb_handle* h, const double Rcw[9], const double Pcw[3], uint8_t* bgr_out, int stride_bytes, int* n_patches);
/* Gives back what the reference frees (opt-in; enqueue-only, no host synchronisation).  A Feature is owned by
 * Point::obs_ alone, so it dies when addObservation evicts it (deleteFeatureRef(getFurthestViewObs),
 * src/lidar_selection.cpp:946-950); its keyframe image (Feature::img, :183, :957) dies with the last Feature that refers
 * to it; Points are never freed (feat_map keeps them).  The call compacts the feature array to the features some
 * observation list names -- creation order kept, the lists remapped -- and puts every keyframe slot no live feature
 * names (except the current frame's) on a free-slot stack that the following frames fill before the pool grows.  Image
 * data never moves.  Selections, patches, errors and observation lists are unchanged by it: nothing refers to a feature
 * id across calls.  Call it between any two visual-map calls (e.g. after flb_vmap_add_observations) at the cadence the
 * caller chooses; without it nothing changes. */
int flb_vmap_reclaim(flb_handle* h);
/* memory of the visual map (blocking; any pointer may be NULL): points; features in the array, of which `dead` are no
 * longer named by any observation list (reclaimable); feature-array capacity; keyframe slots in use, on the free-slot
 * stack, and the pool's capacity in slots; device bytes the visual map holds. */
int flb_vmap_usage(flb_handle* h, int* points, int* features, int* dead_features, int* feature_capacity, int* slots_in_use,
                   int* free_slots, int* pool_slots, int64_t* device_bytes);
/* the keyframe image in pool slot `slot` (tests, debugging; blocking): width x height bytes into gray (capacity bytes). */
int flb_vmap_keyframe(flb_handle* h, int slot, uint8_t* gray, int capacity);
/* sizes (blocking): points, features, keyframe images, patches of the last selection, items appended by the last
 * grow / add_observations call.  Any pointer may be NULL.  After a flb_vmap_reclaim, features is the compacted array's
 * length and images the keyframe slots in use. */
int flb_vmap_counts(flb_handle* h, int* points, int* features, int* images, int* selected, int* last_added);
int flb_vmap_map_value(flb_handle* h, float* out, int capacity);       /* map_value[length] (:356, :455, :162) */
/* the whole map (tests, debugging; blocking): per point pos (3 doubles), value, n_obs, newest-first feature ids
 * (20, -1 padded); per feature px(2) f(3) T_f_w R(9) t(3) = 17 doubles, score, {level, frame id, image slot}.
 * After a flb_vmap_reclaim: the surviving features in creation order, the ids as remapped. */
int flb_vmap_dump(flb_handle* h, int cap_points, int cap_features, double* pos, float* value, int* n_obs, int* obs20, double* ft_geo17,
                  float* ft_score, int* ft_level_id_img);

/* One measurement pass of LidarSelector::UpdateState (src/lidar_selection.cpp:772-857)
 * at pose (R,p) and pyramid level `level`. */
int flb_vio_pass(flb_handle* h, const flb_vio_params* prm, const double R[9], const double p[3], int level,
                 flb_vio_eq* out);
/* Rows of the LAST flb_vio_pass: z Pn*64 doubles, H_sub Pn*64 x 6 row-major,
 * errors Pn floats (sub_sparse_map->errors). */
int flb_vio_export(flb_handle* h, double* z, double* H_sub, float* errors);

/* LidarSelector::ComputeJ (src/lidar_selection.cpp:967-983): UpdateState (:743-902)
 * for level = 2,1,0, then cov -= G*cov, all on the device. */
int flb_vio_update(flb_handle* h, const flb_vio_params* prm, flb_state18* x, const flb_state18* x_prop,
                   flb_vio_report* rep);
/* float LidarSelector::UpdateState(cv::Mat img, float total_residual, int level) (include/lidar_selection.h:72,
 * src/lidar_selection.cpp:743-902) on its own: the iteration loop of ONE pyramid level starting from *x with
 * last_error = total_residual; returns the level's last_error like the reference (0 when there are no patches).
 * G18x6 (may be NULL): the non-zero block (columns 0..5) of the member G after the call (:874), which the caller's
 * ComputeJ applies as state->cov -= G * state->cov (:980) -- this entry point leaves the covariance alone. */
int flb_vio_update_level(flb_handle* h, const flb_vio_params* prm, int level, float total_residual, flb_state18* x,
                         const flb_state18* x_prop, float* last_error, double* G18x6, flb_vio_report* rep);
/* sub_sparse_map->errors[i] as ComputeJ leaves them (src/lidar_selection.cpp:851: the per-patch errors of the
 * LAST pass executed by the last flb_vio_update / flb_vio_update_enqueue; read by display_keypatch, :995).
 * errors: up to `capacity` floats, patch order. */
int flb_vio_errors(flb_handle* h, float* errors, int capacity);

/* ---- device-resident frame loop (benchmark / pipeline use) ---------------------------
 * Enqueue-only variants: state stays on the device between calls, nothing is copied
 * back until flb_state_download.  flb_frame_enqueue = one LIO update followed by one
 * VIO update whose prior is the LIO posterior (zero-motion propagation). */
int flb_state_upload(flb_handle* h, const flb_state18* x, const flb_state18* x_prop);
int flb_state_download(flb_handle* h, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio);
/* One frame in ONE call (the reference's per-frame work on this path: sync_packages -> LIO update -> VIO update,
 * src/laserMapping.cpp:1269-1460): scan upload, state upload, LIO update, and -- when vprm != NULL -- image upload,
 * patch-list upload (patch_pos == NULL: keep the list already on the device, e.g. one built by flb_vmap_select),
 * state_propagat = state, VIO update; result_slot >= 0 also enqueues the read-back into that slot
 * (flb_state_download_wait collects it).  Everything is enqueue-only. */
typedef struct flb_frame_inputs {
    const float*   scan_xyz;  int n_scan, scan_stride;                 /* feats_down_body, floats per point */
    const uint8_t* gray;      int width, height, stride_bytes;         /* NULL: keep the image on the device */
    const double*  patch_pos; const float* patch; const int* search_level; int Pn;
    const flb_state18* x; const flb_state18* x_prop;
} flb_frame_inputs;
int flb_frame_enqueue(flb_handle* h, const flb_frame_inputs* in, const flb_lio_params* lprm, const flb_vio_params* vprm, int result_slot);
/* Pipelined read-back (two result slots): _enqueue copies the state and both reports of everything enqueued so far and
 * returns at once; _wait blocks on that slot only -- frame k's result is collected while frame k+1 already uploads
 * and runs (uploads never overwrite what an enqueued kernel still reads: stream order, and events for the copy stream). */
int flb_state_download_enqueue(flb_handle* h, int slot);
int flb_state_download_wait(flb_handle* h, int slot, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio);
int flb_lio_update_enqueue(flb_handle* h, const flb_lio_params* prm);
int flb_vio_update_enqueue(flb_handle* h, const flb_vio_params* prm);
/* restore x := x_prop := the state given to the last flb_state_upload (device-side copy) */
int flb_state_reset_enqueue(flb_handle* h);
/* x_prop := x on the device: `state_propagat = state` (src/laserMapping.cpp:1292) with a
 * zero-motion IMU propagation between the LIO and the VIO update */
int flb_state_set_prior_enqueue(flb_handle* h);

/* ---- batched frames (SURVEY.md section 7 H2(iv)) ------------------------------------------------------------
 * B independent frames (own scan, own prior) against the handle's map -- and, for the VIO step, its image and
 * patch list -- advanced together: every pass of the iterated update is ONE launch over all B frames (kernel-per-
 * pass path, blockIdx.y = frame), so the grid is B times a frame's.  One frame's passes are latency-bound at the
 * sizes of BASELINE.json (DESIGN.md section 4); this is the mode in which the kernels run at their throughput
 * (relocalisation against a map, multi-hypothesis tracking, offline batches).  Every frame's result is bit-identical
 * to the same frame run alone through the kernel-per-pass path (flb_config.persistent = 0). */
int flb_batch_begin(flb_handle* h, int B, int max_points_per_frame);
int flb_batch_set_frame(flb_handle* h, int frame, const float* body_xyz, int N, int stride_floats, const flb_state18* x,
                        const flb_state18* x_prop);
int flb_batch_state_reset_enqueue(flb_handle* h);
/* LIO update of every frame, then (vprm != NULL) VIO update with the LIO posterior as prior.  Enqueue-only.
 * FLB_ERR_STATE, before anything is enqueued: no batch, a frame not set, and, when the VIO step runs (vprm != NULL,
 * patches uploaded, max_iteration > 0), no camera or no image, or a camera whose size differs from the image's. */
int flb_batch_update_enqueue(flb_handle* h, const flb_lio_params* lprm, const flb_vio_params* vprm);
int flb_batch_state_download(flb_handle* h, int frame, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio);

/* Per-kernel-family device time of the work enqueued between start and stop,
 * measured with CUDA events on the handle's stream (adds one event pair per launch:
 * use for profiling runs, not for headline timing).  ms[0] = LIO rematch passes,
 * ms[1] = LIO plain passes, ms[2] = VIO passes, ms[3] = solves/finalize; launches[i]
 * the matching launch counts. */
int flb_profile_start(flb_handle* h);
int flb_profile_stop(flb_handle* h, double ms[4], int64_t launches[4]);
/* Device-side pass trace of the persistent kernels (profiling aid; %globaltimer).  After an update,
 * flb_trace_download(which = 0 LIO / 1 VIO) returns microseconds since kernel entry, two per pass:
 * [2k] all blocks arrived at the pass barrier, [2k+1] the leader finished the solve and released. */
int flb_trace_enable(flb_handle* h, int on);
int flb_trace_download(flb_handle* h, int which, double* us, int max_entries, int* n_entries);
/* kernels launched by this handle since creation */
int64_t flb_launch_count(const flb_handle* h);

/* ---- multi-GPU (SURVEY.md §8e) -------------------------------------------------------
 * One process per GPU.  Each rank uploads ITS contiguous shard of the scan points and
 * patches, the full map and image, and identical states; every pass all-reduces the
 * packed normal equations (ncclAllReduce, ncclDouble, ncclSum) and every rank runs
 * the identical solve.  unique_id is the 128-byte ncclUniqueId produced by
 * flb_comm_unique_id on rank 0 and distributed by the caller (e.g. torch.distributed). */
int flb_comm_unique_id(void* unique_id_128b);
int flb_comm_init(flb_handle* h, const void* unique_id_128b, int rank, int world_size);
int flb_comm_destroy(flb_handle* h);

/* Fused NVLink exchange: the NVLink-native alternative to the NCCL path.  Inside the persistent update
 * kernel every rank writes its packed sums (leader block) and its VIO per-patch errors (the worker warp that
 * computed each one) straight into every rank's mailbox over NVLink peer memory as self-validating units
 * {payload, exchange tag} -- one store instruction per unit, no separate flag, no system fence, one NVLink
 * traversal per exchange; one kernel per update, no NCCL call, bit-identical results on every rank and to the
 * single-GPU run up to the summation order.  After FLB_ERR_TIMEOUT in this mode the exchange counters of the
 * ranks may differ: repeat flb_p2p_export / flb_p2p_attach on every rank.
 * Each rank: flb_p2p_export() -> 64-byte CUDA IPC handle; gather all handles (rank order) with any host
 * transport; flb_p2p_attach().  One process per GPU, all GPUs NVLink peers; <= 8 ranks. */
int flb_p2p_export(flb_handle* h, void* handle_64b);
int flb_p2p_attach(flb_handle* h, int rank, int world_size, const void* handles_world_x_64b);
int flb_p2p_detach(flb_handle* h);

/* ---- test / tracing aids (not needed by a caller of the path) -------------------------------------------
 * flb_debug_set_packet_epoch: move the pose-packet flag base (wrap-around test).  flb_debug_block_stamps /
 * flb_debug_vio_stamps: per-block %globaltimer stamps of the last traced LIO / VIO update. */
int flb_debug_set_packet_epoch(flb_handle* h, unsigned epoch);
int flb_debug_block_stamps(flb_handle* h, unsigned long long* out, int max_blocks, int* nblocks);
int flb_debug_vio_stamps(flb_handle* h, unsigned long long* out, int max_blocks, int* nblocks, int* words_per_block);
/* flb_debug_scan_order: src_index[i] = index in the caller's scan array of the point at position i of the uploaded
 * (Morton-ordered) scan; capacity >= the scan's point count.  Test aid for the upload's two ordering paths. */
int flb_debug_scan_order(flb_handle* h, int* src_index, int capacity);
/* flb_debug_set_scan_sort: ordering path of the following flb_scan_upload calls -- 0 automatic (by size and by
 * whether the handle's stream is busy), 1 the one-block kernel (scans of <= 25 600 points), 2 the device-wide sort. */
int flb_debug_set_scan_sort(flb_handle* h, int mode);
/* flb_debug_set_map_index: cell index of the following map rebuilds -- 0 automatic (the dense table), 1 dense always,
 * 2 the sparse index at the configured cell.  Test and measurement aid. */
int flb_debug_set_map_index(flb_handle* h, int mode);

#ifdef __cplusplus
}
#endif
#endif /* FASTLIVO_B200_H */
