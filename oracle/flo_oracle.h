/* TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
 *
 * flo_oracle: a dependency-free CPU restatement of FAST-LIVO's per-frame
 * measurement assembly + iterated ESKF update (the hot path of SURVEY.md §8),
 * used ONLY as the checker.  Only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load liboracle.so.  The
 * product library (fast-livo_b200/libfastlivo_b200.so) never links, loads or
 * calls anything in this directory.
 *
 * PARITY STATUS: "parity unpinned".  The reference has no tests, golden vectors
 * or fixtures (SURVEY.md §4), and its node cannot be built here (no Eigen / PCL /
 * OpenCV / Sophus / ROS / vikit).  The one reference translation unit that does
 * compile -- include/ikd-Tree/ikd_Tree.cpp -- is built unmodified into
 * oracle/_ref/libikdtree_ref.so and pins the kNN half; everything else follows
 * the cited reference lines op for op, with Eigen's colPivHouseholderQr /
 * inverse() and vikit's pinhole model restated from their published algorithms
 * (SURVEY.md Appendix C).
 *
 * All citations are relative to the reference tree (hku-mars/FAST-LIVO @ dcebf84).
 */
#ifndef FLO_ORACLE_H
#define FLO_ORACLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 18-DoF state, reference include/common_lib.h:296-381 (StatesGroup).
 * rot is row-major 3x3; cov is row-major 18x18, order [rot,pos,vel,bg,ba,g]. */
typedef struct flo_state18 {
    double rot[9];
    double pos[3];
    double vel[3];
    double bg[3];
    double ba[3];
    double grav[3];
    double cov[324];
} flo_state18;

/* kNN back-end signature; matches ikdref_knn in oracle/ikdtree_ref_wrap.cpp so
 * the reference's own ikd-Tree can be plugged in by function pointer. */
typedef int (*flo_knn_fn)(void* ctx, const float* q, int nq, int k, int* idx, float* d2, int nthreads);

/* ---- SO(3) and state algebra ------------------------------------------------ */
void flo_exp3(const double v[3], double R[9]);           /* so3_math.h:54-72 */
void flo_log3(const double R[9], double out[3]);         /* so3_math.h:75-81 */
void flo_state_boxplus(flo_state18* x, const double d[18]);                 /* common_lib.h:343-352 */
void flo_state_boxminus(const flo_state18* a, const flo_state18* b, double out[18]); /* a - b, common_lib.h:354-365 */
int  flo_inverse(const double* A, int n, double* Ainv);  /* Eigen inverse() = PartialPivLU, App. C */

/* ---- kNN (brute force, float32, reference distance + ordering semantics) ---- */
int flo_knn_brute(void* map_ctx, const float* q, int nq, int k, int* idx, float* d2, int nthreads);
void* flo_knn_brute_ctx(const float* map_xyz, int M);    /* copies; free with flo_free */
void  flo_free(void* p);

/* ---- plane fit, common_lib.h:448-493 (esti_plane<float>) --------------------- */
/* nb: 5 neighbours x 3 floats, ascending distance.  Returns 1 when every
 * neighbour lies within `threshold` of the plane. */
int flo_esti_plane(const float nb[15], float threshold, float pabcd[4]);

/* ---- LIO ---------------------------------------------------------------------- */
typedef struct flo_lio flo_lio;

typedef struct flo_lio_params {
    double R_LI[9];          /* Lidar_rot_to_IMU, laserMapping.cpp:104-105 */
    double t_LI[3];          /* Lidar_offset_to_IMU */
    double laser_point_cov;  /* LASER_POINT_COV, laserMapping.cpp:1109 */
    int    max_iteration;    /* NUM_MAX_ITERATIONS */
    double conv_rot_deg;     /* 0.01  (laserMapping.cpp:1688); 0 disables early stop */
    double conv_pos_cm;      /* 0.015 */
    int    nthreads;         /* MP_PROC_NUM (CMakeLists.txt:19-37) */
} flo_lio_params;

typedef struct flo_lio_report {
    int    passes;           /* loop bodies executed */
    int    knn_passes;       /* passes with nearest_search_en */
    int    n_eff_last;       /* effct_feat_num of the last pass */
    double res_mean_last;    /* laserMapping.cpp:1602 */
    int64_t rows_total;      /* sum of effct_feat_num over passes */
    int    converged_last;
} flo_lio_report;

flo_lio* flo_lio_create(const float* map_xyz, int M, const float* scan_body_xyz, int N,
                        flo_knn_fn knn, void* knn_ctx);
void     flo_lio_destroy(flo_lio*);

/* One pass of the matching loop (laserMapping.cpp:1508-1630) at pose (R,p).
 * Optional outputs (may be NULL), all sized for N points:
 *   world_xyz N*3 float; nn_idx N*5 int (-1 = missing); nn_d2 N*5 float;
 *   pabcd N*4 float (plane of this pass; untouched when not fitted);
 *   pd2 N float; selected N uint8 (point_selected_surf after the pass);
 *   Hsub n*6 double row-major [A, n] (live layout, :1608-1629);
 *   h_x n*12 double row-major [n, A, B, C] (IKFoM layout, :1059-1089);
 *   meas n double; sel_idx n int (scan index of each compacted row);
 *   HTH6 36, HTz6 6, HTH12 144, HTh12 12 (row-major).
 * Returns effct_feat_num (n). */
int flo_lio_pass(flo_lio*, const flo_lio_params*, const double R[9], const double p[3], int rematch,
                 float* world_xyz, int* nn_idx, float* nn_d2, float* pabcd, float* pd2, uint8_t* selected,
                 double* Hsub, double* h_x, double* meas, int* sel_idx,
                 double* HTH6, double* HTz6, double* HTH12, double* HTh12,
                 double* total_residual);

/* Whole iterated update, laserMapping.cpp:1469-1733 (Appendix A of SURVEY.md). */
int flo_lio_update(flo_lio*, const flo_lio_params*, flo_state18* x, const flo_state18* x_prop,
                   flo_lio_report* rep);

/* fresh frame: point_selected_surf = true, res_last = 1000 (src/laserMapping.cpp:1441,1469) */
void flo_lio_reset(flo_lio*);

/* ---- IKFoM-typed estimator (SURVEY.md section 8 row a8; oracle/flo_ikfom.cpp) ---------------------
 * state_ikfom, include/use-ikfom.hpp:12-21.  Quaternions are (x, y, z, w) like Eigen's coeffs();
 * P is the 23x23 covariance, row-major, order [pos, rot, offset_R_L_I, offset_T_L_I, vel, bg, ba, grav(2)]. */
typedef struct flo_state_ikfom {
    double pos[3];
    double rot[4];
    double offset_R_L_I[4];
    double offset_T_L_I[3];
    double vel[3], bg[3], ba[3];
    double grav[3];
    double P[529];
} flo_state_ikfom;

typedef struct flo_ikfom_params {
    double laser_point_cov;   /* R of update_iterated_dyn_share_modified(R, ...) (laserMapping.cpp:1484) */
    int    max_iteration;     /* maximum_iter (init_dyn_share, laserMapping.cpp:1235) */
    double limit[23];         /* epsi = 0.001 each (laserMapping.cpp:1233-1234) */
    int    nthreads;
} flo_ikfom_params;

typedef struct flo_ikfom_report {
    int passes, knn_passes, n_eff_last, converged_last;
    double res_mean_last;
    int64_t rows_total;
} flo_ikfom_report;

void flo_ikfom_boxplus(flo_state_ikfom* x, const double* d23);
void flo_ikfom_boxminus(const flo_state_ikfom* a, const flo_state_ikfom* b, double* res23);   /* a [-] b */
void flo_quat_to_R(const double* q_xyzw, double* R9);
/* esekfom.hpp:1619-1928 driven by h_share_model (laserMapping.cpp:960-1094) */
int  flo_ikfom_update(flo_lio*, const flo_ikfom_params*, flo_state_ikfom* x, flo_ikfom_report* rep);

/* ---- IMU forward propagation + backward undistortion (SURVEY.md section 8 row f3; oracle/flo_imu.cpp) ----
 * ImuProcess::UndistortPcl from :655 on (src/IMU_Processing.cpp:655-808). */
typedef struct flo_imu_sample { double t; double gyr[3]; double acc[3]; } flo_imu_sample;   /* sensor_msgs::Imu */
typedef struct flo_imu_params {
    double cov_gyr[3], cov_acc[3], cov_bias_gyr[3], cov_bias_acc[3];   /* ImuProcess members, :15-20 */
    double G_m_s2, mean_acc_norm;                                      /* :688 */
    double R_LI[9], t_LI[3];                                           /* Lid_rot_to_IMU, Lid_offset_to_IMU */
} flo_imu_params;
typedef struct flo_imu_carry { double last_lidar_end_time; double acc_s_last[3]; double angvel_last[3]; } flo_imu_carry;
/* v_imu = last_imu_ followed by meas.imu (:617-618).  x: state_inout (in/out).  pts_xyz (n_points x 3 float,
 * in/out) with offset_ms = PointType::curvature.  poses_out (optional): IMUpose as 22 doubles per entry
 * [offset_time, acc, gyr, vel, pos, rot]. */
int flo_imu_undistort(const flo_imu_params* prm, flo_imu_carry* carry, const flo_imu_sample* v_imu, int n_imu,
                      double pcl_beg_time, double pcl_end_time, flo_state18* x, float* pts_xyz,
                      const float* offset_ms, int n_points, int* n_poses_out, double* poses_out);

/* ---- VIO ---------------------------------------------------------------------- */
typedef struct flo_vio flo_vio;

typedef struct flo_cam {
    int    width, height;
    double fx, fy, cx, cy;   /* vikit PinholeCamera */
    double d[5];             /* radtan d0..d4; distortion on iff |d0| > 1e-7 */
} flo_cam;

typedef struct flo_vio_params {
    double Rcl[9], Pcl[3];   /* camera<-lidar extrinsic (sparse_map->Rcl/Pcl, laserMapping.cpp:1201-1209) */
    double R_LI[9], t_LI[3]; /* set_extrinsic(transl, rot), lidar_selection.cpp:35-39 */
    double img_point_cov;    /* lidar_selection.cpp:873 */
    int    max_iteration;    /* NUM_MAX_ITERATIONS (lidar_selection.h:42) */
    float  conv_rot_deg;     /* 0.001f (lidar_selection.cpp:883); 0 disables */
    float  conv_pos_cm;      /* 0.001f */
    int    force_all_passes; /* benchmark mode: ignore the error<=last_error test and EKF_end */
} flo_vio_params;

typedef struct flo_vio_report {
    int   passes[3];         /* per level 2,1,0 (index = level) */
    float last_error[3];
    int64_t rows_total;      /* n_meas summed over passes */
    int   skipped_last;      /* patches skipped by the bounds/depth guard in the last pass */
    int   cov_updated;
    int   rejects;           /* passes whose error exceeded last_error (:888-892): test scenarios assert on it */
} flo_vio_report;

flo_vio* flo_vio_create(const uint8_t* gray, int width, int height, int stride,
                        const double* pos, const float* patch, const int* search_level, int Pn,
                        const flo_cam* cam);
void     flo_vio_destroy(flo_vio*);

/* One measurement pass of UpdateState (lidar_selection.cpp:772-857) at the pose in x.
 * Optional outputs: z Pn*64 double, H_sub Pn*64*6 double row-major, errors Pn float,
 * HTH6 36, HTz6 6.  Returns mean error (error/n_meas) as float; *n_meas_out rows. */
float flo_vio_pass(flo_vio*, const flo_vio_params*, const double R[9], const double p[3], int level,
                   double* z, double* H_sub, float* errors, double* HTH6, double* HTz6,
                   int64_t* n_meas_out, int* skipped_out);

/* ComputeJ (lidar_selection.cpp:967-983): levels 2,1,0 of UpdateState (:743-902). */
int flo_vio_update(flo_vio*, const flo_vio_params*, flo_state18* x, const flo_state18* x_prop,
                   flo_vio_report* rep);

/* LidarSelector::UpdateState(img, total_residual, level) alone (lidar_selection.cpp:743-902); G324: the member G
 * (18 x 18, in/out); returns last_error. */
float flo_vio_update_level(flo_vio*, const flo_vio_params*, int level, float total_residual, flo_state18* x,
                           const flo_state18* x_prop, double* G324, flo_vio_report* rep);
/* sub_sparse_map->errors as the last pass executed left them (lidar_selection.cpp:851). */
void flo_vio_errors(const flo_vio*, float* errors);

/* vikit PinholeCamera::world2cam(Vector3d) (SURVEY.md Appendix C). */
void flo_world2cam(const flo_cam* cam, const double pf[3], double px[2]);

/* ---- visual-map growth: candidate scoring (SURVEY.md section 8 row f4; oracle/flo_vmap.cpp) ------------ */
float flo_shi_tomasi(const uint8_t* img, int width, int height, int stride, int u, int v);   /* vk::shiTomasiScore */
/* first loop of LidarSelector::addSparseMap, src/lidar_selection.cpp:150-168 */
void flo_visual_candidates(const flo_cam* cam, const double* Rcw, const double* Pcw, const uint8_t* img, int stride,
                           const float* world_xyz, int n, int grid_size, int border, float* map_value, int* winner);

/* ---- visual map: visible-patch selection + warp (row f2) and growth (row f4); oracle/flo_vmap.cpp -------- */
typedef struct flo_vmap flo_vmap;
flo_vmap* flo_vmap_create(const flo_cam* cam, int grid_size, double outlier_threshold, int ncc_en, double ncc_thre);
void      flo_vmap_destroy(flo_vmap*);
int       flo_vmap_counts(const flo_vmap*, int* n_points, int* n_features, int* n_images);   /* returns the grid length */
void      flo_vmap_map_value(const flo_vmap*, float* out);
/* LidarSelector::addFromSparseMap, src/lidar_selection.cpp:346-587 */
int       flo_vmap_select(flo_vmap*, const uint8_t* img, const double* Rcw, const double* Pcw, const float* pg_down, int n);
void      flo_vmap_selected(const flo_vmap*, int* index, int* point, int* search_level, float* error, double* pos, float* patch);
/* LidarSelector::addSparseMap, :142-202 */
int       flo_vmap_grow(flo_vmap*, const uint8_t* img, const double* Rcw, const double* Pcw, const float* pg, int n, int frame_id);
/* LidarSelector::addObservation, :913-965 */
int       flo_vmap_add_observations(flo_vmap*, const uint8_t* img, const double* Rcw, const double* Pcw, int frame_id);
/* pcl::VoxelGrid centroids on x, y, z (laserMapping.cpp:1398-1399; lidar_selection.cpp:351-352); returns the leaf count */
int       flo_voxel_grid(const float* xyz, int n, float leaf, float* out);
/* publish_frame_world_rgb (laserMapping.cpp:710-745): r g b per point + validity */
void      flo_colorize(const flo_cam* cam, const double* Rcw, const double* Pcw, const uint8_t* bgr, const float* xyz, int n, uint8_t* rgb,
                       uint8_t* valid);
void      flo_vmap_dump_points(const flo_vmap*, double* pos, float* value, int* n_obs, int* obs20);
void      flo_vmap_dump_features(const flo_vmap*, double* geo17, float* score, int* level_id_img);

#ifdef __cplusplus
}
#endif
#endif
