// flb_capi.cu -- the C ABI of include/fastlivo_b200.h over the sm_90a kernels.
// Host side is plain C++ (no Eigen / PCL / torch); the handle owns device memory, three streams (updates; image + patch
// copies; scan copy + ordering -- every input has two device sets, so an upload never waits for the update that is
// running: DESIGN.md section 4.8), CUDA events and an optional NCCL communicator (dlopen'ed lazily).
#include "../../include/fastlivo_b200.h"

#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "flb_kernels.cuh"
#include "flb_vmap.cuh"

using namespace flb;

static_assert(sizeof(flb_state18) == sizeof(State18), "flb_state18 and device State18 must match");
static_assert(sizeof(flb_state_ikfom) == sizeof(StateIkfom), "flb_state_ikfom and device StateIkfom must match");

namespace {

std::string g_create_error;

template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = std::max<size_t>(n, 16);
        cudaError_t e = cudaMalloc(&p, want * sizeof(T));
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

struct PinBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        cudaError_t e = cudaHostAlloc(&p, bytes, cudaHostAllocMapped);   // mapped: small kernels read / write it in place
        if (e == cudaSuccess) cap = bytes;
        return e;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
};

// Pinned staging area for host->device uploads.  An upload packs the caller's data into it and
// enqueues the copy; `done` marks that copy, and the next user of the same area waits on it (normally
// long complete), so uploads never block on the stream and the caller's buffer is free on return.
struct Staging {
    PinBuf buf;
    cudaEvent_t done = nullptr;
    bool pending = false;
    cudaError_t acquire(size_t bytes, void** out) {
        if (pending) {
            cudaError_t e = cudaEventSynchronize(done);
            if (e != cudaSuccess) return e;
            pending = false;
        }
        cudaError_t e = buf.reserve(bytes);
        if (e != cudaSuccess) return e;
        if (!done) {
            e = cudaEventCreateWithFlags(&done, cudaEventDisableTiming);
            if (e != cudaSuccess) return e;
        }
        *out = buf.p;
        return cudaSuccess;
    }
    cudaError_t mark(cudaStream_t s) {
        cudaError_t e = cudaEventRecord(done, s);
        pending = (e == cudaSuccess);
        return e;
    }
    void release() {
        if (done) cudaEventDestroy(done);
        done = nullptr;
        buf.release();
    }
};

// The visual map's coordinate limit: 2^20 voxels of its 0.5 m key on either side of the origin.
constexpr float kVmapCoordLimit = 5.0e5f;

// n caller points of `stride` floats (x, y, z first) into dst as packed xyz.
void pack_points(float* dst, const float* src, int n, int stride) {
    if (stride == 3) {
        if (n > 0) std::memcpy(dst, src, (size_t)n * 3 * sizeof(float));
        return;
    }
    for (int i = 0; i < n; ++i) {
        dst[3 * (size_t)i] = src[(size_t)i * stride];
        dst[3 * (size_t)i + 1] = src[(size_t)i * stride + 1];
        dst[3 * (size_t)i + 2] = src[(size_t)i * stride + 2];
    }
}

// Bounds lo (and, HI, hi) of n packed xyz points; true when a coordinate is non-finite.  24 floats (= 8 points) at a
// time into 24 independent accumulators: no cross-iteration dependency, so the host compiler vectorises the inner loop
// as it stands.  A NaN updates no bound; the returned flag covers it.
template <bool HI>
bool fold_points(const float* xyz, int n, float lo[3], float* hi) {
    float mn[24], mx[24];
    for (int j = 0; j < 24; ++j) { mn[j] = INFINITY; mx[j] = -INFINITY; }
    unsigned bad = 0;
    const size_t n3 = (size_t)n * 3;
    size_t i = 0;
    for (; i + 24 <= n3; i += 24)
        for (int j = 0; j < 24; ++j) {
            const float v = xyz[i + j];
            unsigned bits;
            std::memcpy(&bits, &v, sizeof(bits));
            bad |= ((bits & 0x7F800000u) == 0x7F800000u) ? 1u : 0u;
            mn[j] = v < mn[j] ? v : mn[j];
            if (HI) mx[j] = v > mx[j] ? v : mx[j];
        }
    for (; i < n3; ++i) {
        const float v = xyz[i];
        const int j = (int)(i % 24);
        bad |= std::isfinite(v) ? 0u : 1u;
        mn[j] = v < mn[j] ? v : mn[j];
        if (HI) mx[j] = v > mx[j] ? v : mx[j];
    }
    for (int k = 0; k < 3; ++k) {
        lo[k] = INFINITY;
        if (HI) hi[k] = -INFINITY;
    }
    for (int j = 0; j < 24; ++j) {
        lo[j % 3] = std::min(lo[j % 3], mn[j]);
        if (HI) hi[j % 3] = std::max(hi[j % 3], mx[j]);
    }
    return bad != 0;
}

// The first of n packed xyz points with a coordinate that is non-finite or beyond +-limit, -1 if none: the index a
// refusal names, rescanned only once a fold has found the input bad.
int first_bad_point(const float* xyz, int n, float limit) {
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < 3; ++k) {
            const float v = xyz[3 * (size_t)i + k];
            if (!std::isfinite(v) || std::fabs(v) > limit) return i;
        }
    return -1;
}

// ---- NCCL through dlopen (no link-time dependency) ----------------------------------
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(ncclUniqueId*) = nullptr;
    int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    int (*CommDestroy)(ncclComm_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load() {
        if (lib) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (lib) break;
        }
        if (!lib) return false;
        GetUniqueId = (int (*)(ncclUniqueId*))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (int (*)(ncclComm_t*, int, ncclUniqueId, int))dlsym(lib, "ncclCommInitRank");
        CommDestroy = (int (*)(ncclComm_t))dlsym(lib, "ncclCommDestroy");
        AllReduce = (int (*)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t))dlsym(lib, "ncclAllReduce");
        AllGather = (int (*)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t))dlsym(lib, "ncclAllGather");
        GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
        return GetUniqueId && CommInitRank && CommDestroy && AllReduce && AllGather;
    }
};
NcclApi g_nccl;
constexpr int kNcclInt32 = 2, kNcclFloat32 = 7, kNcclFloat64 = 8, kNcclSum = 0, kNcclMax = 2;  // ncclDataType_t / ncclRedOp_t values (nccl.h)

// flb_scan_from_undistorted's record, read back in one copy: k_cloud_pack's record of the input, k_cloud_bounds' of the
// centroids, voxel_grid_dev's box (box[6] PCL's overflow flag, box[7] the leaf count)
enum { kSfRecInput = 0, kSfRecCentroids = kScanRecWords, kSfRecBox = 2 * kScanRecWords, kSfRecWords = 2 * kScanRecWords + 8 };

}  // namespace

struct flb_handle {
    int device = 0;
    flb_config cfg{};
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    // The VIO inputs (image, patch list) are copied on a second stream so that their H2D transfer
    // overlaps the LIO kernel running on `stream`; two events order them against the VIO kernels.
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_vio_inputs = nullptr;   // recorded on copy_stream after the last image / patch copy
    cudaEvent_t ev_vio_done = nullptr;     // recorded on `stream` after the last kernel that reads them
    bool vio_inputs_pending = false, vio_done_pending = false;
    // The image and the host-built patch list are double-buffered like the scan: an upload fills the set that no kernel
    // reads (on copy_stream), then swaps it in; frame k + 1's copies (2 MB at C2) run under frame k's VIO update.
    struct InSlot {
        cudaEvent_t free_ev[2] = {nullptr, nullptr};   // [slot]: recorded on `stream` once every reader of that slot has been enqueued
        bool valid[2] = {false, false};
        int slot = 0;
    } img_slot, patch_slot;
    std::string err;
    int64_t launches = 0;

    // map
    int M = 0;
    GridDesc grid{};
    int ncell = 0;
    DevBuf<float> map_raw;
    DevBuf<unsigned> keys, keys_sorted;
    DevBuf<int> vals, vals_sorted;
    DevBuf<unsigned char> cub_tmp;
    DevBuf<float4> map_pts, map_pts_alt;       // sorted grid points (double-buffered for the incremental merge)
    DevBuf<int> cell_start, cell_start_alt;
    // sparse cell index (GridDesc), built by rebuild_grid when flb_debug_set_map_index asks for it
    bool sparse = false;
    int map_index_mode = 0;                    // 0 auto, 1 dense always, 2 sparse always (flb_debug_set_map_index)
    DevBuf<SparseCell> cell_table;             // ncell = occupied cells, grid.nx = slot mask
    DevBuf<unsigned long long> cell_keys, cell_keys_alt;   // cell key of every sorted point
    DevBuf<float> map_raw_alt;
    DevBuf<unsigned char> dead, ins;
    DevBuf<int> dead_before, merge_counts, bbox_dev;
    float map_lo[3] = {0, 0, 0}, map_hi[3] = {0, 0, 0};   // tight bounding box of the live map points
    float grid_lo[3] = {0, 0, 0}, grid_hi[3] = {0, 0, 0}; // box the kNN grid covers (= map box + a margin for growth)
    // map maintenance scratch
    DevBuf<float> map_comb, boxes;
    DevBuf<unsigned long long> vkeys, vkeys_sorted;
    DevBuf<unsigned char> keep;
    DevBuf<int> sel_idx;
    DevBuf<float> add_xyz;                     // Add_Points: the new points on the device (packed xyz, input order)
    DevBuf<unsigned> add_rec;                  // flb_map_add_scan: bounds + non-finite record (kScanRec*)
    // flb_map_fov_segment: two records; fov_rec[fov_cur].cube is the local-map cube (LocalMap_Points, Localmap_Initialized),
    // a call writes the other one and makes it current once the call has succeeded.  Allocated (zeroed) by the first call.
    DevBuf<FovRecord> fov_rec;
    int fov_cur = 0;

    // scan + per-point persistent
    int N = 0;
    DevBuf<float> scan_raw;
    DevBuf<unsigned> skeys, skeys_sorted;
    DevBuf<int> svals, svals_sorted;
    DevBuf<float4> scan;
    DevBuf<unsigned char> sel, plane_ok;
    DevBuf<float4> plane;
    // the scan is double-buffered: flb_scan_upload fills the OTHER set on `scan_stream` (copy + ordering kernel) while
    // updates already enqueued on `stream` still read this one, then swaps the two and makes `stream` wait for it
    DevBuf<float4> scan_alt, plane_alt;
    DevBuf<unsigned char> sel_alt, plane_ok_alt;
    cudaStream_t scan_stream = nullptr;
    cudaEvent_t ev_scan_ready = nullptr;
    cudaEvent_t ev_scan_free[2] = {nullptr, nullptr};   // [slot]: everything on `stream` that reads that slot has been enqueued before it
    bool scan_free_valid[2] = {false, false};
    int scan_slot = 0;
    bool scan_valid = false;                            // the current set holds an uploaded scan (not flb_voxel_grid's scratch)
    DevBuf<unsigned char> scan_cub_tmp;                 // the upload's own sort scratch (cub_tmp belongs to `stream`)
    int pers_sms = 0;                                   // SMs the persistent kernels may fill (one is left to the scan stream)
    int scan_sort_mode = 0;                             // 0 auto, 1 one-block ordering kernel, 2 device-wide sort (flb_debug_set_scan_sort)
    bool sort_attr_set[3] = {false, false, false};      // dynamic shared memory opt-in of the three k_scan_sort_block instances

    // LIO exports (lazily allocated)
    DevBuf<float> x_world, x_nn_d2, x_pd2, x_pabcd;
    DevBuf<int> x_nn_idx;
    DevBuf<unsigned char> x_rowmask;
    DevBuf<double> x_rows, x_meas;
    int last_pass_width = 0;
    bool last_pass_valid = false;

    // reductions / solve
    DevBuf<double> partials;     // max(nblocks_lio * 92, nblocks_vio * 29)
    DevBuf<double> packed;       // 128
    DevBuf<double> pose12;       // 12
    DevBuf<PriorBlock> prior;    // P11^-1 and P21*P11^-1 of the running update
    DevBuf<double> G_last;       // 108
    DevBuf<State18> states;      // [0]=x [1]=x_prop [2]=old_state(VIO) [3]=saved x [4]=saved x_prop
    DevBuf<StateIkfom> ik_states;   // [0] = x_/P_, [1] = x_propagated/P_propagated
    DevBuf<IkfomCtrl> ik_ctrl;
    int occ_ik = 0, occ_ik_sparse = 0;
    DevBuf<LioCtrl> lio_ctrl;
    DevBuf<VioCtrl> vio_ctrl;
    DevBuf<GridBarrier> barrier; // grid barrier of the persistent kernels
    DevBuf<unsigned long long> pkt;    // pose packet of the persistent kernels (kPktUnits flagged words)
    unsigned pkt_epoch = 0;            // flag base of the next launch (flags are never reused, see next_epoch)
    DevBuf<P2PLine> arrive_lines;      // persistent kernels: the worker blocks' sums of a pass, tagged with its flag
    DevBuf<unsigned long long> trace;  // [0..kTraceLen) LIO, [kTraceLen..2*kTraceLen) VIO
    DevBuf<unsigned long long> dbg;    // per-block stage stamps of the last LIO pass (tracing only)
    DevBuf<unsigned long long> dbg_vio;
    DevBuf<double> imu_buf;            // flb_imu_undistort: samples | carry | aux | poses
    DevBuf<float4> imu_pts;            // in | out
    DevBuf<int> imu_heads;
    // the output of the last successful flb_imu_undistort (feats_undistort): inside imu_pts, where depends on its point
    // count.  undist_n < 0: none (no call yet, or the last one failed)
    const float4* undist_pts = nullptr;
    int undist_n = -1;
    // flb_lidar_upload: the decoded, time-sorted cloud of the current driver message (meas.lidar) as {x, y, z, curvature}.
    // Double-buffered like the image: an upload decodes into lid_cloud_alt on copy_stream and swaps once it has
    // succeeded.  lid_n < 0: no cloud; lid_cursor: lidar_scan_index_now.  The scratch below belongs to copy_stream,
    // whose order fences its reuse.
    DevBuf<float4> lid_cloud, lid_cloud_alt;
    InSlot lid_slot;
    int lid_n = -1, lid_cursor = 0;
    DevBuf<unsigned char> lid_raw, lid_cub;    // the raw records; cub's scratch
    DevBuf<float4> lid_dec, lid_sorted;        // every record decoded; the radix sort's output
    DevBuf<int> lid_flags;                     // valid -> valid_num | kept | pos, n each; then the LidarRecord
    DevBuf<int> lid_win;                       // flb_imu_undistort_lidar: the window's point count (on `stream`)
    DevBuf<unsigned> lid_keys, lid_keys_sorted;
    DevBuf<int> lid_idx;                       // flb_lidar_upload_velodyne's yaw route: record indices, then in ring order
    DevBuf<VeloMap> lid_map;                   // its per-record time maps in ring order, scanned in place
    // flb_lidar_upload_features: the line-major points, their per-point ints (line, jump levels, scans), doubles
    // (range, dista, intersect), plane_judge results and byte flags (visited, small-plane condition)
    DevBuf<float4> feat_pts;
    DevBuf<int> feat_i;
    DevBuf<double> feat_d;
    DevBuf<FeatStep> feat_st;
    DevBuf<unsigned char> feat_u8;
    Staging st_lidar;
    PinBuf pin_lidar;
    // flb_world_cloud: pcl_wait_pub (packed xyz, the caller's order) with its exact bounds; wc_n < 0: no cloud held
    DevBuf<float> wc_xyz;
    DevBuf<unsigned> wc_rec;           // bounds + non-finite record of the transform (kScanRec*)
    int wc_n = -1;
    float wc_lo[3] = {0, 0, 0}, wc_hi[3] = {0, 0, 0};
    // flb_effect_cloud: laserCloudOri of the last LIO pass.  scan_gen counts scan installs; a pass records the generation
    // and point count of the set it ran on (ef_gen, ef_N) and is pending until captured.  The set survives one more
    // install (it becomes scan_alt), not two, nor flb_voxel_grid: then the pass is lost.  The capture keeps the rows'
    // body points (ef_body, ef_n of them, scan-index order); ef_xyz holds their world transform (ef_wn < 0: none).
    enum { kEfNone = 0, kEfPending = 1, kEfLost = 2 };
    long long scan_gen = 0, ef_gen = 0;
    int ef_state = kEfNone, ef_N = 0, ef_n = 0, ef_wn = -1;
    DevBuf<float4> ef_scatter, ef_body;
    DevBuf<unsigned char> ef_flag;
    DevBuf<int> ef_count;
    DevBuf<float> ef_xyz;
    DevBuf<unsigned> ef_rec;
    // flb_rgb_cloud: laserCloudWorldRGB as 32-byte records (rc_out, rc_n of them; rc_n < 0: none held), the per-point
    // colour words, keep flags and their exclusive sum (n + 1 each), and the caller's colour frame when it passes one.
    // Buffers of its own: the LIO export's row mask (x_rowmask) stays valid.
    DevBuf<uint4> rc_out;
    DevBuf<unsigned> rc_bgra;
    DevBuf<int> rc_flag, rc_pos;
    DevBuf<unsigned char> rc_img;
    int rc_n = -1;
    // flb_rgb_save_*: pcl_wait_save as 16-byte records in chunks of 2^kRgbChunkLog2 (rs_chunks), rs_table their pointers
    // on the device (rs_table_n entries uploaded), rs_pack the download's staging.
    bool rs_on = false;
    long long rs_max = 0, rs_n = 0, rs_dropped = 0;
    std::vector<uint4*> rs_chunks;
    size_t rs_table_n = 0;
    DevBuf<uint4*> rs_table;
    DevBuf<uint4> rs_pack;
    // flb_vmap_select_cloud: downSizeFilter of the world cloud and its scratch (the scan slot's stays untouched)
    DevBuf<float> wc_down;
    DevBuf<unsigned> wc_keys, wc_keys_sorted;
    DevBuf<int> wc_vals, wc_vals_sorted, wc_heads, wc_box;   // heads: head flags | ranks; box: k_bbox box | overflow | count
    // flb_scan_from_undistorted: downSizeFilterSurf of the undistortion output (packed input, centroids) and its scratch;
    // the scan slot's scratch stays untouched.  sf_rec: input record | centroid record (kScanRec*) | VgScratch box (kSfRec*)
    DevBuf<float> sf_xyz, sf_down;
    DevBuf<unsigned> sf_keys, sf_keys_sorted, sf_rec;
    DevBuf<int> sf_vals, sf_vals_sorted, sf_heads;
    DevBuf<unsigned long long> vm_key;   // flb_visual_candidates: per-cell {score, ~index}
    DevBuf<float> vm_val, vm_pts;
    DevBuf<int> vm_win;
    DevBuf<double> vm_pose;
    int dbg_vio_blocks = 0;
    int dbg_blocks = 0;
    bool tracing = false;
    int num_sms = 0;
    int occ_lio = 0, occ_lio_sparse = 0, occ_vio = 0;
    Staging st_map, st_scan, st_img, st_patch, st_state, st_misc;   // per-kind upload staging
    PinBuf pin_out;              // staging for downloads
    PinBuf pin_res[2];           // flb_state_download_enqueue / _wait: two result slots in flight
    cudaEvent_t ev_res[2] = {nullptr, nullptr};
    bool res_pending[2] = {false, false};
    bool state_valid = false;
    // device-side state moves that the next persistent kernel performs itself instead of a separate D2D copy
    bool reset_pending = false;   // flb_state_reset_enqueue: x, x_prop := the saved pair
    bool prior_pending = false;   // flb_state_set_prior_enqueue: x_prop := x

    // VIO inputs
    int img_w = 0, img_h = 0;
    DevBuf<unsigned char> img, img_alt;
    // a set's colour frame (img_rgb, W x H x 3) beside its gray image: flb_image_upload_bgr fills both, flb_image_upload
    // only the gray one (img_bgr_valid = false); the two swap together
    DevBuf<unsigned char> img_bgr, img_bgr_alt;
    bool img_bgr_valid = false;
    // flb_image_upload_bgr's raw frame on the device.  Its H2D copy and k_image_prep, its only reader, both run on
    // copy_stream, so the next frame's copy into it is ordered after that kernel: stream order is its reuse fence.
    DevBuf<unsigned char> img_raw;
    int Pn = 0;
    DevBuf<double> patch_pos, patch_pos_alt;
    DevBuf<float> patch_ref, patch_ref_alt;
    DevBuf<int> patch_level, patch_level_alt;
    DevBuf<float> errors;        // 2 x err_stride (local shard; the persistent kernel's passes alternate between the halves)
    DevBuf<unsigned long long> err_units;   // 2 x err_stride {tag : error} units (persistent kernel, single GPU: what its leader polls)
    int err_stride = 0;
    DevBuf<float> errors_all;    // padded shard * world (multi-GPU)
    DevBuf<double> x_z, x_H;
    bool cam_set = false;
    CamModel cam{};

    bool last_vio_valid = false;

    // device-resident visual map (rows f2 / f4)
    struct Vm {
        bool on = false;
        VmParams prm{};
        double Rci_Pci[12] = {0};            // camera <- IMU extrinsic (LidarSelector::init, :44-45)
        DevBuf<VmPoint> pts;
        DevBuf<VmFeature> fts;
        DevBuf<unsigned char> pool;          // keyframe images, pool_slots x (w * h)
        int pool_slots = 0;
        int pts_ub = 0, fts_ub = 0, img_ub = 0;   // host-side upper bounds of the device counters (img_ub: slots in use)
        // flb_vmap_reclaim (allocated by its first call): the compaction target (swapped with fts), the free-slot stack of
        // the pool, scratch for the feature ranks (fts.cap + 1) and the slot flags / ranks (3 x pool_slots), cub's scan scratch
        DevBuf<VmFeature> fts_alt;
        DevBuf<int> free_slots, rc_rank, rc_slot;
        DevBuf<unsigned char> rc_cub;
        size_t rc_cub_bytes = 0;
        DevBuf<int> counters;
        DevBuf<double> pose, rci;            // T_f_w of the current frame (12) ; Rci | Pci (12)
        DevBuf<float> pg;                    // scan points of the current call
        DevBuf<unsigned long long> depth, keyset, cell_best, cand_key;
        unsigned key_mask = 0;
        DevBuf<unsigned char> cell_type;
        DevBuf<float> map_value, cell_err, cell_patch, sel_error;
        DevBuf<int> cell_flag, cell_rank, cell_level, cell_point, sel_index, sel_point, winner, scan_tmp;
        Staging st_pg;
    } vm;
    bool pn_on_device = false;   // the patch list was built on the device (flb_vmap_select without a count readback)
    bool patches_set = false;    // a patch list exists (flb_patches_upload or a visual-map selection)
    // sub_sparse_map->errors still holds the selection's errors (vm.sel_error, :576): no VIO pass has run on the list
    bool err_from_sel = false;
    // flb_keypatch_image: the owner of each pixel (W x H) and the annotated frame (W x H x 3)
    DevBuf<int> kp_owner;
    DevBuf<unsigned char> kp_out;

    // batched frames (SURVEY.md section 7 H2(iv)): B independent frames per launch, all against the handle's map
    struct Batch {
        int B = 0, n_max = 0, n_cap = 0;
        std::vector<int> N;                  // points per frame
        DevBuf<float4> scan, plane;          // B x n_cap
        DevBuf<unsigned char> sel, plane_ok;
        DevBuf<double> partials;             // B x max(nb_lio * 29, nb_vio * 29)
        size_t partials_per = 0;
        DevBuf<State18> states;              // B x {x, x_prop, old_state, saved x, saved x_prop}
        DevBuf<LioCtrl> lio_ctrl;
        DevBuf<VioCtrl> vio_ctrl;
        DevBuf<PriorBlock> prior;
        DevBuf<double> G_last;               // B x 108
        DevBuf<float> errors;                // B x 2 x err_stride
        DevBuf<LioArgs> lio_args;
        DevBuf<LioSolveArgs> lio_solve;
        DevBuf<VioArgs> vio_args;
        DevBuf<VioSolveArgs> vio_solve;
        DevBuf<LioCtrl*> lio_ctrl_ptrs;
        DevBuf<VioCtrl*> vio_ctrl_ptrs;
    } batch;

    // multi-GPU
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;
    int err_shard = 0;           // max patches per rank (equal-size ncclAllGather shards)
    // fused NVLink exchange (persistent kernels, no NCCL in the data path)
    DevBuf<P2PMailbox> mailbox;
    DevBuf<unsigned long long> p2p_seq;
    P2PArgs p2p{};               // world <= 1: not attached
    void* p2p_peer_ptr[kP2PMaxWorld] = {nullptr};

    // profiling
    bool profiling = false;
    struct Ev { cudaEvent_t a, b; int fam; };
    std::vector<Ev> evs;
};

namespace {

int fail(flb_handle* h, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    else g_create_error = buf;
    return code;
}

#define FLB_CUDA(h, expr)                                                                         \
    do {                                                                                          \
        cudaError_t _e = (expr);                                                                  \
        if (_e != cudaSuccess)                                                                    \
            return fail(h, FLB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

#define FLB_CHECK_H(h)                                   \
    do {                                                 \
        if (!(h)) return FLB_ERR_INVALID;                \
        cudaError_t _e = cudaSetDevice((h)->device);     \
        if (_e != cudaSuccess) return fail(h, FLB_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(_e)); \
    } while (0)

// launch bookkeeping: count every kernel; when profiling, bracket it with an event pair
struct LaunchScope {
    flb_handle* h;
    int fam;
    cudaEvent_t a = nullptr, b = nullptr;
    LaunchScope(flb_handle* h_, int fam_) : h(h_), fam(fam_) {
        h->launches++;
        if (h->profiling) {
            cudaEventCreate(&a);
            cudaEventCreate(&b);
            cudaEventRecord(a, h->stream);
        }
    }
    ~LaunchScope() {
        if (h->profiling) {
            cudaEventRecord(b, h->stream);
            h->evs.push_back({a, b, fam});
        }
    }
};
enum { FAM_LIO_KNN = 0, FAM_LIO_PLAIN = 1, FAM_VIO = 2, FAM_SOLVE = 3, FAM_OTHER = 4 };
constexpr int kVioErrCapMax = 40960;     // floats of dynamic shared memory (160 KB) for the VIO leader's error staging

void to_dev_params(const flb_lio_params* p, LioParamsDev& d) {
    std::memcpy(d.R_LI, p->R_LI, sizeof(d.R_LI));
    std::memcpy(d.t_LI, p->t_LI, sizeof(d.t_LI));
    d.sigma = p->laser_point_cov;
    d.max_iteration = p->max_iteration;
    d.conv_rot_deg = p->conv_rot_deg;
    d.conv_pos_cm = p->conv_pos_cm;
}

// LidarSelector::init() constants, src/lidar_selection.cpp:41-52 + set_extrinsic :35-39 (host, once per call)
void to_dev_params(const flb_vio_params* p, VioParamsDev& d) {
    double Rli[9], Pli[3], t[3];
    m3_T(p->R_LI, Rli);
    m3_vec(Rli, p->t_LI, t);
    for (int i = 0; i < 3; ++i) Pli[i] = -t[i];
    m3_mul(p->Rcl, Rli, d.Rci);
    m3_vec(p->Rcl, Pli, t);
    for (int i = 0; i < 3; ++i) d.Pci[i] = t[i] + p->Pcl[i];
    vio_pose_constants(d.Rci, d.Pci, d.Jdphi_dR, d.Jdp_dR);
    d.sigma = p->img_point_cov;
    d.max_iteration = p->max_iteration;
    d.conv_rot_deg = p->conv_rot_deg;
    d.conv_pos_cm = p->conv_pos_cm;
    d.force_all_passes = p->force_all_passes;
    d.single_level = 0;
}

int lio_nblocks(const flb_handle* h) { return (h->N + kLioBlock - 1) / kLioBlock; }
int vio_nblocks(const flb_handle* h) { return (h->Pn + (kVioBlock / 32) - 1) / (kVioBlock / 32); }

int ensure_common(flb_handle* h) {
    FLB_CUDA(h, h->packed.reserve(128));
    FLB_CUDA(h, h->pose12.reserve(12));
    FLB_CUDA(h, h->prior.reserve(1));
    FLB_CUDA(h, h->G_last.reserve(108));
    FLB_CUDA(h, h->states.reserve(5));
    FLB_CUDA(h, h->lio_ctrl.reserve(1));
    FLB_CUDA(h, h->vio_ctrl.reserve(1));
    FLB_CUDA(h, h->barrier.reserve(1));
    FLB_CUDA(h, h->trace.reserve(2 * kTraceLen));
    FLB_CUDA(h, cudaMemset(h->trace.p, 0, 2 * kTraceLen * sizeof(unsigned long long)));
    FLB_CUDA(h, cudaMemset(h->barrier.p, 0, sizeof(GridBarrier)));
    FLB_CUDA(h, h->pkt.reserve(kPktUnits));
    FLB_CUDA(h, cudaMemset(h->pkt.p, 0, kPktUnits * sizeof(unsigned long long)));
    FLB_CUDA(h, cudaMemset(h->lio_ctrl.p, 0, sizeof(LioCtrl)));
    FLB_CUDA(h, cudaMemset(h->vio_ctrl.p, 0, sizeof(VioCtrl)));
    FLB_CUDA(h, cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, h->device));
    {
        // the per-frame persistent kernels fill all SMs but one: the next frame's scan ordering (one block on `scan_stream`)
        // runs there concurrently.  FLB_RESERVE_SM=0 gives that SM back (A/B measurement).
        static const int env_reserve = [] { const char* e = getenv("FLB_RESERVE_SM"); return e ? atoi(e) : 1; }();
        h->pers_sms = (env_reserve && h->num_sms > 2) ? h->num_sms - 1 : h->num_sms;
    }
    FLB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ_lio, k_lio_update_persistent<kLioPersBlock, false>, kLioPersBlock, 0));
    FLB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ_lio_sparse, k_lio_update_persistent<kLioPersBlock, true>, kLioPersBlock, 0));
    FLB_CUDA(h, h->ik_states.reserve(2));
    FLB_CUDA(h, h->ik_ctrl.reserve(1));
    FLB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ_ik, k_lio_update_ikfom_persistent<kLioBlock, false>, kLioBlock, 0));
    FLB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ_ik_sparse, k_lio_update_ikfom_persistent<kLioBlock, true>, kLioBlock, 0));
    // the VIO leader stages the per-patch errors of a pass in dynamic shared memory (up to kVioErrCapMax floats)
    FLB_CUDA(h, cudaFuncSetAttribute(k_vio_update_persistent<kVioPersBlock>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     kVioErrCapMax * (int)sizeof(float)));
    FLB_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ_vio, k_vio_update_persistent<kVioPersBlock>, kVioPersBlock,
                                                             kVioErrCapMax * sizeof(float)));
    FLB_CUDA(h, h->pin_out.reserve(1 << 16));
    return FLB_OK;
}

// the cell index the kNN reads: dense cell_start, or the sparse table (GridDesc)
const int* cell_index(const flb_handle* h) {
    return h->sparse ? reinterpret_cast<const int*>(h->cell_table.p) : h->cell_start.p;
}
size_t index_bytes(const flb_handle* h) {
    return h->sparse ? ((size_t)(unsigned)h->grid.nx + 1) * sizeof(SparseCell) : ((size_t)h->ncell + 1) * sizeof(int);
}

// The device buffers of one frame that the update kernels read and write: the handle's own (handle_frame), or frame i's
// slice of the batch buffers (flb_batch_update_enqueue).
struct FrameBufs {
    const float4* scan;
    int N;
    State18* states;             // x, x_prop, old_state (VIO), saved x, saved x_prop
    LioCtrl* lio_ctrl;
    VioCtrl* vio_ctrl;
    PriorBlock* prior;
    unsigned char* sel;
    float4* plane;
    unsigned char* plane_ok;
    double* partials;
    float* errors;
    int err_stride;
    double* G_last;
};

FrameBufs handle_frame(flb_handle* h) {
    return {h->scan.p, h->N, h->states.p, h->lio_ctrl.p, h->vio_ctrl.p, h->prior.p, h->sel.p, h->plane.p, h->plane_ok.p,
            h->partials.p, h->errors.p, h->err_stride, h->G_last.p};
}

// The argument blocks of the update kernels.  Each builder sets the fields every caller sets alike; a field that one
// path alone sets is set at its call site.
LioArgs make_lio_args(flb_handle* h, const LioParamsDev& prm, const FrameBufs& fb) {
    LioArgs a{};
    a.scan = fb.scan;
    a.N = fb.N;
    a.grid = h->grid;
    a.cell_start = cell_index(h);
    a.map_pts = h->map_pts.p;
    a.state = fb.states;
    a.prm = prm;
    a.plane_thr = (float)h->cfg.plane_threshold;
    a.ctrl = fb.lio_ctrl;
    a.force_rematch = -1;
    a.sel = fb.sel;
    a.plane = fb.plane;
    a.plane_ok = fb.plane_ok;
    a.partials = fb.partials;
    a.M = h->M;
    return a;
}

LioSolveArgs make_lio_solve_args(flb_handle* h, const LioParamsDev& prm, const FrameBufs& fb) {
    LioSolveArgs s{};
    s.state = fb.states;
    s.state_prop = fb.states + 1;
    s.ctrl = fb.lio_ctrl;
    s.prior = fb.prior;
    s.partials = fb.partials;
    s.nblocks = (fb.N + kLioBlock - 1) / kLioBlock;
    s.prm = prm;
    s.timeout_flag = &h->barrier.p->timeout;
    return s;
}

VioArgs make_vio_args(flb_handle* h, const VioParamsDev& prm, const FrameBufs& fb) {
    VioArgs a{};
    a.img = h->img.p;
    a.cam = h->cam;
    a.pos = h->patch_pos.p;
    a.patch = h->patch_ref.p;
    a.search_level = h->patch_level.p;
    a.Pn = h->Pn;
    a.state = fb.states;
    a.prm = prm;
    a.ctrl = fb.vio_ctrl;
    a.force_level = -1;
    a.errors = fb.errors;
    a.err_stride = fb.err_stride;
    a.partials = fb.partials;
    return a;
}

VioSolveArgs make_vio_solve_args(flb_handle* h, const VioParamsDev& prm, const FrameBufs& fb) {
    VioSolveArgs s{};
    s.state = fb.states;
    s.state_prop = fb.states + 1;
    s.old_state = fb.states + 2;
    s.ctrl = fb.vio_ctrl;
    s.prior = fb.prior;
    s.G_last = fb.G_last;
    s.partials = fb.partials;
    s.nblocks = vio_nblocks(h);
    s.errors = fb.errors;
    s.err_stride = fb.err_stride;
    s.Pn_total = h->Pn;
    s.prm = prm;
    s.timeout_flag = &h->barrier.p->timeout;
    return s;
}

// (R, p) as 12 doubles at `dst` on the device, through the misc staging area in stream order
int upload_pose(flb_handle* h, double* dst, const double* R, const double* p) {
    void* stv = nullptr;
    FLB_CUDA(h, h->st_misc.acquire(12 * sizeof(double), &stv));
    double* st = static_cast<double*>(stv);
    std::memcpy(st, R, 9 * sizeof(double));
    std::memcpy(st + 9, p, 3 * sizeof(double));
    FLB_CUDA(h, cudaMemcpyAsync(dst, st, 12 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_misc.mark(h->stream));
    return FLB_OK;
}

// The packed sums of one pass: HTH's upper triangle row by row (written out symmetric, width x width), then the
// right-hand side (width)
void unpack_normal_eq(const double* po, int width, double* HTH, double* rhs) {
    int k = 0;
    for (int r = 0; r < width; ++r)
        for (int c = r; c < width; ++c) {
            HTH[r * width + c] = po[k];
            HTH[c * width + r] = po[k];
            ++k;
        }
    for (int r = 0; r < width; ++r) rhs[r] = po[k + r];
}

// Every caller that reads the image needs a camera and an image of the camera's size.
int vio_image_check(flb_handle* h, const char* who) {
    if (!h->cam_set || h->img_w <= 0) return fail(h, FLB_ERR_STATE, "%s: camera and image must be set first", who);
    if (h->cam.width != h->img_w || h->cam.height != h->img_h) return fail(h, FLB_ERR_STATE, "camera / image size mismatch");
    return FLB_OK;
}

int launch_lio_pass(flb_handle* h, const LioArgs& a, int width, bool knn_family) {
    const int nb = lio_nblocks(h);
    if (nb == 0) return FLB_OK;
    LaunchScope ls(h, knn_family ? FAM_LIO_KNN : FAM_LIO_PLAIN);
    if (h->sparse) {
        if (width == 6) k_lio_pass<6, kLioBlock, true><<<nb, kLioBlock, 0, h->stream>>>(a);
        else k_lio_pass<12, kLioBlock, true><<<nb, kLioBlock, 0, h->stream>>>(a);
    } else {
        if (width == 6) k_lio_pass<6, kLioBlock, false><<<nb, kLioBlock, 0, h->stream>>>(a);
        else k_lio_pass<12, kLioBlock, false><<<nb, kLioBlock, 0, h->stream>>>(a);
    }
    FLB_CUDA(h, cudaGetLastError());
    return FLB_OK;
}

// all-reduce of the packed sums (and all-gather of the per-patch errors) for multi-GPU
int allreduce_packed(flb_handle* h, const double* partials, int nblocks, int K) {
    {
        LaunchScope ls(h, FAM_SOLVE);
        k_reduce_only<<<1, 32, 0, h->stream>>>(partials, nblocks, K, h->packed.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    int r = g_nccl.AllReduce(h->packed.p, h->packed.p, (size_t)K, kNcclFloat64, kNcclSum, h->comm, h->stream);
    if (r != 0) return fail(h, FLB_ERR_COMM, "ncclAllReduce: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    h->launches++;
    return FLB_OK;
}

// The kernel-per-pass VIO update: up to `passes` rounds of k_vio_pass then k_vio_finalize; the kernels return at once
// when the update (or the level) has ended.
int vio_pass_loop(flb_handle* h, const VioArgs& a, VioSolveArgs s, int passes) {
    const int nb = vio_nblocks(h);
    for (int it = 0; it < passes && h->Pn > 0; ++it) {
        {
            LaunchScope ls(h, FAM_VIO);
            k_vio_pass<kVioBlock><<<nb, kVioBlock, 0, h->stream>>>(a);
            FLB_CUDA(h, cudaGetLastError());
        }
        if (h->comm) {
            int rc = allreduce_packed(h, h->partials.p, nb, kVioPacked);
            if (rc) return rc;
            s.partials = h->packed.p;
            s.nblocks = 1;
            // gather every rank's per-patch errors in patch order (shards padded to errors.cap/world)
            const size_t shard = (size_t)h->err_shard;
            int r = g_nccl.AllGather(h->errors.p, h->errors_all.p, shard, kNcclFloat32, h->comm, h->stream);
            if (r != 0) return fail(h, FLB_ERR_COMM, "ncclAllGather failed");
            h->launches++;
            s.errors = h->errors_all.p;
            s.Pn_total = (int)(shard * (size_t)h->world);
        }
        LaunchScope ls(h, FAM_SOLVE);
        k_vio_finalize<<<1, kLeaderBlock, 0, h->stream>>>(s);
        FLB_CUDA(h, cudaGetLastError());
    }
    return FLB_OK;
}

// true when p is page-locked host memory (flb_host_alloc / cudaHostAlloc / cudaHostRegister): the copy engine
// can read it directly, so the staging memcpy is skipped
bool is_pinned(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// copy_stream is about to fill the OTHER set of a double-buffered input.  Every reader of the current set has been
// enqueued on `stream` by now (record its event); the other set's readers were all enqueued before the previous upload,
// whose event the copy waits for.
int vio_copy_begin(flb_handle* h, flb_handle::InSlot& s) {
    for (int k = 0; k < 2; ++k)
        if (!s.free_ev[k]) FLB_CUDA(h, cudaEventCreateWithFlags(&s.free_ev[k], cudaEventDisableTiming));
    FLB_CUDA(h, cudaEventRecord(s.free_ev[s.slot], h->stream));
    s.valid[s.slot] = true;
    if (s.valid[s.slot ^ 1]) FLB_CUDA(h, cudaStreamWaitEvent(h->copy_stream, s.free_ev[s.slot ^ 1], 0));
    return FLB_OK;
}
int vio_copy_end(flb_handle* h) {
    FLB_CUDA(h, cudaEventRecord(h->ev_vio_inputs, h->copy_stream));
    h->vio_inputs_pending = true;
    return FLB_OK;
}
// a kernel on `stream` is about to read the image / patches
int vio_inputs_acquire(flb_handle* h) {
    if (h->vio_inputs_pending) {
        FLB_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_vio_inputs, 0));
        h->vio_inputs_pending = false;
    }
    return FLB_OK;
}

// The camera-size outputs of image_upload_frame from the dense frame `src` (packed encoding ENC) on copy_stream.
template <int ENC>
void launch_image_out(flb_handle* h, const unsigned char* src, int width, int height, int gray_rule) {
    const int W = h->cam.width, H = h->cam.height;
    const unsigned rows = (unsigned)std::min(H, 65535);
    const dim3 grid4((unsigned)((W + 4 * 128 - 1) / (4 * 128)), rows);
    const bool vec = (W % 4) == 0;
    if (width == W && height == H) {
        if (vec) k_image_prep<false, true, ENC><<<grid4, 128, 0, h->copy_stream>>>(src, W, H, gray_rule, h->img_bgr_alt.p, h->img_alt.p);
        else k_image_prep<false, false, ENC><<<grid4, 128, 0, h->copy_stream>>>(src, W, H, gray_rule, h->img_bgr_alt.p, h->img_alt.p);
    } else if (width == 2 * W && height == 2 * H) {
        if (vec) k_image_prep<true, true, ENC><<<grid4, 128, 0, h->copy_stream>>>(src, W, H, gray_rule, h->img_bgr_alt.p, h->img_alt.p);
        else k_image_prep<true, false, ENC><<<grid4, 128, 0, h->copy_stream>>>(src, W, H, gray_rule, h->img_bgr_alt.p, h->img_alt.p);
    } else {
        const dim3 grid((unsigned)((W + 127) / 128), rows);
        k_image_resize_linear<ENC><<<grid, 128, 0, h->copy_stream>>>(src, width, height, W, H, gray_rule, h->img_bgr_alt.p, h->img_alt.p);
    }
}

// flb_image_upload_bgr / flb_image_upload_msg once their arguments are checked: the frame (width x height pixels of
// `encoding`, step_bytes a row) into the idle image set as the camera-size colour frame and gray image.  The frame's
// rows go up dense into img_raw, a Bayer mosaic behind the room for its demosaiced BGR8 frame, which k_bayer_bgr fills
// before the outputs are made from it.  The copy and every kernel run on copy_stream, so stream order fences img_raw's
// reuse by the next frame.
int image_upload_frame(flb_handle* h, const uint8_t* src, int width, int height, int step_bytes, int encoding, int gray_rule) {
    const int W = h->cam.width, H = h->cam.height;
    const bool bayer = encoding >= kEncBayerRggb8;
    const size_t row = (size_t)width * enc_bpp(encoding), raw_bytes = row * height, px = (size_t)W * H;
    const size_t decoded = bayer ? (size_t)width * height * 3 : 0;
    FLB_CUDA(h, h->img_raw.reserve(decoded + raw_bytes));
    FLB_CUDA(h, h->img_alt.reserve(px));
    FLB_CUDA(h, h->img_bgr_alt.reserve(px * 3));
    unsigned char* raw = h->img_raw.p + decoded;
    // the raw frame goes up before the wait for the idle set's readers: only the kernel that writes the set waits for them
    if (is_pinned(src)) {
        FLB_CUDA(h, cudaMemcpy2DAsync(raw, row, src, step_bytes, row, height, cudaMemcpyHostToDevice, h->copy_stream));
    } else {
        void* stv = nullptr;
        FLB_CUDA(h, h->st_img.acquire(raw_bytes, &stv));
        unsigned char* st = static_cast<unsigned char*>(stv);
        if ((size_t)step_bytes == row) std::memcpy(st, src, raw_bytes);
        else for (int r = 0; r < height; ++r) std::memcpy(st + (size_t)r * row, src + (size_t)r * step_bytes, row);
        FLB_CUDA(h, cudaMemcpyAsync(raw, st, raw_bytes, cudaMemcpyHostToDevice, h->copy_stream));
        FLB_CUDA(h, h->st_img.mark(h->copy_stream));
    }
    if (bayer) {
        const dim3 grid((unsigned)((width + 127) / 128), (unsigned)std::min(height, 65535));
        k_bayer_bgr<<<grid, 128, 0, h->copy_stream>>>(raw, width, height, encoding, h->img_raw.p);
        FLB_CUDA(h, cudaGetLastError());
        h->launches++;
    }
    { int rcq = vio_copy_begin(h, h->img_slot); if (rcq) return rcq; }
    switch (bayer ? (int)kEncBgr8 : encoding) {
        case kEncRgb8: launch_image_out<kEncRgb8>(h, raw, width, height, gray_rule); break;
        case kEncMono8: launch_image_out<kEncMono8>(h, raw, width, height, gray_rule); break;
        case kEncBgra8: launch_image_out<kEncBgra8>(h, raw, width, height, gray_rule); break;
        case kEncRgba8: launch_image_out<kEncRgba8>(h, raw, width, height, gray_rule); break;
        default: launch_image_out<kEncBgr8>(h, h->img_raw.p, width, height, gray_rule); break;
    }
    FLB_CUDA(h, cudaGetLastError());
    h->launches++;
    { int rcq = vio_copy_end(h); if (rcq) return rcq; }
    std::swap(h->img, h->img_alt);
    std::swap(h->img_bgr, h->img_bgr_alt);
    h->img_bgr_valid = true;
    h->img_slot.slot ^= 1;
    h->img_w = W;
    h->img_h = H;
    h->last_vio_valid = false;
    return FLB_OK;
}

// Perform the deferred device-side state moves with plain copies (every consumer other than the persistent kernels).
int flush_state_ops(flb_handle* h) {
    if (h->reset_pending) {
        FLB_CUDA(h, cudaMemcpyAsync(&h->states.p[0], &h->states.p[3], 2 * sizeof(State18), cudaMemcpyDeviceToDevice, h->stream));
        h->reset_pending = false;
    }
    if (h->prior_pending) {
        FLB_CUDA(h, cudaMemcpyAsync(&h->states.p[1], &h->states.p[0], sizeof(State18), cudaMemcpyDeviceToDevice, h->stream));
        h->prior_pending = false;
    }
    return FLB_OK;
}

// A LIO pass was enqueued on the current scan set: its sel bytes (lio_sel_byte) are laserCloudOri until captured.
void note_lio_pass(flb_handle* h) {
    h->ef_state = flb_handle::kEfPending;
    h->ef_gen = h->scan_gen;
    h->ef_N = h->N;
}

// flb_rgb_save_end / flb_destroy: the save's chunks, table and staging (cudaFree waits for the kernels that use them).
void rgb_save_free(flb_handle* h) {
    for (uint4* c : h->rs_chunks) cudaFree(c);
    h->rs_chunks.clear();
    h->rs_table_n = 0;
    h->rs_table.release();
    h->rs_pack.release();
    h->rs_on = false;
    h->rs_max = h->rs_n = h->rs_dropped = 0;
}

// Flag base for one persistent launch: flags epoch+1 .. epoch+4095 belong to it alone.  On wrap-around the
// packet and the arrival lines are cleared (stream-ordered) so that no stale unit can ever match.
int next_epoch(flb_handle* h, unsigned* epoch) {
    if (h->pkt_epoch >= 0xFFFF0000u || h->pkt_epoch == 0) {
        if (h->pkt_epoch) {
            FLB_CUDA(h, cudaMemsetAsync(h->pkt.p, 0, kPktUnits * sizeof(unsigned long long), h->stream));
            if (h->arrive_lines.p)
                FLB_CUDA(h, cudaMemsetAsync(h->arrive_lines.p, 0, h->arrive_lines.cap * sizeof(P2PLine), h->stream));
        }
        h->pkt_epoch = 4096;
    }
    *epoch = h->pkt_epoch;
    h->pkt_epoch += 4096;
    return FLB_OK;
}

// Arrival by lines (kernels: "Arrival by lines"): grid x 29 lines, shared by the LIO and VIO launches (their flags
// differ).  Zeroed when allocated and, by next_epoch, when the flags wrap.  *lines = null selects the counter path:
// FLB_LL_ARRIVE=0 (A/B measurement).
int arrive_lines(flb_handle* h, int grid, P2PLine** lines) {
    static const int env = [] { const char* e = getenv("FLB_LL_ARRIVE"); return e ? atoi(e) : 1; }();
    *lines = nullptr;
    if (!env) return FLB_OK;
    const size_t need = (size_t)grid * std::max(lio_packed(6), kVioPacked);
    if (need > h->arrive_lines.cap) {
        FLB_CUDA(h, h->arrive_lines.reserve(need));
        FLB_CUDA(h, cudaMemsetAsync(h->arrive_lines.p, 0, h->arrive_lines.cap * sizeof(P2PLine), h->stream));
    }
    *lines = h->arrive_lines.p;
    return FLB_OK;
}

int enqueue_lio_update(flb_handle* h, const flb_lio_params* prm) {
    // fused multi-GPU mode: a rank whose shard is empty still launches (its leader takes part in every exchange)
    if (h->M <= 0 || (h->N <= 0 && !(h->p2p.world > 1 && h->scan.p)))
        return fail(h, FLB_ERR_STATE, "flb_lio_update: map and scan must be uploaded first");
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_lio_update: no device state (flb_state_upload)");
    if (prm->max_iteration < 0 || prm->max_iteration > 1000) return fail(h, FLB_ERR_INVALID, "max_iteration outside [0, 1000]");
    if (h->p2p.world > 1 && !h->cfg.persistent)
        return fail(h, FLB_ERR_STATE, "the fused NVLink exchange lives in the persistent kernels (flb_config.persistent = 1)");
    LioParamsDev d;
    to_dev_params(prm, d);
    const FrameBufs fb = handle_frame(h);
    LioSolveArgs s = make_lio_solve_args(h, d, fb);
    s.p2p = h->p2p;
    LioArgs a = make_lio_args(h, d, fb);
    const bool lio_persistent = h->cfg.persistent && (!h->comm || h->p2p.world > 1);
    if (h->prior_pending || (h->reset_pending && !lio_persistent)) { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    if (h->reset_pending) {              // the kernel starts from the saved pair and restores state / state_prop itself
        s.init_x = &h->states.p[3];
        s.init_xp = &h->states.p[4];
        h->reset_pending = false;
    }
    if (lio_persistent) {
        // one cooperative launch for the whole iterated update; grid = min(needed, co-resident capacity)
        // whole multiples of the SM count (<= co-resident capacity): chunks are dealt round-robin to blocks
        // worker blocks (one per SM, chunks dealt round-robin) + one leader block
        const int cap = std::min((h->sparse ? h->occ_lio_sparse : h->occ_lio) * h->num_sms, h->pers_sms);
        if (cap < 2) return fail(h, FLB_ERR_STATE, "persistent mode needs two co-resident blocks");
        const int workers = std::max(1, std::min((h->N + 31) / 32, cap - 1));
        const int grid = workers + 1;
        FLB_CUDA(h, h->partials.reserve(std::max<size_t>((size_t)grid * lio_packed(12), h->partials.cap)));
        a.partials = h->partials.p;
        s.partials = h->partials.p;
        s.nblocks = workers;
        { int rcl = arrive_lines(h, grid, &s.lines); if (rcl) return rcl; }
        GridBarrier* bar = h->barrier.p;
        unsigned long long* trace = h->tracing ? h->trace.p : nullptr;
        a.probe = h->tracing ? h->trace.p + 112 : nullptr;
        a.chunk = std::max(1, std::min(32, (h->N + workers * (kLioPersBlock / 32) - 1) / (workers * (kLioPersBlock / 32))));
        {
            static const int env_warm = [] { const char* e = getenv("FLB_WARM"); return e ? atoi(e) : 1; }();
            if (env_warm) {
                WarmList& w = a.warm;
                const size_t n1 = (size_t)std::max(h->N, 1);
                const void* sums = s.lines ? (const void*)s.lines : (const void*)h->partials.p;
                const void* ptr[] = {h->scan.p, h->map_pts.p, cell_index(h), h->plane.p, h->sel.p, h->plane_ok.p, sums, h->states.p};
                const size_t len[] = {n1 * 16, (size_t)h->M * 16, index_bytes(h), n1 * 16, n1, n1,
                                      (size_t)grid * lio_packed(6) * (s.lines ? sizeof(P2PLine) : 8), 5 * sizeof(State18)};
                w.n = 8;
                for (int k = 0; k < 8; ++k) { w.p[k] = ptr[k]; w.bytes[k] = len[k]; }
            }
        }
        {
            // L2 prefetch of the map (points + cell table) at kernel start: on by default above 1 MB (H100, FLB_PREFETCH=0 vs 1,
            // device-resident frames/s: C2 (5.3 MB) 5505 -> 5557, C3 (27 MB) 1502 -> 1515, C4 2557 -> 2568); FLB_PREFETCH=0/1 overrides
            const size_t bytes = (size_t)h->M * 16 + index_bytes(h);
            static const int env = [] { const char* e = getenv("FLB_PREFETCH"); return e ? atoi(e) : -1; }();
            a.prefetch = env >= 0 ? env : (bytes > (1u << 20) ? 1 : 0);
        }
        unsigned long long* dbg = nullptr;
        if (h->tracing) {
            FLB_CUDA(h, h->dbg.reserve((size_t)grid * 16));
            FLB_CUDA(h, cudaMemsetAsync(h->dbg.p, 0, (size_t)grid * 16 * sizeof(unsigned long long), h->stream));
            h->dbg_blocks = grid;
            dbg = h->dbg.p;
        }
        unsigned long long* pkt = h->pkt.p;
        unsigned epoch = 0;
        { int rce = next_epoch(h, &epoch); if (rce) return rce; }
        void* args[] = {&a, &s, &bar, &pkt, &epoch, &trace, &dbg};
        LaunchScope ls(h, FAM_LIO_KNN);
        void* kern = h->sparse ? (void*)k_lio_update_persistent<kLioPersBlock, true> : (void*)k_lio_update_persistent<kLioPersBlock, false>;
        FLB_CUDA(h, cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kLioPersBlock), args, 0,
                                                h->stream));
        h->last_pass_valid = false;
        note_lio_pass(h);
        return FLB_OK;
    }
    {
        LaunchScope ls(h, FAM_SOLVE);
        k_lio_begin<<<1, 32, 0, h->stream>>>(h->lio_ctrl.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    const int T = prm->max_iteration;
    for (int it = -1; it < T; ++it) {
        // Statically known rematch schedule when early stop is disabled is NOT assumed here:
        // the kernel reads ctrl->nearest_search_en / ctrl->stop on the device.
        int rc = launch_lio_pass(h, a, 6, it == -1);
        if (rc) return rc;
        if (h->comm) {
            rc = allreduce_packed(h, h->partials.p, lio_nblocks(h), lio_packed(6));
            if (rc) return rc;
            s.partials = h->packed.p;
            s.nblocks = 1;
        }
        LaunchScope ls(h, FAM_SOLVE);
        k_lio_finalize<<<1, kLeaderBlock, 0, h->stream>>>(s);
        FLB_CUDA(h, cudaGetLastError());
    }
    h->last_pass_valid = false;
    note_lio_pass(h);                    // the passes after the stop pass return at once: its sel bytes stay
    return FLB_OK;
}

// The patch list of the last flb_vmap_select lives on the device; calls that need its length on the host fetch it here.
int resolve_pn(flb_handle* h) {
    if (!h->pn_on_device) return FLB_OK;
    int n = 0;
    FLB_CUDA(h, cudaMemcpyAsync(&n, h->vm.counters.p + VM_N_SEL, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    h->Pn = n;
    h->pn_on_device = false;
    return FLB_OK;
}

int enqueue_vio_update(flb_handle* h, const flb_vio_params* prm) {
    { int rc = vio_image_check(h, "flb_vio_update"); if (rc) return rc; }
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_vio_update: no device state (flb_state_upload)");
    if (prm->max_iteration > 1000) return fail(h, FLB_ERR_INVALID, "max_iteration outside [0, 1000]");
    if (h->pn_on_device && !(h->cfg.persistent && h->p2p.world <= 1 && !h->comm && prm->max_iteration > 0)) {
        int rcp = resolve_pn(h);             // only the single-GPU persistent kernel reads the count on the device
        if (rcp) return rcp;
    }
    VioParamsDev d;
    to_dev_params(prm, d);
    const FrameBufs fb = handle_frame(h);
    VioSolveArgs s = make_vio_solve_args(h, d, fb);
    s.p2p = h->p2p;
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    const bool fused = h->p2p.world > 1;
    if (fused && !h->cfg.persistent)
        return fail(h, FLB_ERR_STATE, "the fused NVLink exchange lives in the persistent kernels (flb_config.persistent = 1)");
    if (fused && h->Pn > kP2PErrCap) return fail(h, FLB_ERR_INVALID, "fused multi-GPU mode: at most %d patches per rank", kP2PErrCap);
    const bool persistent = h->cfg.persistent && (fused || (!h->comm && (h->Pn > 0 || h->pn_on_device))) && prm->max_iteration > 0;
    if (h->reset_pending || (h->prior_pending && !persistent)) { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    if (h->prior_pending) {              // the kernel takes state_propagat = state itself
        s.prior_from_state = 1;
        h->prior_pending = false;
    }
    if (!persistent) {
        LaunchScope ls(h, FAM_SOLVE);
        k_vio_begin<<<1, 32, 0, h->stream>>>(h->vio_ctrl.p, h->Pn);
        FLB_CUDA(h, cudaGetLastError());
    }
    if (prm->max_iteration > 0) h->err_from_sel = false;        // the passes below write sub_sparse_map->errors (:851)
    VioArgs a = make_vio_args(h, d, fb);
    a.p2p = h->p2p;
    if (h->pn_on_device) {                   // capacity = one patch per grid cell; the kernel reads the real count
        a.Pn = h->vm.prm.length;
        a.Pn_dev = h->vm.counters.p + VM_N_SEL;
        s.Pn_total = a.Pn;
    }
    static const int env_defer = [] { const char* e = getenv("FLB_DEFER"); return e ? atoi(e) : 1; }();
    if (persistent && !fused && env_defer) {
        // per-patch errors as self-validating units (zeroed once per allocation: a tag always has its top bit set)
        const size_t need = 2 * (size_t)std::max(h->err_stride, 1);
        if (need > h->err_units.cap) {
            FLB_CUDA(h, h->err_units.reserve(need));
            FLB_CUDA(h, cudaMemsetAsync(h->err_units.p, 0, h->err_units.cap * sizeof(unsigned long long), h->stream));
        }
        a.err_units = h->err_units.p;
        s.err_units = h->err_units.p;
    }
    if (persistent) {
        // patches are dealt warp-round-robin over the worker blocks; one more block is the leader
        const int cap = std::min(h->occ_vio * h->num_sms, h->pers_sms);
        if (cap < 2) return fail(h, FLB_ERR_STATE, "persistent mode needs two co-resident blocks");
        const int workers = std::max(1, std::min(std::max(a.Pn, 1), cap - 1));
        const int grid = workers + 1;
        FLB_CUDA(h, h->partials.reserve(std::max<size_t>((size_t)grid * kVioPacked, h->partials.cap)));
        a.partials = h->partials.p;
        s.partials = h->partials.p;
        s.nblocks = workers;
        // plain per-patch errors (FLB_DEFER=0, single GPU) are ordered for the leader only by the counter: keep it
        if (fused || s.err_units) { int rcl = arrive_lines(h, grid, &s.lines); if (rcl) return rcl; }
        GridBarrier* bar = h->barrier.p;
        unsigned long long* trace = h->tracing ? h->trace.p + kTraceLen : nullptr;
        unsigned long long* pkt = h->pkt.p;
        unsigned epoch = 0;
        { int rce = next_epoch(h, &epoch); if (rce) return rce; }
        unsigned long long* dbg = nullptr;
        if (h->tracing) {
            FLB_CUDA(h, h->dbg_vio.reserve((size_t)grid * kVioDbg));
            FLB_CUDA(h, cudaMemsetAsync(h->dbg_vio.p, 0, (size_t)grid * kVioDbg * sizeof(unsigned long long), h->stream));
            dbg = h->dbg_vio.p;
            h->dbg_vio_blocks = grid;
        }
        // staging capacity for the errors of ALL ranks (the peers' shard sizes are not known here: assume like ours + slack)
        int err_cap = (int)std::min<long long>(kVioErrCapMax, std::max<long long>(2048, ((long long)a.Pn * std::max(h->p2p.world, 1) * 5 / 4 + 319) / 256 * 256));
        {
            static const int env_warm = [] { const char* e = getenv("FLB_WARM"); return e ? atoi(e) : 1; }();
            if (env_warm) {
                WarmList& w = a.warm;
                const size_t pn = (size_t)std::max(a.Pn, 1);
                const void* sums = s.lines ? (const void*)s.lines : (const void*)h->partials.p;
                const void* ptr[] = {h->img.p, h->patch_pos.p, h->patch_ref.p, h->patch_level.p, h->errors.p, sums};
                const size_t len[] = {(size_t)h->img_w * h->img_h, pn * 24, pn * 768, pn * 4, 2 * (size_t)h->err_stride * 4,
                                      (size_t)grid * kVioPacked * (s.lines ? sizeof(P2PLine) : 8)};
                w.n = 6;
                for (int k = 0; k < 6; ++k) { w.p[k] = ptr[k]; w.bytes[k] = len[k]; }
            }
        }
        const size_t dyn = (size_t)err_cap * sizeof(float);
        void* args[] = {&a, &s, &bar, &pkt, &epoch, &trace, &dbg, &err_cap};
        LaunchScope ls(h, FAM_VIO);
        FLB_CUDA(h, cudaLaunchCooperativeKernel((void*)k_vio_update_persistent<kVioPersBlock>, dim3(grid), dim3(kVioPersBlock), args, dyn,
                                                h->stream));
        h->last_vio_valid = false;
        return FLB_OK;
    }
    { int rc = vio_pass_loop(h, a, s, 3 * std::max(prm->max_iteration, 0)); if (rc) return rc; }
    h->last_vio_valid = false;
    return FLB_OK;
}

void fill_lio_report(const LioCtrl& c, flb_lio_report* rep) {
    rep->passes = c.passes;
    rep->knn_passes = c.knn_passes;
    rep->n_eff_last = c.n_eff_last;
    rep->res_mean_last = c.res_mean_last;
    rep->rows_total = c.rows_total;
    rep->converged_last = c.converged_last;
    rep->status = c.status;
}
void fill_vio_report(const VioCtrl& c, flb_vio_report* rep) {
    for (int l = 0; l < 3; ++l) { rep->passes[l] = c.passes[l]; rep->last_error[l] = c.level_error[l]; }
    rep->rows_total = c.rows_total;
    rep->skipped_last = c.skipped_last;
    rep->cov_updated = c.cov_updated;
    rep->status = c.status;
}

// A persistent kernel whose grid barrier timed out has set GridBarrier::timeout.  `bar` is the barrier as read back:
// when it is set, clear the device barrier for the next launch and report the timeout.
int watchdog_check(flb_handle* h, const char* bar) {
    GridBarrier b;
    std::memcpy(&b, bar, sizeof(b));
    if (!b.timeout) return FLB_OK;
    cudaMemset(h->barrier.p, 0, sizeof(GridBarrier));
    return fail(h, FLB_ERR_TIMEOUT, "device-side grid barrier watchdog tripped");
}

// The result block {State18, LioCtrl, VioCtrl, GridBarrier} as flb_state_download and k_pack_result lay it out.
constexpr size_t kResLio = sizeof(State18), kResVio = kResLio + sizeof(LioCtrl), kResBarrier = kResVio + sizeof(VioCtrl);
constexpr size_t kResBytes = kResBarrier + sizeof(GridBarrier);

int read_result(flb_handle* h, const char* po, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio) {
    { int rc = watchdog_check(h, po + kResBarrier); if (rc) return rc; }
    if (x) std::memcpy(x, po, sizeof(State18));
    if (lio) { LioCtrl c; std::memcpy(&c, po + kResLio, sizeof(c)); fill_lio_report(c, lio); }
    if (vio) { VioCtrl c; std::memcpy(&c, po + kResVio, sizeof(c)); fill_vio_report(c, vio); }
    return FLB_OK;
}

}  // namespace

template <int kScanSortBlock, int ITEMS>
static int launch_scan_sort_block(flb_handle* h, cudaStream_t ss, const float* xyz, int N, const float lo[3], float inv_cell) {
    using Sort = cub::BlockRadixSort<unsigned, kScanSortBlock, ITEMS, int, 6>;
    const size_t smem = std::max(sizeof(typename Sort::TempStorage), (size_t)kScanSortBlock * ITEMS * sizeof(unsigned));
    bool& attr_set = h->sort_attr_set[ITEMS == 17 ? 0 : (ITEMS == 33 ? 1 : 2)];      // per handle: the attribute is per device
    if (!attr_set) {
        FLB_CUDA(h, cudaFuncSetAttribute(k_scan_sort_block<kScanSortBlock, ITEMS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    k_scan_sort_block<kScanSortBlock, ITEMS><<<1, kScanSortBlock, smem, ss>>>(xyz, N, lo[0], lo[1], lo[2], inv_cell, h->scan_alt.p, h->sel_alt.p,
                                                             h->plane_ok_alt.p);
    FLB_CUDA(h, cudaGetLastError());
    return FLB_OK;
}

extern "C" {

int flb_abi_version(void) { return FLB_ABI_VERSION; }

const char* flb_last_error(const flb_handle* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int flb_create(const flb_config* cfg, flb_handle** out) {
    if (!out) return FLB_ERR_INVALID;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, FLB_ERR_NO_DEVICE,
                    "no CUDA device (%s): fastlivo_b200 has no CPU fallback", e == cudaSuccess ? "count = 0" : cudaGetErrorString(e));
    flb_config c{};
    c.persistent = 1;
    if (cfg) c = *cfg;
    if (c.device < 0 || c.device >= ndev) return fail(nullptr, FLB_ERR_INVALID, "device %d out of range [0,%d)", c.device, ndev);
    if (!(c.cell_size > 0)) c.cell_size = 0.6;
    if (!(c.knn_max_d2 > 0)) c.knn_max_d2 = 5.0;
    if (!(c.plane_threshold > 0)) c.plane_threshold = 0.1;
    e = cudaSetDevice(c.device);
    if (e != cudaSuccess) return fail(nullptr, FLB_ERR_CUDA, "cudaSetDevice(%d): %s", c.device, cudaGetErrorString(e));
    flb_handle* h = new flb_handle;
    h->device = c.device;
    h->cfg = c;
    e = cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        delete h;
        return fail(nullptr, FLB_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e));
    }
    h->stream = h->own_stream;
    if (cudaStreamCreateWithFlags(&h->scan_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_scan_ready, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_scan_free[0], cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_scan_free[1], cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_vio_inputs, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&h->ev_vio_done, cudaEventDisableTiming) != cudaSuccess) {
        cudaStreamDestroy(h->own_stream);
        delete h;
        return fail(nullptr, FLB_ERR_CUDA, "copy stream / event creation failed");
    }
    int rc = ensure_common(h);
    if (rc) {
        g_create_error = h->err;
        cudaStreamDestroy(h->own_stream);
        delete h;
        return rc;
    }
    *out = h;
    return FLB_OK;
}

int flb_destroy(flb_handle* h) {
    if (!h) return FLB_OK;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    for (int r = 0; r < kP2PMaxWorld; ++r)
        if (h->p2p_peer_ptr[r]) cudaIpcCloseMemHandle(h->p2p_peer_ptr[r]);
    h->mailbox.release();
    h->p2p_seq.release();
    {
        auto& b = h->batch;
        b.scan.release(); b.plane.release(); b.sel.release(); b.plane_ok.release(); b.partials.release(); b.states.release();
        b.lio_ctrl.release(); b.vio_ctrl.release(); b.prior.release(); b.G_last.release(); b.errors.release(); b.lio_args.release();
        b.lio_solve.release(); b.vio_args.release(); b.vio_solve.release(); b.lio_ctrl_ptrs.release(); b.vio_ctrl_ptrs.release();
    }
    {
        auto& vm = h->vm;
        vm.pts.release(); vm.fts.release(); vm.pool.release(); vm.counters.release(); vm.pose.release(); vm.rci.release(); vm.pg.release();
        vm.depth.release(); vm.keyset.release(); vm.cell_best.release(); vm.cand_key.release(); vm.cell_type.release(); vm.map_value.release();
        vm.cell_err.release(); vm.cell_patch.release(); vm.sel_error.release(); vm.cell_flag.release(); vm.cell_rank.release();
        vm.cell_level.release(); vm.cell_point.release(); vm.sel_index.release(); vm.sel_point.release(); vm.winner.release();
        vm.scan_tmp.release(); vm.st_pg.release();
        vm.fts_alt.release(); vm.free_slots.release(); vm.rc_rank.release(); vm.rc_slot.release(); vm.rc_cub.release();
    }
    for (auto& ev : h->evs) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    h->map_raw.release(); h->keys.release(); h->keys_sorted.release(); h->vals.release(); h->vals_sorted.release();
    h->map_comb.release(); h->boxes.release(); h->vkeys.release(); h->vkeys_sorted.release(); h->keep.release(); h->sel_idx.release();
    h->add_xyz.release(); h->add_rec.release(); h->fov_rec.release();
    h->wc_xyz.release(); h->wc_rec.release(); h->wc_down.release(); h->wc_keys.release(); h->wc_keys_sorted.release();
    h->wc_vals.release(); h->wc_vals_sorted.release(); h->wc_heads.release(); h->wc_box.release();
    h->ef_scatter.release(); h->ef_body.release(); h->ef_flag.release(); h->ef_count.release(); h->ef_xyz.release(); h->ef_rec.release();
    h->rc_out.release(); h->rc_bgra.release(); h->rc_flag.release(); h->rc_pos.release(); h->rc_img.release();
    rgb_save_free(h);
    h->sf_keys.release(); h->sf_keys_sorted.release(); h->sf_rec.release(); h->sf_vals.release(); h->sf_vals_sorted.release();
    h->sf_heads.release(); h->sf_xyz.release();
    h->cell_table.release(); h->cell_keys.release(); h->cell_keys_alt.release();
    h->map_pts_alt.release(); h->cell_start_alt.release(); h->map_raw_alt.release(); h->dead.release(); h->ins.release();
    h->dead_before.release(); h->merge_counts.release(); h->bbox_dev.release();
    h->cub_tmp.release(); h->map_pts.release(); h->cell_start.release(); h->scan.release(); h->sel.release();
    h->plane_ok.release(); h->plane.release(); h->x_world.release(); h->x_nn_d2.release(); h->x_pd2.release();
    h->x_nn_idx.release(); h->x_rowmask.release(); h->x_rows.release(); h->x_meas.release(); h->partials.release();
    h->packed.release(); h->pose12.release(); h->prior.release(); h->scan_raw.release(); h->skeys.release(); h->skeys_sorted.release(); h->svals.release(); h->svals_sorted.release(); h->x_pabcd.release(); h->G_last.release(); h->states.release();
    h->lio_ctrl.release(); h->vio_ctrl.release(); h->ik_states.release(); h->ik_ctrl.release(); h->barrier.release(); h->pkt.release(); h->arrive_lines.release(); h->trace.release(); h->dbg.release(); h->dbg_vio.release(); h->imu_buf.release(); h->imu_pts.release(); h->imu_heads.release(); h->vm_key.release(); h->vm_val.release(); h->vm_pts.release(); h->vm_win.release(); h->vm_pose.release(); h->img.release(); h->img_bgr.release(); h->img_bgr_alt.release(); h->img_raw.release(); h->patch_pos.release(); h->patch_ref.release();
    h->patch_level.release(); h->kp_owner.release(); h->kp_out.release(); h->errors.release(); h->err_units.release(); h->errors_all.release(); h->x_z.release(); h->x_H.release();
    h->st_map.release(); h->st_scan.release(); h->st_img.release(); h->st_patch.release(); h->st_state.release();
    h->st_misc.release(); h->pin_out.release();
    for (int k = 0; k < 2; ++k) { h->pin_res[k].release(); if (h->ev_res[k]) cudaEventDestroy(h->ev_res[k]); }
    cudaStreamSynchronize(h->copy_stream);
    cudaStreamSynchronize(h->scan_stream);
    h->scan_alt.release(); h->plane_alt.release(); h->sel_alt.release(); h->plane_ok_alt.release(); h->sf_down.release();
    h->lid_cloud.release(); h->lid_cloud_alt.release(); h->lid_raw.release(); h->lid_cub.release(); h->lid_dec.release();
    h->lid_sorted.release(); h->lid_flags.release(); h->lid_win.release(); h->lid_keys.release(); h->lid_keys_sorted.release();
    h->lid_idx.release(); h->lid_map.release();
    h->st_lidar.release(); h->pin_lidar.release();
    h->img_alt.release(); h->patch_pos_alt.release(); h->patch_ref_alt.release(); h->patch_level_alt.release();
    for (int k = 0; k < 2; ++k) {
        if (h->img_slot.free_ev[k]) cudaEventDestroy(h->img_slot.free_ev[k]);
        if (h->patch_slot.free_ev[k]) cudaEventDestroy(h->patch_slot.free_ev[k]);
        if (h->lid_slot.free_ev[k]) cudaEventDestroy(h->lid_slot.free_ev[k]);
    }
    cudaEventDestroy(h->ev_scan_ready);
    cudaEventDestroy(h->ev_scan_free[0]);
    cudaEventDestroy(h->ev_scan_free[1]);
    h->scan_cub_tmp.release();
    cudaStreamDestroy(h->scan_stream);
    cudaEventDestroy(h->ev_vio_inputs);
    cudaEventDestroy(h->ev_vio_done);
    cudaStreamDestroy(h->copy_stream);
    cudaStreamDestroy(h->own_stream);
    delete h;
    return FLB_OK;
}

int flb_set_stream(flb_handle* h, void* cuda_stream) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    h->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
    return FLB_OK;
}

int flb_synchronize(flb_handle* h) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->copy_stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->scan_stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_host_alloc(flb_handle* h, size_t bytes, void** out) {
    FLB_CHECK_H(h);
    if (!out || bytes == 0) return fail(h, FLB_ERR_INVALID, "flb_host_alloc: bad arguments");
    FLB_CUDA(h, cudaHostAlloc(out, bytes, cudaHostAllocDefault));
    return FLB_OK;
}

int flb_host_free(flb_handle* h, void* p) {
    FLB_CHECK_H(h);
    if (p) FLB_CUDA(h, cudaFreeHost(p));
    return FLB_OK;
}

int64_t flb_launch_count(const flb_handle* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------
constexpr int kDenseCellCap = 1 << 25;      // largest dense cell table (cells); beyond it the cell is enlarged

// Hash table of the occupied cells of the sorted key array h->cell_keys[0..M): >= 2x as many slots as cells.
static int build_sparse_table(flb_handle* h, int M) {
    FLB_CUDA(h, h->merge_counts.reserve(2));
    FLB_CUDA(h, cudaMemsetAsync(h->merge_counts.p, 0, sizeof(int), h->stream));
    const int nb = (M + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_sparse_count_cells<<<nb, 256, 0, h->stream>>>(h->cell_keys.p, M, h->merge_counts.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    int occupied = 0;
    FLB_CUDA(h, cudaMemcpyAsync(&occupied, h->merge_counts.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    size_t slots = 16;
    while (slots < 2 * (size_t)occupied) slots <<= 1;
    FLB_CUDA(h, h->cell_table.reserve(slots));
    FLB_CUDA(h, cudaMemsetAsync(h->cell_table.p, 0xff, slots * sizeof(SparseCell), h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_sparse_insert<<<nb, 256, 0, h->stream>>>(h->cell_keys.p, M, h->cell_table.p, (unsigned)(slots - 1));
        FLB_CUDA(h, cudaGetLastError());
        h->launches++;
    }
    h->grid.nx = (int)(slots - 1);
    h->ncell = occupied;
    return FLB_OK;
}

// Sparse cell index over h->map_raw[0..M): anchored where the dense grid would be (h->grid_lo), at the configured cell.
static int rebuild_sparse(flb_handle* h, int M) {
    GridDesc g{};
    g.ox = h->grid_lo[0]; g.oy = h->grid_lo[1]; g.oz = h->grid_lo[2];
    g.cell = (float)h->cfg.cell_size;
    g.inv_cell = 1.0f / g.cell;
    g.max_d2 = (float)h->cfg.knn_max_d2;
    g.max_ring = (int)std::ceil(std::sqrt(h->cfg.knn_max_d2) / h->cfg.cell_size) + 1;
    FLB_CUDA(h, h->vkeys.reserve(M));
    FLB_CUDA(h, h->cell_keys.reserve(M));
    FLB_CUDA(h, h->vals.reserve(M));
    FLB_CUDA(h, h->vals_sorted.reserve(M));
    FLB_CUDA(h, h->map_pts.reserve(M));
    const int nb = (M + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_sparse_cell_keys<<<nb, 256, 0, h->stream>>>(h->map_raw.p, M, g, h->vkeys.p, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    size_t tmp_bytes = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, h->vkeys.p, h->cell_keys.p, h->vals.p, h->vals_sorted.p, M, 0, 63,
                                                h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, tmp_bytes, h->vkeys.p, h->cell_keys.p, h->vals.p, h->vals_sorted.p, M, 0,
                                                63, h->stream));
    h->launches += 4;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_map_gather<<<nb, 256, 0, h->stream>>>(h->map_raw.p, M, 3, h->vals_sorted.p, h->map_pts.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    h->grid = g;
    h->sparse = true;
    h->M = M;
    return build_sparse_table(h, M);
}

// Build the sorted uniform kNN grid over h->map_raw[0..M) with the bounding box h->map_lo/hi.
static int rebuild_grid(flb_handle* h, int M) {
    // the grid covers the map box plus a margin, so that points added next to the map (a moving sensor) fall inside
    // it and take the incremental path of flb_map_add_points; kNN is exact for any cell geometry
    for (int k = 0; k < 3; ++k) {
        // a whole number of cells, so that the cell boundaries stay where a grid anchored at the map's own corner puts them
        const float cs = (float)h->cfg.cell_size;
        const float m = cs * std::ceil(std::max(2.0f * cs, 0.05f * (h->map_hi[k] - h->map_lo[k])) / cs);
        h->grid_lo[k] = h->map_lo[k] - m;
        h->grid_hi[k] = h->map_hi[k] + m;
    }
    const float* lo = h->grid_lo;
    const float* hi = h->grid_hi;
    // dense table or sparse index.  The automatic choice is the dense table at every extent: measured on H100
    // (DESIGN.md section 8) the sparse index beats the coarsened dense grid at a 3 km map but not at 1 km, so it is only
    // taken when flb_debug_set_map_index asks for it (and the box fits the cell keys)
    if (h->map_index_mode == 2) {
        double span = 0.0;
        for (int k = 0; k < 3; ++k) span = std::max(span, (double)(hi[k] - lo[k]) / h->cfg.cell_size);
        if (span < (double)(kCellKeyBias - 1)) return rebuild_sparse(h, M);
    }
    h->sparse = false;
    // grid geometry; enlarge the cell if the dense grid would exceed kDenseCellCap cells (still exact, just slower)
    double cell = h->cfg.cell_size;
    for (;;) {
        const double nx = std::floor((hi[0] - lo[0]) / cell) + 1, ny = std::floor((hi[1] - lo[1]) / cell) + 1,
                     nz = std::floor((hi[2] - lo[2]) / cell) + 1;
        if (nx * ny * nz <= (double)kDenseCellCap) break;
        cell *= 1.26;
    }
    GridDesc g{};
    g.ox = lo[0]; g.oy = lo[1]; g.oz = lo[2];
    g.cell = (float)cell;
    g.inv_cell = 1.0f / g.cell;
    g.nx = (int)std::floor((hi[0] - lo[0]) / cell) + 1;
    g.ny = (int)std::floor((hi[1] - lo[1]) / cell) + 1;
    g.nz = (int)std::floor((hi[2] - lo[2]) / cell) + 1;
    g.max_d2 = (float)h->cfg.knn_max_d2;
    g.max_ring = (int)std::ceil(std::sqrt(h->cfg.knn_max_d2) / cell) + 1;
    const int ncell = g.nx * g.ny * g.nz;
    FLB_CUDA(h, h->keys.reserve(M));
    FLB_CUDA(h, h->keys_sorted.reserve(M));
    FLB_CUDA(h, h->vals.reserve(M));
    FLB_CUDA(h, h->vals_sorted.reserve(M));
    FLB_CUDA(h, h->map_pts.reserve(M));
    FLB_CUDA(h, h->cell_start.reserve((size_t)ncell + 1));
    const int nb = (M + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_map_cell_ids<<<nb, 256, 0, h->stream>>>(h->map_raw.p, M, 3, g, h->keys.p, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    int end_bit = 1;
    while ((1u << end_bit) < (unsigned)ncell && end_bit < 32) ++end_bit;
    size_t tmp_bytes = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, h->keys.p, h->keys_sorted.p, h->vals.p, h->vals_sorted.p, M,
                                                0, end_bit, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, tmp_bytes, h->keys.p, h->keys_sorted.p, h->vals.p,
                                                h->vals_sorted.p, M, 0, end_bit, h->stream));
    h->launches += 4;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_map_gather<<<nb, 256, 0, h->stream>>>(h->map_raw.p, M, 3, h->vals_sorted.p, h->map_pts.p);
        k_cell_starts<<<(ncell + 256) / 256, 256, 0, h->stream>>>(h->keys_sorted.p, M, h->cell_start.p, ncell);
        FLB_CUDA(h, cudaGetLastError());
        h->launches++;
    }
    h->M = M;
    h->grid = g;
    h->ncell = ncell;
    return FLB_OK;
}

int flb_map_upload(flb_handle* h, const float* xyz, int M, int stride) {
    FLB_CHECK_H(h);
    if (!xyz || M < 1 || stride < 3) return fail(h, FLB_ERR_INVALID, "flb_map_upload: bad arguments (M=%d stride=%d)", M, stride);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    void* stv = nullptr;
    FLB_CUDA(h, h->st_map.acquire((size_t)M * 3 * sizeof(float), &stv));
    float* st = static_cast<float*>(stv);
    pack_points(st, xyz, M, stride);
    float lo[3], hi[3];
    if (fold_points<true>(st, M, lo, hi))
        return fail(h, FLB_ERR_INVALID, "flb_map_upload: non-finite coordinate at point %d", first_bad_point(st, M, INFINITY));
    for (int k = 0; k < 3; ++k) { h->map_lo[k] = lo[k]; h->map_hi[k] = hi[k]; }
    FLB_CUDA(h, h->map_raw.reserve((size_t)M * 3));
    FLB_CUDA(h, cudaMemcpyAsync(h->map_raw.p, st, (size_t)M * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    int rc = rebuild_grid(h, M);
    if (rc) return rc;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

// ---- device-resident map maintenance (SURVEY.md section 8 row f1) -----------------------------------
// Compact h->map_comb by h->keep flags (positions given by idx_in) into map_raw, then rebuild the grid.
static int compact_and_rebuild(flb_handle* h, const int* idx_in, int total) {
    FLB_CUDA(h, h->sel_idx.reserve((size_t)total + 1));
    size_t tmp_bytes = 0;
    int* d_count = h->sel_idx.p + total;
    FLB_CUDA(h, cub::DeviceSelect::Flagged(nullptr, tmp_bytes, idx_in, h->keep.p, h->sel_idx.p, d_count, total, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    FLB_CUDA(h, cub::DeviceSelect::Flagged(h->cub_tmp.p, tmp_bytes, idx_in, h->keep.p, h->sel_idx.p, d_count, total, h->stream));
    h->launches += 2;
    int count = 0;
    FLB_CUDA(h, cudaMemcpyAsync(&count, d_count, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (count < 1) return fail(h, FLB_ERR_STATE, "map maintenance would leave an empty map");
    FLB_CUDA(h, h->map_raw.reserve((size_t)count * 3));   // never shrinks; grows only if count > capacity
    FLB_CUDA(h, h->bbox_dev.reserve(6));
    const int init[6] = {0x7fffffff, 0x7fffffff, 0x7fffffff, (int)0x80000000, (int)0x80000000, (int)0x80000000};
    FLB_CUDA(h, cudaMemcpyAsync(h->bbox_dev.p, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_gather_xyz<<<(count + 255) / 256, 256, 0, h->stream>>>(h->map_comb.p, h->sel_idx.p, count, h->map_raw.p);
        k_bbox<<<std::min((count + 255) / 256, 4 * std::max(h->num_sms, 1)), 256, 0, h->stream>>>(h->map_raw.p, count, h->bbox_dev.p);
        FLB_CUDA(h, cudaGetLastError());
        h->launches++;
    }
    // the box follows the LIVE points: it shrinks when Delete_Point_Boxes drops the part of the map the sensor left
    int box[6];
    FLB_CUDA(h, cudaMemcpyAsync(box, h->bbox_dev.p, sizeof(box), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int k = 0; k < 6; ++k) {
        const int b = box[k] >= 0 ? box[k] : (box[k] ^ 0x7fffffff);
        float f;
        std::memcpy(&f, &b, sizeof(f));
        (k < 3 ? h->map_lo[k] : h->map_hi[k - 3]) = f;
    }
    return rebuild_grid(h, count);
}

// Full path of Add_Points: (existing + new) points sorted by downsample voxel, one thread per voxel, compaction, grid
// rebuilt from scratch.  Taken when a new point lies outside the box the kNN grid covers (the grid has to grow).
static int map_add_points_full(flb_handle* h, const float* nxyz, int n, float downsample_size) {
    const int M = h->M, total = M + n;
    FLB_CUDA(h, h->map_comb.reserve((size_t)total * 3));
    FLB_CUDA(h, h->vkeys.reserve(total));
    FLB_CUDA(h, h->vkeys_sorted.reserve(total));
    FLB_CUDA(h, h->vals.reserve(total));
    FLB_CUDA(h, h->vals_sorted.reserve(total));
    FLB_CUDA(h, h->keep.reserve(total));
    FLB_CUDA(h, cudaMemcpyAsync(h->map_comb.p, h->map_raw.p, (size_t)M * 3 * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    // The new points arrive in add_xyz (both entry points fill it before the path is known), so this path -- the rare one,
    // whose cost is the radix sort of all M + n points -- pays one n x 12 B device-to-device copy to put them behind the map.
    FLB_CUDA(h, cudaMemcpyAsync(h->map_comb.p + (size_t)M * 3, nxyz, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    const int nb = (total + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vox_keys<<<nb, 256, 0, h->stream>>>(h->map_comb.p, total, downsample_size, h->vkeys.p, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    size_t tmp_bytes = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, h->vkeys.p, h->vkeys_sorted.p, h->vals.p, h->vals_sorted.p, total,
                                                0, 63, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, tmp_bytes, h->vkeys.p, h->vkeys_sorted.p, h->vals.p, h->vals_sorted.p,
                                                total, 0, 63, h->stream));
    h->launches += 4;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vox_resolve<<<nb, 256, 0, h->stream>>>(h->vkeys_sorted.p, h->vals_sorted.p, h->map_comb.p, total, M, downsample_size,
                                                  h->keep.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    return compact_and_rebuild(h, h->vals_sorted.p, total);
}

static int bits_for(long long span) {
    int b = 1;
    while ((1ll << b) <= span) ++b;
    return b;
}

}  // extern "C"

// The merge of the incremental Add_Points and of the cube delete, once h->dead[0..M) flags the points that go (sorted
// order) and, for n new points in nxyz, ins_keys / ins_vals hold their cell keys sorted ("no cell" for the ones not
// inserted) and their indices.  Survivors keep their order, inserts go behind their cell's survivors, the _alt buffers
// become the map; the dense table merges its cell_start, the sparse index rebuilds its hash table from the merged keys.
// The grid box, the dense table's geometry and the sparse index's anchor stay as they are.  map_raw becomes the sorted
// order, so map indices still refer to flb_map_download's array.  n = 0 (a delete): the caller knows the number of
// flagged points, n_del, and the counts are not read back; only the sparse table rebuild reads its cell count.
template <bool SPARSE>
static int map_merge(flb_handle* h, const float* nxyz, int n, const CellKey<SPARSE>* ins_keys, const int* ins_vals, int n_del) {
    const int M = h->M, ncell = h->ncell, gm = (M + 255) / 256;
    FLB_CUDA(h, h->dead_before.reserve((size_t)M + 1));
    FLB_CUDA(h, h->merge_counts.reserve(2));
    FLB_CUDA(h, h->map_pts_alt.reserve((size_t)M + n));
    FLB_CUDA(h, h->map_raw_alt.reserve(((size_t)M + n) * 3));
    if constexpr (SPARSE) FLB_CUDA(h, h->cell_keys_alt.reserve((size_t)M + n));
    else FLB_CUDA(h, h->cell_start_alt.reserve((size_t)ncell + 1));
    size_t tmp_bytes = 0;
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, h->dead_before.p, h->dead_before.p, M, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_dead_to_int<<<gm, 256, 0, h->stream>>>(h->dead.p, M, h->dead_before.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(h->cub_tmp.p, tmp_bytes, h->dead_before.p, h->dead_before.p, M, h->stream));
    h->launches += 2;
    {
        LaunchScope ls(h, FAM_OTHER);
        const CellKey<SPARSE>* keys_old = nullptr;
        CellKey<SPARSE>* keys_new = nullptr;
        if constexpr (SPARSE) {
            keys_old = h->cell_keys.p;
            keys_new = h->cell_keys_alt.p;
        }
        k_merge_counts<SPARSE><<<1, 32, 0, h->stream>>>(h->dead_before.p, h->dead.p, M, ins_keys, n, ncell, h->merge_counts.p);
        if constexpr (!SPARSE) {
            k_merge_cell_starts<<<(ncell + 256) / 256, 256, 0, h->stream>>>(h->cell_start.p, h->dead_before.p, h->merge_counts.p, M,
                                                                             ins_keys, n, ncell, h->cell_start_alt.p);
            h->launches++;
        }
        k_merge_existing<SPARSE><<<gm, 256, 0, h->stream>>>(h->map_pts.p, keys_old, h->dead.p, h->dead_before.p, M, h->grid, ins_keys,
                                                            n, h->map_pts_alt.p, h->map_raw_alt.p, keys_new);
        h->launches++;
        if (n > 0) {
            k_merge_inserts<SPARSE><<<(n + 255) / 256, 256, 0, h->stream>>>(nxyz, ins_keys, ins_vals, h->merge_counts.p, h->cell_start.p,
                                                                            keys_old, h->dead_before.p, M, h->map_pts_alt.p,
                                                                            h->map_raw_alt.p, keys_new);
            h->launches++;
        }
        FLB_CUDA(h, cudaGetLastError());
    }
    int counts[2] = {n_del, 0};                       // dead points, inserted points
    if (n > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(counts, h->merge_counts.p, sizeof(counts), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    std::swap(h->map_pts, h->map_pts_alt);
    std::swap(h->map_raw, h->map_raw_alt);
    h->M = M - counts[0] + counts[1];
    h->last_pass_valid = false;
    if constexpr (SPARSE) {
        std::swap(h->cell_keys, h->cell_keys_alt);
        return build_sparse_table(h, h->M);
    } else {
        std::swap(h->cell_start, h->cell_start_alt);
        return FLB_OK;
    }
}

// Incremental Add_Points: the new points sorted by downsample voxel, one thread per touched voxel resolves it against
// the live points (k_vox_resolve_incremental), the inserted points sorted by cell key, then map_merge.  The voxel keys
// are packed into as few bits as their box needs (fewer radix passes): on the dense table the grid box, which every new
// point lies in (else the full path runs); on the sparse index, which has no box to leave, the new points' own box,
// with absolute 21-bit keys if that box needs more than 62 bits.  Nothing on the sparse index scales with the extent.
template <bool SPARSE>
static int map_add_points_inc(flb_handle* h, const float* nxyz, int n, float ds, const float* lo, const float* hi) {
    const int M = h->M;
    const GridDesc g = h->grid;
    const float* klo = SPARSE ? lo : h->grid_lo;
    const float* khi = SPARSE ? hi : h->grid_hi;
    const int bx = (int)std::floor(klo[0] / ds) - 1, by = (int)std::floor(klo[1] / ds) - 1, bz = (int)std::floor(klo[2] / ds) - 1;
    const int wx = bits_for((long long)std::floor(khi[0] / ds) + 2 - bx), wy = bits_for((long long)std::floor(khi[1] / ds) + 2 - by),
              wz = bits_for((long long)std::floor(khi[2] / ds) + 2 - bz);
    const bool rel = wx + wy + wz <= 62;
    if (!SPARSE && !rel) return map_add_points_full(h, nxyz, n, ds);
    const int vbits = rel ? wx + wy + wz : 63;
    const int key_bits = SPARSE ? 64 : bits_for((long long)h->ncell);
    FLB_CUDA(h, h->vkeys.reserve(n));
    FLB_CUDA(h, h->vkeys_sorted.reserve(n));
    FLB_CUDA(h, h->vals.reserve(std::max(n, M)));
    FLB_CUDA(h, h->vals_sorted.reserve(std::max(n, M)));
    FLB_CUDA(h, h->dead.reserve(M));
    FLB_CUDA(h, h->ins.reserve(n));
    // the inserts' cell keys: the sparse index's reuse the voxel-key buffers (spent by then)
    CellKey<SPARSE>* keys;
    CellKey<SPARSE>* keys_sorted;
    if constexpr (SPARSE) {
        keys = h->vkeys.p;
        keys_sorted = h->vkeys_sorted.p;
    } else {
        FLB_CUDA(h, h->keys.reserve(std::max(n, M)));
        FLB_CUDA(h, h->keys_sorted.reserve(std::max(n, M)));
        keys = h->keys.p;
        keys_sorted = h->keys_sorted.p;
    }
    FLB_CUDA(h, cudaMemsetAsync(h->dead.p, 0, M, h->stream));
    FLB_CUDA(h, cudaMemsetAsync(h->ins.p, 0, n, h->stream));
    const int gn = (n + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        if (rel) k_vox_keys_rel<<<gn, 256, 0, h->stream>>>(nxyz, n, ds, bx, by, bz, wx, wx + wy, h->vkeys.p, h->vals.p);
        else k_vox_keys<<<gn, 256, 0, h->stream>>>(nxyz, n, ds, h->vkeys.p, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    // cub_tmp also covers map_merge's scan, so that it is not reallocated under the sorts enqueued here
    size_t t1 = 0, t2 = 0, t3 = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t1, h->vkeys.p, h->vkeys_sorted.p, h->vals.p, h->vals_sorted.p, n, 0, vbits, h->stream));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t2, keys, keys_sorted, h->vals.p, h->vals_sorted.p, n, 0, key_bits, h->stream));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, t3, h->dead_before.p, h->dead_before.p, M, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(std::max(t1, std::max(t2, t3))));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, t1, h->vkeys.p, h->vkeys_sorted.p, h->vals.p, h->vals_sorted.p, n, 0, vbits, h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vox_resolve_incremental<SPARSE><<<gn, 256, 0, h->stream>>>(h->vkeys_sorted.p, h->vals_sorted.p, nxyz, n, ds, g, cell_index(h),
                                                                     h->map_pts.p, h->dead.p, h->ins.p);
        // inserted points sorted by cell key (not-inserted ones carry "no cell": behind every cell)
        k_insert_keys<SPARSE><<<gn, 256, 0, h->stream>>>(nxyz, n, h->ins.p, g, h->ncell, keys, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, t2, keys, keys_sorted, h->vals.p, h->vals_sorted.p, n, 0, key_bits, h->stream));
    h->launches += 5;                                 // the second kernel above, two launches per radix sort
    return map_merge<SPARSE>(h, nxyz, n, keys_sorted, h->vals_sorted.p, 0);
}

extern "C" {

// The voxel-key and cell-key limits of new points with bounds lo / hi (shared by both Add_Points entry points).
static int map_add_check_bounds(flb_handle* h, const char* who, const float* lo, const float* hi, float downsample_size) {
    const float lim = 1.0e6f * downsample_size;
    for (int k = 0; k < 3; ++k)
        if (lo[k] < -lim || hi[k] > lim) return fail(h, FLB_ERR_INVALID, "%s: coordinate / downsample_size exceeds 2^20 voxels", who);
    if (h->sparse) {
        // the sparse index has no box to leave, but every cell needs a key: within 2^20 cells of the anchor
        const float o[3] = {h->grid.ox, h->grid.oy, h->grid.oz}, lk = (float)kCellKeyBias;
        for (int k = 0; k < 3; ++k) {
            const float a = (lo[k] - o[k]) * h->grid.inv_cell, b = (hi[k] - o[k]) * h->grid.inv_cell;
            if (!(a >= -lk && b < lk)) return fail(h, FLB_ERR_INVALID, "%s: point more than 2^20 cells from the map's anchor", who);
        }
    }
    return FLB_OK;
}

// Add_Points (downsample = true) of n >= 1 validated new points already on the device (nxyz, packed, in input order;
// bounds lo / hi): the map box takes them in, then the sparse-index merge, the full rebuild or the dense incremental
// merge runs.  flb_map_add_points and flb_map_add_scan differ only in how the points get to nxyz.
static int map_add_points_dev(flb_handle* h, const float* nxyz, int n, float downsample_size, const float* lo, const float* hi) {
    bool inside = true;
    for (int k = 0; k < 3; ++k) inside = inside && lo[k] >= h->grid_lo[k] && hi[k] <= h->grid_hi[k];
    for (int k = 0; k < 3; ++k) { h->map_lo[k] = std::min(h->map_lo[k], lo[k]); h->map_hi[k] = std::max(h->map_hi[k], hi[k]); }
    if (h->sparse) return map_add_points_inc<true>(h, nxyz, n, downsample_size, lo, hi);
    if (!inside) return map_add_points_full(h, nxyz, n, downsample_size);
    return map_add_points_inc<false>(h, nxyz, n, downsample_size, lo, hi);
}

int flb_map_add_points(flb_handle* h, const float* world_xyz, int n, int stride, float downsample_size) {
    FLB_CHECK_H(h);
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_map_add_points: no map uploaded");
    if (!world_xyz || n < 0 || stride < 3 || !(downsample_size > 0)) return fail(h, FLB_ERR_INVALID, "flb_map_add_points: bad arguments");
    if (n == 0) return FLB_OK;
    void* stv = nullptr;
    FLB_CUDA(h, h->st_map.acquire((size_t)n * 3 * sizeof(float), &stv));
    float* st = static_cast<float*>(stv);
    pack_points(st, world_xyz, n, stride);
    float lo[3], hi[3];
    if (fold_points<true>(st, n, lo, hi)) return fail(h, FLB_ERR_INVALID, "flb_map_add_points: non-finite coordinate");
    { int rcb = map_add_check_bounds(h, "flb_map_add_points", lo, hi, downsample_size); if (rcb) return rcb; }
    // the input is valid from here on: only now does it go to the device and the map box take it in
    FLB_CUDA(h, h->add_xyz.reserve((size_t)n * 3));
    FLB_CUDA(h, cudaMemcpyAsync(h->add_xyz.p, st, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_map.mark(h->stream));
    return map_add_points_dev(h, h->add_xyz.p, n, downsample_size, lo, hi);
}

// lo / hi of a bounds record (kScanRec*: the per-axis ~min and max order keys)
static void scan_rec_bounds(const unsigned* rec, float lo[3], float hi[3]) {
    for (int k = 0; k < 3; ++k) {
        lo[k] = f32_from_order_key(~rec[kScanRecMin + k]);
        hi[k] = f32_from_order_key(rec[kScanRecMax + k]);
    }
}

// pointBodyToWorld of the n >= 1 points of src into out (k_map_scan_world; scan_order: src is the ordered scan, each
// point goes to its caller's index; else src is in the caller's order) at (R, p), or -- R null -- at the device state x
// once the pending state operations are flushed.  The bounds record is read back: bad = a non-finite coordinate, else
// the points lie in lo / hi.  Ends with a stream synchronise: src may change once it returns, out is a copy.
static int scan_to_world(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3], const float4* src, int n,
                         bool scan_order, DevBuf<float>& out, DevBuf<unsigned>& rec_dev, bool* bad, float lo[3], float hi[3]) {
    if (!R) { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    LioPose pose{};
    std::memcpy(pose.R_LI, prm->R_LI, sizeof(pose.R_LI));
    std::memcpy(pose.t_LI, prm->t_LI, sizeof(pose.t_LI));
    if (R) {
        std::memcpy(pose.R, R, sizeof(pose.R));
        std::memcpy(pose.p, p, sizeof(pose.p));
    }
    FLB_CUDA(h, out.reserve((size_t)n * 3));
    FLB_CUDA(h, rec_dev.reserve(kScanRecWords));
    FLB_CUDA(h, cudaMemsetAsync(rec_dev.p, 0, kScanRecWords * sizeof(unsigned), h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        const State18* x = R ? nullptr : &h->states.p[0];
        if (scan_order) k_map_scan_world<true><<<(n + 255) / 256, 256, 0, h->stream>>>(src, n, pose, x, out.p, rec_dev.p);
        else k_map_scan_world<false><<<(n + 255) / 256, 256, 0, h->stream>>>(src, n, pose, x, out.p, rec_dev.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    unsigned* rec = static_cast<unsigned*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(rec, rec_dev.p, kScanRecWords * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    *bad = rec[kScanRecBad] != 0;
    scan_rec_bounds(rec, lo, hi);
    return FLB_OK;
}

// map_incremental (src/laserMapping.cpp:692-706) from what is on the device: the uploaded scan, transformed at (R, p) or
// at the device state x, enters Add_Points in the caller's order.  One kernel (transform + bounds) and one small
// readback replace flb_map_add_points' staging, host checks and copy; the merge is the same code.
int flb_map_add_scan(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3], float downsample_size) {
    FLB_CHECK_H(h);
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_map_add_scan: no map uploaded");
    if (!prm || (R == nullptr) != (p == nullptr) || !(downsample_size > 0))
        return fail(h, FLB_ERR_INVALID, "flb_map_add_scan: bad arguments (prm, R and p both or neither, downsample_size > 0)");
    if (h->comm || h->p2p.world > 0)
        return fail(h, FLB_ERR_STATE, "flb_map_add_scan: single GPU only (each rank holds only its shard of the scan)");
    if (!h->scan_valid)
        return fail(h, FLB_ERR_STATE, "flb_map_add_scan: no scan uploaded since the last flb_voxel_grid (or ever)");
    if (!R && !h->state_valid) return fail(h, FLB_ERR_STATE, "flb_map_add_scan: no pose given and no device state");
    const int n = h->N;
    if (n == 0) return FLB_OK;
    // h->scan is the current set of the double-buffered scan.  scan_to_world ends with a stream synchronise, so a later
    // flb_scan_upload (which fills the other set, and this one only after the next swap) cannot overwrite it under us.
    bool bad = false;
    float lo[3], hi[3];
    { int rcw = scan_to_world(h, prm, R, p, h->scan.p, n, true, h->add_xyz, h->add_rec, &bad, lo, hi); if (rcw) return rcw; }
    if (bad) return fail(h, FLB_ERR_INVALID, "flb_map_add_scan: non-finite coordinate");
    { int rcb = map_add_check_bounds(h, "flb_map_add_scan", lo, hi, downsample_size); if (rcb) return rcb; }
    return map_add_points_dev(h, h->add_xyz.p, n, downsample_size, lo, hi);
}

// pcl_wait_pub (src/laserMapping.cpp:1763-1772) from what is on the device: the uploaded scan (feats_down_body) or the
// last flb_imu_undistort output (feats_undistort), transformed at (R, p) or at the device state x into wc_xyz, in the
// caller's order.  The kernel of flb_map_add_scan; its bounds record is the one read back, and it is kept for the
// overflow test of flb_vmap_select_cloud.  The visual-map consumers (*_cloud) read wc_xyz on the device.
int flb_world_cloud(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3], int source, int* n_out) {
    FLB_CHECK_H(h);
    h->wc_n = -1;                                     // on any error below, no cloud is held
    if (n_out) *n_out = 0;
    if (!prm || (R == nullptr) != (p == nullptr) || (source != FLB_CLOUD_SCAN && source != FLB_CLOUD_UNDISTORTED))
        return fail(h, FLB_ERR_INVALID, "flb_world_cloud: bad arguments (prm, R and p both or neither, source)");
    const float4* src = nullptr;
    int n = 0;
    if (source == FLB_CLOUD_SCAN) {
        if (h->comm || h->p2p.world > 0)
            return fail(h, FLB_ERR_STATE, "flb_world_cloud: FLB_CLOUD_SCAN is single GPU only (each rank holds only its shard of the scan)");
        if (!h->scan_valid) return fail(h, FLB_ERR_STATE, "flb_world_cloud: no scan uploaded since the last flb_voxel_grid (or ever)");
        src = h->scan.p;
        n = h->N;
    } else {
        if (h->undist_n < 0) return fail(h, FLB_ERR_STATE, "flb_world_cloud: no flb_imu_undistort output (none yet, or the last call failed)");
        src = h->undist_pts;
        n = h->undist_n;
    }
    if (!R && !h->state_valid) return fail(h, FLB_ERR_STATE, "flb_world_cloud: no pose given and no device state");
    float lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    if (n > 0) {
        // Both sources stay put until scan_to_world's synchronise: a later flb_scan_upload fills the other scan set, and
        // flb_imu_undistort is blocking.  wc_xyz is a copy, so neither changes the cloud afterwards.
        bool bad = false;
        { int rcw = scan_to_world(h, prm, R, p, src, n, source == FLB_CLOUD_SCAN, h->wc_xyz, h->wc_rec, &bad, lo, hi); if (rcw) return rcw; }
        if (bad) return fail(h, FLB_ERR_INVALID, "flb_world_cloud: non-finite coordinate");
        for (int k = 0; k < 3; ++k)
            if (lo[k] < -kVmapCoordLimit || hi[k] > kVmapCoordLimit) return fail(h, FLB_ERR_INVALID, "flb_world_cloud: coordinate beyond 2^20 visual-map voxels");
    }
    std::memcpy(h->wc_lo, lo, sizeof(lo));
    std::memcpy(h->wc_hi, hi, sizeof(hi));
    h->wc_n = n;
    if (n_out) *n_out = n;
    return FLB_OK;
}

int flb_world_cloud_download(flb_handle* h, float* xyz, int capacity, int* n_out) {
    FLB_CHECK_H(h);
    if (capacity < 0 || (capacity > 0 && !xyz)) return fail(h, FLB_ERR_INVALID, "flb_world_cloud_download: bad arguments");
    if (h->wc_n < 0) return fail(h, FLB_ERR_STATE, "flb_world_cloud_download: no world cloud (flb_world_cloud first, or it failed)");
    if (n_out) *n_out = h->wc_n;
    const int m = std::min(capacity, h->wc_n);
    if (m > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(xyz, h->wc_xyz.p, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    return FLB_OK;
}

// laserCloudOri of the pending pass into ef_body: the rows of the scan set it ran on (the current one, or scan_alt after
// one more install), scattered to their caller's index by k_effect_scatter and compacted in that order by cub's select.
// Runs on `stream` after the pass; the count read ends with a stream synchronise, so a later install cannot overwrite
// the set under it.
static int effect_capture(flb_handle* h) {
    const bool cur = h->scan_gen == h->ef_gen;
    const float4* scan = cur ? h->scan.p : h->scan_alt.p;
    const unsigned char* sel = cur ? h->sel.p : h->sel_alt.p;
    const int N = h->ef_N;
    int n = 0;
    if (N > 0) {
        FLB_CUDA(h, h->ef_scatter.reserve(N));
        FLB_CUDA(h, h->ef_flag.reserve(N));
        FLB_CUDA(h, h->ef_body.reserve(N));
        FLB_CUDA(h, h->ef_count.reserve(1));
        {
            LaunchScope ls(h, FAM_OTHER);
            k_effect_scatter<<<(N + 255) / 256, 256, 0, h->stream>>>(scan, sel, N, h->ef_flag.p, h->ef_scatter.p);
            FLB_CUDA(h, cudaGetLastError());
        }
        size_t tmp_bytes = 0;
        FLB_CUDA(h, cub::DeviceSelect::Flagged(nullptr, tmp_bytes, h->ef_scatter.p, h->ef_flag.p, h->ef_body.p, h->ef_count.p, N, h->stream));
        FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
        FLB_CUDA(h, cub::DeviceSelect::Flagged(h->cub_tmp.p, tmp_bytes, h->ef_scatter.p, h->ef_flag.p, h->ef_body.p, h->ef_count.p, N, h->stream));
        h->launches++;
        int* cnt = static_cast<int*>(h->pin_out.p);
        FLB_CUDA(h, cudaMemcpyAsync(cnt, h->ef_count.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        n = *cnt;
    }
    h->ef_n = n;
    h->ef_state = flb_handle::kEfNone;
    return FLB_OK;
}

// publish_effect_world (src/laserMapping.cpp:871-885): laserCloudOri (:1588-1600) of the last LIO pass, transformed
// by RGBpointBodyToWorld at (R, p) or at the device state x -- scan_to_world, the kernel of flb_world_cloud.
int flb_effect_cloud(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3], int* n_out) {
    FLB_CHECK_H(h);
    h->ef_wn = -1;                                    // on any error below, no world cloud is held
    if (n_out) *n_out = 0;
    if (!prm || (R == nullptr) != (p == nullptr))
        return fail(h, FLB_ERR_INVALID, "flb_effect_cloud: bad arguments (prm, R and p both or neither)");
    if (h->comm || h->p2p.world > 0)
        return fail(h, FLB_ERR_STATE, "flb_effect_cloud: single GPU only (each rank holds only its shard of the scan)");
    if (!R && !h->state_valid) return fail(h, FLB_ERR_STATE, "flb_effect_cloud: no pose given and no device state");
    if (h->ef_state == flb_handle::kEfPending && h->scan_gen - h->ef_gen >= 2) h->ef_state = flb_handle::kEfLost;
    if (h->ef_state == flb_handle::kEfLost)
        return fail(h, FLB_ERR_STATE, "flb_effect_cloud: the last LIO pass's scan was replaced (two scan uploads or flb_voxel_grid) before capture");
    if (h->ef_state == flb_handle::kEfPending) { int rcc = effect_capture(h); if (rcc) return rcc; }
    const int n = h->ef_n;
    if (n > 0) {
        bool bad = false;
        float lo[3], hi[3];
        { int rcw = scan_to_world(h, prm, R, p, h->ef_body.p, n, false, h->ef_xyz, h->ef_rec, &bad, lo, hi); if (rcw) return rcw; }
        if (bad) return fail(h, FLB_ERR_INVALID, "flb_effect_cloud: non-finite coordinate");
    }
    h->ef_wn = n;
    if (n_out) *n_out = n;
    return FLB_OK;
}

int flb_effect_cloud_download(flb_handle* h, float* xyz, int capacity, int* n_out) {
    FLB_CHECK_H(h);
    if (capacity < 0 || (capacity > 0 && !xyz)) return fail(h, FLB_ERR_INVALID, "flb_effect_cloud_download: bad arguments");
    if (h->ef_wn < 0) return fail(h, FLB_ERR_STATE, "flb_effect_cloud_download: no effect cloud (flb_effect_cloud first, or it failed)");
    if (n_out) *n_out = h->ef_wn;
    const int m = std::min(capacity, h->ef_wn);
    if (m > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(xyz, h->ef_xyz.p, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    return FLB_OK;
}

int flb_map_delete_boxes(flb_handle* h, const float* boxes, int nb) {
    FLB_CHECK_H(h);
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_map_delete_boxes: no map uploaded");
    if (nb < 0 || (nb > 0 && !boxes)) return fail(h, FLB_ERR_INVALID, "flb_map_delete_boxes: bad arguments");
    if (nb == 0) return FLB_OK;
    const int M = h->M;
    void* stv = nullptr;
    FLB_CUDA(h, h->st_misc.acquire((size_t)nb * 6 * sizeof(float), &stv));
    std::memcpy(stv, boxes, (size_t)nb * 6 * sizeof(float));
    FLB_CUDA(h, h->boxes.reserve((size_t)nb * 6));
    FLB_CUDA(h, cudaMemcpyAsync(h->boxes.p, stv, (size_t)nb * 6 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_misc.mark(h->stream));
    FLB_CUDA(h, h->map_comb.reserve((size_t)M * 3));
    FLB_CUDA(h, h->vals.reserve(M));
    FLB_CUDA(h, h->keep.reserve(M));
    FLB_CUDA(h, cudaMemcpyAsync(h->map_comb.p, h->map_raw.p, (size_t)M * 3 * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_box_flags<<<(M + 255) / 256, 256, 0, h->stream>>>(h->map_comb.p, M, h->boxes.p, nb, h->keep.p, h->vals.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    return compact_and_rebuild(h, h->vals.p, M);
}

// lasermap_fov_segment (src/laserMapping.cpp:363-421): the cube step on the device (k_fov_step), the points inside its
// boxes flagged and counted there (k_fov_flags), one read of the record, then -- only if a point goes -- map_merge with
// no inserts: survivors keep their order, and the grid box stays (the next Add_Points that leaves it takes the full path).
// A frame whose boxes hold no map point costs two tiny kernels and the read; the map, grid and box stay untouched.
int flb_map_fov_segment(flb_handle* h, const flb_fov_params* prm, const double pos[3], int* n_boxes, float boxes[18],
                        float local_box[6], int* n_deleted) {
    FLB_CHECK_H(h);
    if (!prm || !(std::isfinite(prm->cube_len) && prm->cube_len > 0) || !(std::isfinite(prm->det_range) && prm->det_range > 0) ||
        !(std::isfinite(prm->mov_threshold) && prm->mov_threshold > 0))
        return fail(h, FLB_ERR_INVALID, "flb_map_fov_segment: bad arguments (prm; cube_len, det_range, mov_threshold finite and > 0)");
    if (!pos && !h->state_valid) return fail(h, FLB_ERR_STATE, "flb_map_fov_segment: no pose given and no device state");
    if (!pos) { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    if (!h->fov_rec.p) {
        FLB_CUDA(h, h->fov_rec.reserve(2));
        FLB_CUDA(h, cudaMemsetAsync(h->fov_rec.p, 0, 2 * sizeof(FovRecord), h->stream));   // Localmap_Initialized = false
        h->fov_cur = 0;
    }
    FovRecord* cur = h->fov_rec.p + h->fov_cur;
    FovRecord* next = h->fov_rec.p + (1 - h->fov_cur);
    const int M = h->M;
    if (M > 0) FLB_CUDA(h, h->dead.reserve(M));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_fov_step<<<1, 1, 0, h->stream>>>(cur, next, pos ? pos[0] : 0.0, pos ? pos[1] : 0.0, pos ? pos[2] : 0.0,
                                            pos ? nullptr : &h->states.p[0], prm->cube_len, prm->det_range, prm->mov_threshold);
        if (M > 0) {
            k_fov_flags<<<(M + 255) / 256, 256, 0, h->stream>>>(h->map_pts.p, M, next, h->dead.p);
            h->launches++;
        }
        FLB_CUDA(h, cudaGetLastError());
    }
    FovRecord* rec = static_cast<FovRecord*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(rec, next, sizeof(FovRecord), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    const FovRecord r = *rec;
    if (M > 0 && r.n_deleted >= M)
        return fail(h, FLB_ERR_STATE, "flb_map_fov_segment: the boxes hold every map point (the map would be empty)");
    h->fov_cur = 1 - h->fov_cur;                      // the cube moves: LocalMap_Points = New_LocalMap_Points (:413)
    if (r.n_deleted > 0) {
        const int rcd = h->sparse ? map_merge<true>(h, nullptr, 0, nullptr, nullptr, r.n_deleted)
                                  : map_merge<false>(h, nullptr, 0, nullptr, nullptr, r.n_deleted);
        if (rcd) return rcd;
    }
    if (n_boxes) *n_boxes = r.n_boxes;
    if (boxes) std::memcpy(boxes, r.boxes, sizeof(r.boxes));
    if (local_box) {
        std::memcpy(local_box, r.cube.vmin, 3 * sizeof(float));
        std::memcpy(local_box + 3, r.cube.vmax, 3 * sizeof(float));
    }
    if (n_deleted) *n_deleted = r.n_deleted;
    return FLB_OK;
}

int flb_map_fov_reset(flb_handle* h) {
    FLB_CHECK_H(h);
    if (h->fov_rec.p) FLB_CUDA(h, cudaMemsetAsync(h->fov_rec.p, 0, 2 * sizeof(FovRecord), h->stream));
    return FLB_OK;
}

int flb_map_size(const flb_handle* h) { return h ? h->M : 0; }

int flb_map_grid_info(flb_handle* h, double* cell_size, int* sparse, int64_t* cells, int64_t* index_bytes_out) {
    FLB_CHECK_H(h);
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_map_grid_info: no map uploaded");
    if (cell_size) *cell_size = (double)h->grid.cell;
    if (sparse) *sparse = h->sparse ? 1 : 0;
    if (cells) *cells = (int64_t)h->ncell;
    if (index_bytes_out) *index_bytes_out = (int64_t)index_bytes(h);
    return FLB_OK;
}

int flb_map_download(flb_handle* h, float* xyz, int capacity, int* M_out) {
    FLB_CHECK_H(h);
    if (M_out) *M_out = h->M;
    if (!xyz || capacity <= 0) return FLB_OK;
    const int n = std::min(capacity, h->M);
    FLB_CUDA(h, cudaMemcpyAsync(xyz, h->map_raw.p, (size_t)n * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

namespace {

// flb_imu_undistort and flb_imu_undistort_lidar from the argument checks on.  The n_points points are either the
// caller's (pts, packed into the staging area and uploaded) or, with dev_pts, already on the device as {x, y, z, offset}
// and read in place.
int imu_undistort_core(flb_handle* h, const char* who, const flb_imu_params* prm, flb_imu_carry* carry, const flb_imu_sample* v_imu,
                       int n_imu, double pcl_beg_time, double pcl_end_time, const float* pts, int stride, int offset_index,
                       const float4* dev_pts, int n_points, float* out_xyz, double* poses_out, int* n_poses_out) {
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "%s: no device state (flb_state_upload)", who);
    { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    for (int i = 0; i + 1 < n_imu; ++i)
        if (!(v_imu[i + 1].t >= v_imu[i].t)) return fail(h, FLB_ERR_INVALID, "%s: IMU times must be non-decreasing", who);
    static_assert(sizeof(ImuSampleDev) == sizeof(flb_imu_sample) && sizeof(ImuCarryDev) == sizeof(flb_imu_carry), "ABI layout");
    static_assert(sizeof(ImuPose) == 22 * sizeof(double), "IMUpose layout");
    ImuParamsDev d;
    std::memcpy(d.cov_gyr, prm->cov_gyr, sizeof(d.cov_gyr));
    std::memcpy(d.cov_acc, prm->cov_acc, sizeof(d.cov_acc));
    std::memcpy(d.cov_bias_gyr, prm->cov_bias_gyr, sizeof(d.cov_bias_gyr));
    std::memcpy(d.cov_bias_acc, prm->cov_bias_acc, sizeof(d.cov_bias_acc));
    d.G_m_s2 = prm->G_m_s2;
    d.mean_acc_norm = prm->mean_acc_norm;
    std::memcpy(d.R_LI, prm->R_LI, sizeof(d.R_LI));
    std::memcpy(d.t_LI, prm->t_LI, sizeof(d.t_LI));
    const size_t n1 = (size_t)std::max(n_points, 1);
    // device buffers: samples + carry + aux + poses packed in one double array, points as float4 in/out
    const size_t off_carry = (size_t)n_imu * 7, off_aux = off_carry + 7, off_poses = off_aux + 16, total = off_poses + (size_t)n_imu * 22;
    FLB_CUDA(h, h->imu_buf.reserve(total));
    FLB_CUDA(h, h->imu_pts.reserve(n1 * 2));
    FLB_CUDA(h, h->imu_heads.reserve(n1));
    void* stv = nullptr;
    FLB_CUDA(h, h->st_scan.acquire((dev_pts ? 0 : n1 * 4 * sizeof(float)) + (off_aux) * sizeof(double), &stv));
    double* st_d = static_cast<double*>(stv);
    std::memcpy(st_d, v_imu, (size_t)n_imu * sizeof(flb_imu_sample));
    std::memcpy(st_d + off_carry, carry, sizeof(flb_imu_carry));
    float* st_p = reinterpret_cast<float*>(st_d + off_aux);
    for (int i = 0; !dev_pts && i < n_points; ++i) {
        st_p[4 * (size_t)i] = pts[(size_t)i * stride];
        st_p[4 * (size_t)i + 1] = pts[(size_t)i * stride + 1];
        st_p[4 * (size_t)i + 2] = pts[(size_t)i * stride + 2];
        st_p[4 * (size_t)i + 3] = pts[(size_t)i * stride + offset_index];
    }
    FLB_CUDA(h, cudaMemcpyAsync(h->imu_buf.p, st_d, off_aux * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    const float4* d_in = dev_pts ? dev_pts : h->imu_pts.p;
    float4* d_out = h->imu_pts.p + n1;
    if (n_points > 0 && !dev_pts)
        FLB_CUDA(h, cudaMemcpyAsync(h->imu_pts.p, st_p, (size_t)n_points * 4 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_scan.mark(h->stream));
    const ImuSampleDev* d_imu = reinterpret_cast<const ImuSampleDev*>(h->imu_buf.p);
    ImuCarryDev* d_carry = reinterpret_cast<ImuCarryDev*>(h->imu_buf.p + off_carry);
    ImuAux* d_aux = reinterpret_cast<ImuAux*>(h->imu_buf.p + off_aux);
    ImuPose* d_poses = reinterpret_cast<ImuPose*>(h->imu_buf.p + off_poses);
    {
        LaunchScope ls(h, FAM_OTHER);
        k_imu_propagate<<<1, 352, 0, h->stream>>>(&h->states.p[0], d_imu, n_imu, d, pcl_beg_time, pcl_end_time, d_carry, d_poses, d_aux);
        FLB_CUDA(h, cudaGetLastError());
    }
    if (n_points > 0) {                                                           // :776
        const int g = (n_points + 255) / 256;
        const float* in_f = reinterpret_cast<const float*>(d_in);
        LaunchScope ls(h, FAM_OTHER);
        k_imu_heads<<<g, 256, 0, h->stream>>>(in_f + 3, 4, n_points, d_poses, d_aux, h->imu_heads.p);
        k_suffix_min<<<1, 1024, 0, h->stream>>>(h->imu_heads.p, n_points);
        k_imu_undistort<<<g, 256, 0, h->stream>>>(in_f, 4, in_f + 3, 4, n_points, d_poses, d_aux, h->imu_heads.p, d, d_out);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 2;
    }
    // results: carry, aux (n_poses), poses, points (out_xyz == NULL: the points stay on the device only, for
    // flb_scan_from_undistorted / flb_world_cloud)
    const size_t out_bytes = (7 + 16 + (size_t)n_imu * 22) * sizeof(double) + n1 * 4 * sizeof(float);
    FLB_CUDA(h, h->pin_out.reserve(out_bytes));
    char* po = static_cast<char*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(po, h->imu_buf.p + off_carry, (7 + 16 + (size_t)n_imu * 22) * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    float* po_pts = reinterpret_cast<float*>(po + (7 + 16 + (size_t)n_imu * 22) * sizeof(double));
    if (n_points > 0 && out_xyz)
        FLB_CUDA(h, cudaMemcpyAsync(po_pts, d_out, (size_t)n_points * 4 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    std::memcpy(carry, po, sizeof(flb_imu_carry));
    ImuAux aux;
    std::memcpy(&aux, po + 7 * sizeof(double), sizeof(aux));
    if (n_poses_out) *n_poses_out = aux.n_poses;
    if (poses_out) std::memcpy(poses_out, po + (7 + 16) * sizeof(double), (size_t)aux.n_poses * 22 * sizeof(double));
    for (int i = 0; out_xyz && i < n_points; ++i) {
        out_xyz[3 * (size_t)i] = po_pts[4 * (size_t)i];
        out_xyz[3 * (size_t)i + 1] = po_pts[4 * (size_t)i + 1];
        out_xyz[3 * (size_t)i + 2] = po_pts[4 * (size_t)i + 2];
    }
    h->undist_pts = d_out;
    h->undist_n = n_points;
    h->last_pass_valid = false;
    h->last_vio_valid = false;
    return FLB_OK;
}

}  // namespace

int flb_imu_undistort(flb_handle* h, const flb_imu_params* prm, flb_imu_carry* carry, const flb_imu_sample* v_imu, int n_imu,
                      double pcl_beg_time, double pcl_end_time, const float* pts, int stride, int offset_index, int n_points,
                      float* out_xyz, double* poses_out, int* n_poses_out) {
    FLB_CHECK_H(h);
    h->undist_n = -1;                 // flb_world_cloud's FLB_CLOUD_UNDISTORTED source is this call's output, or none
    if (!prm || !carry || !v_imu || n_imu < 1 || n_points < 0 || (n_points > 0 && !pts) || stride < 4 ||
        offset_index < 3 || offset_index >= stride)
        return fail(h, FLB_ERR_INVALID, "flb_imu_undistort: bad arguments");
    return imu_undistort_core(h, "flb_imu_undistort", prm, carry, v_imu, n_imu, pcl_beg_time, pcl_end_time, pts, stride, offset_index,
                              nullptr, n_points, out_xyz, poses_out, n_poses_out);
}

// ---- the driver's LiDAR message on the device ----------------------------------------------------------------------
namespace {

// byte size and alignment of the time field of each kind
int lidar_time_bytes(int kind) { return kind == kLidarXt32 ? 8 : 4; }

bool lidar_field_ok(int off, int bytes, int step) { return off >= 0 && off % bytes == 0 && off + bytes <= step; }
// Velodyne drivers place their fields anywhere, so no alignment is asked of them
bool velo_field_ok(int off, int bytes, int step) { return off >= 0 && off <= step - bytes; }

// flb_lidar_format -> LidarFmt, the checks in the order flb_lidar_upload and (features) flb_lidar_upload_features
// report them.  The features call also checks dis_b, refuses the Velodyne and the XT32 (so its time field is 4 bytes),
// caps n_scans at pl_buff's 128, and always reads off_line: the Livox line or the Ouster's ring.
int lidar_format(flb_handle* h, const char* who, const flb_lidar_format* fmt, const void* records, int n_records, bool features,
                 double dis_b, LidarFmt* f) {
    if (n_records < 0 || !fmt || (n_records > 0 && !records) || (features && !std::isfinite(dis_b)))
        return fail(h, FLB_ERR_INVALID, "%s: bad arguments", who);
    if (features && (fmt->kind == kLidarVelodyne || fmt->kind == kLidarXt32))
        return fail(h, FLB_ERR_INVALID, "%s: kind %d: a Velodyne cloud goes to flb_lidar_upload_velodyne_features; the XT32 "
                    "has no feature branch (src/preprocess.cpp:432-464), so flb_lidar_upload serves it", who, fmt->kind);
    if (fmt->kind < kLidarLivox || fmt->kind > kLidarXt32) return fail(h, FLB_ERR_INVALID, "%s: unknown kind %d", who, fmt->kind);
    if (fmt->point_filter_num < 1 || fmt->n_scans < 1 || (features && fmt->n_scans > 128) || !std::isfinite(fmt->blind))
        return fail(h, FLB_ERR_INVALID, "%s: point_filter_num %d, n_scans %d%s, blind %g", who, fmt->point_filter_num,
                    fmt->n_scans, features ? " (1..128: pl_buff[128])" : "", fmt->blind);
    const int step = fmt->point_step;
    const bool livox = fmt->kind == kLidarLivox, line = livox || features;
    if (step < 1 || !lidar_field_ok(fmt->off_x, 4, step) || !lidar_field_ok(fmt->off_y, 4, step) || !lidar_field_ok(fmt->off_z, 4, step) ||
        !lidar_field_ok(fmt->off_time, lidar_time_bytes(fmt->kind), step) || (line && !lidar_field_ok(fmt->off_line, 1, step)) ||
        (livox && !lidar_field_ok(fmt->off_tag, 1, step)))
        return fail(h, FLB_ERR_INVALID, "%s: a field does not fit in point_step %d or is not aligned to its type", who, step);
    *f = LidarFmt{};
    f->kind = fmt->kind, f->step = step, f->off_x = fmt->off_x, f->off_y = fmt->off_y, f->off_z = fmt->off_z, f->off_time = fmt->off_time;
    f->off_tag = livox ? fmt->off_tag : 0, f->off_line = line ? fmt->off_line : 0;
    f->n_scans = fmt->n_scans, f->filter_num = fmt->point_filter_num, f->blind = fmt->blind;
    return FLB_OK;
}

// flb_velodyne_format -> LidarFmt for flb_lidar_upload_velodyne and (features) flb_lidar_upload_velodyne_features, which
// also checks dis_b, caps n_scans at pl_buff's 128 and reads the ring as the line.  *given: given_offset_time (:279), the
// last record's time > 0; without a time field the reference reads 0.
int velo_format(flb_handle* h, const char* who, const flb_velodyne_format* fmt, const void* records, int n_records, bool features,
                double dis_b, LidarFmt* f, bool* given) {
    if (n_records < 0 || !fmt || (n_records > 0 && !records) || (features && !std::isfinite(dis_b)))
        return fail(h, FLB_ERR_INVALID, "%s: bad arguments", who);
    if (fmt->point_filter_num < 1 || fmt->n_scans < 1 || (features && fmt->n_scans > 128) || !std::isfinite(fmt->blind))
        return fail(h, FLB_ERR_INVALID, "%s: point_filter_num %d, n_scans %d%s, blind %g", who, fmt->point_filter_num,
                    fmt->n_scans, features ? " (1..128: pl_buff[128])" : "", fmt->blind);
    const int step = fmt->point_step;
    if (step < 1 || !velo_field_ok(fmt->off_x, 4, step) || !velo_field_ok(fmt->off_y, 4, step) || !velo_field_ok(fmt->off_z, 4, step) ||
        !velo_field_ok(fmt->off_ring, 2, step) || (fmt->off_time != -1 && !velo_field_ok(fmt->off_time, 4, step)))
        return fail(h, FLB_ERR_INVALID, "%s: a field does not fit in point_step %d", who, step);
    *f = LidarFmt{};
    f->kind = kLidarVelodyne, f->step = step, f->off_x = fmt->off_x, f->off_y = fmt->off_y, f->off_z = fmt->off_z;
    f->off_time = fmt->off_time >= 0 ? fmt->off_time : 0, f->off_line = features ? fmt->off_ring : 0;
    f->n_scans = fmt->n_scans, f->filter_num = fmt->point_filter_num, f->blind = fmt->blind;
    *given = n_records == 0;
    if (n_records > 0 && fmt->off_time >= 0) {
        float t_last;
        std::memcpy(&t_last, static_cast<const unsigned char*>(records) + (size_t)(n_records - 1) * step + fmt->off_time, sizeof(t_last));
        *given = t_last > 0;
    }
    return FLB_OK;
}

struct VeloYaw { int off_ring, n_scans; };      // flb_lidar_upload_velodyne's route without per-point times

// lid_flags as every route lays it out (3 * n1 + 8 ints): n1 ints of the route's own, kept[n1], pos[n1], the
// LidarRecord, and one int of the route's own right after it (the yaw route's bad ring, the features' point count)
struct LidarFlags {
    int *own, *kept, *pos;
    LidarRecord* rec;
    int* after;
    LidarFlags(int* p, size_t n1)
        : own(p), kept(p + n1), pos(p + 2 * n1), rec(reinterpret_cast<LidarRecord*>(p + 3 * n1)), after(reinterpret_cast<int*>(rec + 1)) {}
};
static_assert(sizeof(LidarRecord) == 4 * sizeof(int), "LidarRecord sits in lid_flags");

// Every route's start: reserve what all routes write, send the raw records to lid_raw on copy_stream (a page-locked
// source read in place), then wait for the idle cloud set's readers: only the kernels that write that set wait.
int lidar_begin(flb_handle* h, const void* records, int n_records, int step) {
    const size_t n1 = std::max(n_records, 1), raw_bytes = (size_t)n_records * step;
    FLB_CUDA(h, h->lid_raw.reserve(std::max<size_t>(raw_bytes, 4)));
    FLB_CUDA(h, h->lid_cloud_alt.reserve(n1));
    FLB_CUDA(h, h->lid_dec.reserve(n1));
    FLB_CUDA(h, h->lid_sorted.reserve(n1));
    FLB_CUDA(h, h->lid_keys.reserve(n1));
    FLB_CUDA(h, h->lid_keys_sorted.reserve(n1));
    FLB_CUDA(h, h->lid_flags.reserve(3 * n1 + 8));
    FLB_CUDA(h, h->pin_lidar.reserve(64));
    cudaStream_t cs = h->copy_stream;
    if (n_records > 0) {
        if (is_pinned(records)) {
            FLB_CUDA(h, cudaMemcpyAsync(h->lid_raw.p, records, raw_bytes, cudaMemcpyHostToDevice, cs));
        } else {
            void* stv = nullptr;
            FLB_CUDA(h, h->st_lidar.acquire(raw_bytes, &stv));
            std::memcpy(stv, records, raw_bytes);
            FLB_CUDA(h, cudaMemcpyAsync(h->lid_raw.p, stv, raw_bytes, cudaMemcpyHostToDevice, cs));
            FLB_CUDA(h, h->st_lidar.mark(cs));
        }
    }
    return vio_copy_begin(h, h->lid_slot);
}

// the idle cloud set, holding rec.n_kept points, becomes the current cloud with its cursor at the start
int lidar_publish(flb_handle* h, const LidarRecord& rec, int* n_points, float* last_offset_ms) {
    std::swap(h->lid_cloud, h->lid_cloud_alt);
    h->lid_slot.slot ^= 1;
    h->lid_n = rec.n_kept;
    h->lid_cursor = 0;
    if (n_points) *n_points = rec.n_kept;
    if (last_offset_ms) *last_offset_ms = rec.n_kept > 0 ? rec.last : 0.f;
    return FLB_OK;
}

// Every route's end, from n > 0 candidates (lid_dec, lf.kept): compact them into the idle cloud set, refuse (yaw: a ring
// >= n_scans, named from the host records; then a kept value that is not finite, in the caller's words `what`), re-sort
// the times when they are out of order, and publish.  t_sum, t_sort: lid_cub's sizes for the ExclusiveSum and the 32-bit
// SortPairs over n items.  A refusal publishes nothing.
int lidar_tail(flb_handle* h, const char* who, const char* what, const LidarFlags& lf, int n, size_t t_sum, size_t t_sort,
               const VeloYaw* yaw, const void* records, int step, int* n_points, float* last_offset_ms) {
    cudaStream_t cs = h->copy_stream;
    const int g = (n + 255) / 256;
    FLB_CUDA(h, cudaMemsetAsync(lf.rec, 0, sizeof(LidarRecord), cs));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(h->lid_cub.p, t_sum, lf.kept, lf.pos, n, cs));
    k_lidar_scatter<<<g, 256, 0, cs>>>(h->lid_dec.p, lf.kept, lf.pos, n, h->lid_cloud_alt.p, h->lid_keys.p, lf.rec);
    k_lidar_order<<<g, 256, 0, cs>>>(h->lid_cloud_alt.p, h->lid_keys.p, n, lf.rec);
    FLB_CUDA(h, cudaGetLastError());
    h->launches += 3;
    LidarRecord rec{};
    int bad_ring = INT_MAX;
    FLB_CUDA(h, cudaMemcpyAsync(h->pin_lidar.p, lf.rec, sizeof(rec) + (yaw ? sizeof(int) : 0), cudaMemcpyDeviceToHost, cs));
    FLB_CUDA(h, cudaStreamSynchronize(cs));
    std::memcpy(&rec, h->pin_lidar.p, sizeof(rec));
    if (yaw) std::memcpy(&bad_ring, static_cast<const char*>(h->pin_lidar.p) + sizeof(rec), sizeof(int));
    if (bad_ring < n) {
        uint16_t ring;
        std::memcpy(&ring, static_cast<const unsigned char*>(records) + (size_t)bad_ring * step + yaw->off_ring, sizeof(ring));
        return fail(h, FLB_ERR_INVALID, "%s: record %d has ring %u >= n_scans %d (the per-ring yaw state has no such ring)", who,
                    bad_ring, (unsigned)ring, yaw->n_scans);
    }
    if (rec.bad) return fail(h, FLB_ERR_INVALID, "%s: %s is not finite", who, what);
    if (rec.unsorted) {
        // stable: equal times keep the candidates' order, record order or pl_surf's line-major order (std::sort leaves it
        // unspecified in the reference)
        FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->lid_cub.p, t_sort, h->lid_keys.p, h->lid_keys_sorted.p, h->lid_cloud_alt.p,
                                                    h->lid_sorted.p, rec.n_kept, 0, 32, cs));
        FLB_CUDA(h, cudaMemcpyAsync(h->lid_cloud_alt.p, h->lid_sorted.p, (size_t)rec.n_kept * sizeof(float4), cudaMemcpyDeviceToDevice, cs));
        k_lidar_last<<<1, 1, 0, cs>>>(h->lid_cloud_alt.p, lf.rec);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 3;
        FLB_CUDA(h, cudaMemcpyAsync(h->pin_lidar.p, lf.rec, sizeof(rec), cudaMemcpyDeviceToHost, cs));
        FLB_CUDA(h, cudaStreamSynchronize(cs));
        std::memcpy(&rec, h->pin_lidar.p, sizeof(rec));
    }
    return lidar_publish(h, rec, n_points, last_offset_ms);
}

// flb_lidar_upload and flb_lidar_upload_velodyne from the argument checks on: decode and filter the records into
// candidates, then lidar_tail.  yaw: the Velodyne route without per-point times; nullptr: the handler's own per-record
// times.
int lidar_upload_core(flb_handle* h, const char* who, const LidarFmt& f, const void* records, int n_records, const VeloYaw* yaw,
                      int* n_points, float* last_offset_ms) {
    const int step = f.step;
    const bool livox = f.kind == kLidarLivox;
    const size_t n1 = std::max(n_records, 1);
    { int rcq = lidar_begin(h, records, n_records, step); if (rcq) return rcq; }
    if (n_records == 0) return lidar_publish(h, LidarRecord{}, n_points, last_offset_ms);
    cudaStream_t cs = h->copy_stream;
    const LidarFlags lf(h->lid_flags.p, n1);
    int* d_vnum = lf.own;
    size_t t1 = 0, t2 = 0, t3 = 0;
    FLB_CUDA(h, cub::DeviceScan::InclusiveSum(nullptr, t1, d_vnum, d_vnum, n_records, cs));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, t2, lf.kept, lf.pos, n_records, cs));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t3, h->lid_keys.p, h->lid_keys_sorted.p, h->lid_cloud_alt.p, h->lid_sorted.p,
                                                n_records, 0, 32, cs));
    // the yaw route: ring keys in [0, n_rings], record indices, and the ring-order maps
    const int n_rings = yaw ? std::min(yaw->n_scans, 65536) : 0;
    int key_bits = 1;
    while (key_bits < 17 && (1 << key_bits) <= n_rings) ++key_bits;
    int* d_idx = nullptr;
    int* d_idx_sorted = nullptr;
    size_t t4 = 0, t5 = 0;
    if (yaw) {
        FLB_CUDA(h, h->lid_idx.reserve(2 * n1));
        FLB_CUDA(h, h->lid_map.reserve(n1));
        d_idx = h->lid_idx.p, d_idx_sorted = h->lid_idx.p + n1;
        FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t4, h->lid_keys.p, h->lid_keys_sorted.p, d_idx, d_idx_sorted, n_records,
                                                    0, key_bits, cs));
        FLB_CUDA(h, cub::DeviceScan::InclusiveScan(nullptr, t5, h->lid_map.p, h->lid_map.p, VeloComposeOp(), n_records, cs));
    }
    FLB_CUDA(h, h->lid_cub.reserve(std::max(std::max(t1, std::max(t2, t3)), std::max(t4, t5))));
    const int g = (n_records + 255) / 256;
    if (yaw) {
        FLB_CUDA(h, cudaMemsetAsync(lf.after, 0x7f, sizeof(int), cs));         // 0x7f7f7f7f: no bad ring
        k_velo_rings<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, step, yaw->off_ring, yaw->n_scans, n_rings, h->lid_keys.p, d_idx,
                                       lf.after);
        FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->lid_cub.p, t4, h->lid_keys.p, h->lid_keys_sorted.p, d_idx, d_idx_sorted,
                                                    n_records, 0, key_bits, cs));
        k_velo_maps<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, n_rings, h->lid_keys_sorted.p, d_idx_sorted, h->lid_map.p);
        FLB_CUDA(h, cub::DeviceScan::InclusiveScan(h->lid_cub.p, t5, h->lid_map.p, h->lid_map.p, VeloComposeOp(), n_records, cs));
        k_velo_flags<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, n_rings, h->lid_keys_sorted.p, d_idx_sorted, h->lid_map.p,
                                       h->lid_dec.p, lf.kept);
        h->launches += 5;
    } else {
        if (livox) {
            k_lidar_valid<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, d_vnum);
            FLB_CUDA(h, cub::DeviceScan::InclusiveSum(h->lid_cub.p, t1, d_vnum, d_vnum, n_records, cs));
            h->launches += 2;
        }
        k_lidar_flags<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, d_vnum, h->lid_dec.p, lf.kept);
        h->launches += 1;
    }
    return lidar_tail(h, who, "a kept point or time", lf, n_records, t2, t3, yaw, records, step, n_points, last_offset_ms);
}

}  // namespace

int flb_lidar_upload(flb_handle* h, const flb_lidar_format* fmt, const void* records, int n_records, int* n_points,
                     float* last_offset_ms) {
    FLB_CHECK_H(h);
    const char* who = "flb_lidar_upload";
    LidarFmt f;
    { int rcq = lidar_format(h, who, fmt, records, n_records, false, 0.0, &f); if (rcq) return rcq; }
    const unsigned char* rec_h = static_cast<const unsigned char*>(records);
    if (n_records > 0 && f.kind == kLidarVelodyne) {
        float t_last;                                                              // given_offset_time, :279
        std::memcpy(&t_last, rec_h + (size_t)(n_records - 1) * f.step + f.off_time, sizeof(t_last));
        if (!(t_last > 0))
            return fail(h, FLB_ERR_INVALID, "%s: a Velodyne cloud without per-point times (last time %g): its times come from "
                        "the yaw angle (src/preprocess.cpp:389-419), which flb_lidar_upload_velodyne derives", who, (double)t_last);
    }
    if (n_records > 0 && f.kind == kLidarXt32) std::memcpy(&f.time_head, rec_h + f.off_time, sizeof(double));   // :441
    return lidar_upload_core(h, who, f, records, n_records, nullptr, n_points, last_offset_ms);
}

int flb_lidar_upload_velodyne(flb_handle* h, const flb_velodyne_format* fmt, const void* records, int n_records, int* n_points,
                              float* last_offset_ms, int* yaw_times) {
    FLB_CHECK_H(h);
    const char* who = "flb_lidar_upload_velodyne";
    LidarFmt f;
    bool given = false;
    { int rcq = velo_format(h, who, fmt, records, n_records, false, 0.0, &f, &given); if (rcq) return rcq; }
    VeloYaw yaw{fmt->off_ring, fmt->n_scans};
    const int rc = lidar_upload_core(h, who, f, records, n_records, given ? nullptr : &yaw, n_points, last_offset_ms);
    if (rc) return rc;
    if (yaw_times) *yaw_times = given ? 0 : 1;
    return FLB_OK;
}

// ---- the feature branches: give_feature's pl_surf ------------------------------------------------------------------
namespace {

// Preprocess's constants (:9-30): the four thresholds are the constructor's std::cos values, computed here on the host
// because the device cos may differ from libm in the last ulp.
FeatConst feat_const(const LidarFmt& f, double dis_b) {
    FeatConst c;
    c.blind = f.blind, c.dis_b = dis_b, c.avia = f.kind == kLidarLivox ? 1 : 0;
    c.jump_up = std::cos(170.0 / 180 * M_PI);
    c.jump_down = std::cos(8.0 / 180 * M_PI);
    c.cos160 = std::cos(160.0 / 180 * M_PI);
    c.smallp_intersect = std::cos(172.5 / 180 * M_PI);
    return c;
}

// flb_lidar_upload_features and flb_lidar_upload_velodyne_features from the argument checks on: pl_surf's points as
// candidates, then lidar_tail.  f.off_line: the Livox line, the Ouster's u8 ring or the Velodyne's u16 ring.  yaw:
// Velodyne times from the yaw angle.
int lidar_features_core(flb_handle* h, const char* who, const LidarFmt& f, double dis_b, const void* records, int n_records,
                        bool yaw, int* n_points, float* last_offset_ms) {
    const FeatConst c = feat_const(f, dis_b);
    const int min_size = f.kind == kLidarLivox ? 6 : f.kind == kLidarVelodyne ? 2 : 1;   // :117, :357; the Ouster: any
    const size_t n1 = std::max(n_records, 1);
    const int ns = f.n_scans;
    int levels = 1;                                      // 2^levels > any chain length (<= the point count)
    while (levels < 31 && ((size_t)1 << levels) <= n1) ++levels;
    FLB_CUDA(h, h->lid_idx.reserve(2 * n1));
    FLB_CUDA(h, h->lid_map.reserve(n1));
    FLB_CUDA(h, h->feat_pts.reserve(n1));
    FLB_CUDA(h, h->feat_i.reserve((size_t)(levels + 8) * n1 + 3 * (size_t)ns + 1));
    FLB_CUDA(h, h->feat_d.reserve(3 * n1));
    FLB_CUDA(h, h->feat_st.reserve(n1));
    FLB_CUDA(h, h->feat_u8.reserve(2 * n1));
    { int rcq = lidar_begin(h, records, n_records, f.step); if (rcq) return rcq; }
    if (n_records == 0) return lidar_publish(h, LidarRecord{}, n_points, last_offset_ms);
    cudaStream_t cs = h->copy_stream;
    const LidarFlags lf(h->lid_flags.p, n1);
    int* d_take = lf.own;
    int* d_count = lf.after;
    int* d_idx = h->lid_idx.p;
    int* d_idx_sorted = h->lid_idx.p + n1;
    // per-point ints: lkey | pv | rs | rs2 | seed | ft | fin | J[levels] | lbeg | lend | lhead
    int* d_lkey = h->feat_i.p;
    int* d_pv = d_lkey + n1;
    int* d_rs = d_pv + n1;
    int* d_rs2 = d_rs + n1;
    int* d_seed = d_rs2 + n1;
    int* d_ft = d_seed + n1;
    int* d_fin = d_ft + n1;
    int* d_J = d_fin + n1;
    int* d_lbeg = d_J + (size_t)levels * n1;
    int* d_lend = d_lbeg + ns;
    int* d_lhead = d_lend + ns;
    double* d_rng = h->feat_d.p;
    double* d_dista = d_rng + n1;
    double* d_isect = d_dista + n1;
    unsigned char* d_vis = h->feat_u8.p;
    unsigned char* d_small = d_vis + n1;
    const int g = (n_records + 255) / 256;
    size_t t1 = 0, t2 = 0, t3 = 0, t4 = 0, t5 = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t1, h->lid_keys.p, h->lid_keys_sorted.p, d_idx, d_idx_sorted, n_records,
                                                0, 8, cs));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, t2, d_take, lf.pos, n_records, cs));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t3, h->lid_keys.p, h->lid_keys_sorted.p, h->lid_cloud_alt.p, h->lid_sorted.p,
                                                n_records, 0, 32, cs));
    FLB_CUDA(h, cub::DeviceScan::InclusiveScan(nullptr, t4, h->lid_map.p, h->lid_map.p, VeloComposeOp(), n_records, cs));
    FLB_CUDA(h, cub::DeviceScan::InclusiveScan(nullptr, t5, d_seed, d_rs, FeatMaxOp(), n_records, cs));
    size_t t6 = 0;
    FLB_CUDA(h, cub::DeviceScan::ExclusiveScan(nullptr, t6, d_seed, d_pv, FeatMaxOp(), -1, n_records, cs));
    FLB_CUDA(h, h->lid_cub.reserve(std::max(std::max(std::max(t1, t2), std::max(t3, t4)), std::max(t5, t6))));
    // the records into line order
    k_feat_keys<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, h->lid_keys.p, d_idx);
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->lid_cub.p, t1, h->lid_keys.p, h->lid_keys_sorted.p, d_idx, d_idx_sorted,
                                                n_records, 0, 8, cs));
    if (yaw) {
        k_velo_maps<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, ns, h->lid_keys_sorted.p, d_idx_sorted, h->lid_map.p);
        FLB_CUDA(h, cub::DeviceScan::InclusiveScan(h->lid_cub.p, t4, h->lid_map.p, h->lid_map.p, VeloComposeOp(), n_records, cs));
        h->launches += 2;
    }
    k_feat_take<<<g, 256, 0, cs>>>(h->lid_keys_sorted.p, n_records, ns, yaw ? 1 : 0, d_take);
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(h->lid_cub.p, t2, d_take, lf.pos, n_records, cs));
    k_feat_gather<<<g, 256, 0, cs>>>(h->lid_raw.p, n_records, f, yaw ? 1 : 0, h->lid_keys_sorted.p, d_idx_sorted, h->lid_map.p,
                                     d_take, lf.pos, h->feat_pts.p, d_lkey, d_count);
    FLB_CUDA(h, cudaGetLastError());
    h->launches += 6;
    int M = 0;
    FLB_CUDA(h, cudaMemcpyAsync(h->pin_lidar.p, d_count, sizeof(int), cudaMemcpyDeviceToHost, cs));
    FLB_CUDA(h, cudaStreamSynchronize(cs));
    std::memcpy(&M, h->pin_lidar.p, sizeof(int));
    if (M == 0) return lidar_publish(h, LidarRecord{}, n_points, last_offset_ms);
    const int gm = (M + 255) / 256;
    int lv = 1;
    while (lv < levels && (1 << lv) <= M) ++lv;
    FLB_CUDA(h, cudaMemsetAsync(d_lbeg, 0, 2 * ns * sizeof(int), cs));
    FLB_CUDA(h, cudaMemsetAsync(d_lhead, 0x7f, ns * sizeof(int), cs));      // 0x7f7f7f7f: no head
    k_feat_range<<<gm, 256, 0, cs>>>(h->feat_pts.p, d_lkey, M, c.avia, c.blind, d_rng, d_dista, d_lbeg, d_lend, d_lhead);
    k_feat_steps<<<gm, 256, 0, cs>>>(h->feat_pts.p, d_rng, d_dista, d_lkey, d_lbeg, d_lend, d_lhead, M, min_size, c,
                                     h->feat_st.p, d_J, d_vis);
    for (int l = 0; l + 1 < lv; ++l) k_feat_jump<<<gm, 256, 0, cs>>>(d_J + (size_t)l * n1, M, d_J + (size_t)(l + 1) * n1);
    for (int l = lv - 1; l >= 0; --l) k_feat_mark<<<gm, 256, 0, cs>>>(d_J + (size_t)l * n1, M, d_vis);
    k_feat_vis_index<<<gm, 256, 0, cs>>>(d_vis, M, d_seed);
    FLB_CUDA(h, cub::DeviceScan::ExclusiveScan(h->lid_cub.p, t6, d_seed, d_pv, FeatMaxOp(), -1, M, cs));
    k_feat_types<<<gm, 256, 0, cs>>>(h->feat_pts.p, d_rng, d_dista, d_lkey, d_lbeg, d_lend, d_lhead, M, min_size, c,
                                     h->feat_st.p, d_vis, d_pv, d_ft, d_isect);
    k_feat_small<<<gm, 256, 0, cs>>>(d_rng, d_dista, d_lkey, d_lbeg, d_lend, d_lhead, M, min_size, c, d_ft, d_isect, d_small);
    k_feat_small_seed<<<gm, 256, 0, cs>>>(d_small, M, d_seed);
    FLB_CUDA(h, cub::DeviceScan::InclusiveScan(h->lid_cub.p, t5, d_seed, d_rs, FeatMaxOp(), M, cs));
    k_feat_final<<<gm, 256, 0, cs>>>(d_ft, d_small, d_rs, d_lkey, d_lbeg, d_lend, d_lhead, M, min_size, d_fin, d_seed);
    FLB_CUDA(h, cub::DeviceScan::InclusiveScan(h->lid_cub.p, t5, d_seed, d_rs2, FeatMaxOp(), M, cs));
    k_feat_emit<<<gm, 256, 0, cs>>>(h->feat_pts.p, d_fin, d_rs2, d_lkey, d_lbeg, d_lend, d_lhead, M, min_size, f.filter_num,
                                    h->lid_dec.p, lf.kept);
    h->launches += 12 + 2 * lv;
    return lidar_tail(h, who, "a point of pl_surf or its time", lf, M, t2, t3, nullptr, records, f.step, n_points, last_offset_ms);
}

}  // namespace

int flb_lidar_upload_features(flb_handle* h, const flb_lidar_format* fmt, double dis_b, const void* records, int n_records,
                              int* n_points, float* last_offset_ms) {
    FLB_CHECK_H(h);
    const char* who = "flb_lidar_upload_features";
    LidarFmt f;
    { int rcq = lidar_format(h, who, fmt, records, n_records, true, dis_b, &f); if (rcq) return rcq; }
    return lidar_features_core(h, who, f, dis_b, records, n_records, false, n_points, last_offset_ms);
}

int flb_lidar_upload_velodyne_features(flb_handle* h, const flb_velodyne_format* fmt, double dis_b, const void* records,
                                       int n_records, int* n_points, float* last_offset_ms, int* yaw_times) {
    FLB_CHECK_H(h);
    const char* who = "flb_lidar_upload_velodyne_features";
    LidarFmt f;
    bool given = false;
    { int rcq = velo_format(h, who, fmt, records, n_records, true, dis_b, &f, &given); if (rcq) return rcq; }
    const int rc = lidar_features_core(h, who, f, dis_b, records, n_records, !given, n_points, last_offset_ms);
    if (rc) return rc;
    if (yaw_times) *yaw_times = given ? 0 : 1;
    return FLB_OK;
}

int flb_lidar_download(flb_handle* h, float* xyzt, int capacity_points, int* n_out) {
    FLB_CHECK_H(h);
    if (h->lid_n < 0) return fail(h, FLB_ERR_STATE, "flb_lidar_download: no cloud (flb_lidar_upload)");
    if (n_out) *n_out = h->lid_n;
    if (!xyzt) return FLB_OK;
    if (capacity_points < h->lid_n) return fail(h, FLB_ERR_INVALID, "flb_lidar_download: capacity %d < %d points", capacity_points, h->lid_n);
    if (h->lid_n > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(xyzt, h->lid_cloud.p, (size_t)h->lid_n * sizeof(float4), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    return FLB_OK;
}

int flb_imu_undistort_lidar(flb_handle* h, const flb_imu_params* prm, flb_imu_carry* carry, const flb_imu_sample* v_imu, int n_imu,
                            double pcl_beg_time, double pcl_end_time, double pcl_offset_time, int is_lidar_end, int* n_taken,
                            float* out_xyz, int capacity_points, double* poses_out, int* n_poses_out) {
    FLB_CHECK_H(h);
    h->undist_n = -1;
    if (!prm || !carry || !v_imu || n_imu < 1 || std::isnan(pcl_offset_time))
        return fail(h, FLB_ERR_INVALID, "flb_imu_undistort_lidar: bad arguments");
    if (h->lid_n < 0) return fail(h, FLB_ERR_STATE, "flb_imu_undistort_lidar: no cloud (flb_lidar_upload)");
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_imu_undistort_lidar: no device state (flb_state_upload)");
    // the window, :634-639 (the cloud is complete: flb_lidar_upload returned after its last kernel)
    int taken = 0;
    const int begin = h->lid_cursor;
    if (begin < h->lid_n) {
        FLB_CUDA(h, h->lid_win.reserve(1));
        int* d_taken = h->lid_win.p;
        FLB_CUDA(h, h->pin_out.reserve(64));
        {
            LaunchScope ls(h, FAM_OTHER);
            k_lidar_window<<<1, 1, 0, h->stream>>>(h->lid_cloud.p, begin, h->lid_n, pcl_offset_time, d_taken);
            FLB_CUDA(h, cudaGetLastError());
        }
        FLB_CUDA(h, cudaMemcpyAsync(h->pin_out.p, d_taken, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        std::memcpy(&taken, h->pin_out.p, sizeof(int));
    }
    if (out_xyz && capacity_points < taken)
        return fail(h, FLB_ERR_INVALID, "flb_imu_undistort_lidar: capacity %d < the %d points of this update", capacity_points, taken);
    const int rc = imu_undistort_core(h, "flb_imu_undistort_lidar", prm, carry, v_imu, n_imu, pcl_beg_time, pcl_end_time, nullptr, 4, 3,
                                      h->lid_cloud.p + begin, taken, out_xyz, poses_out, n_poses_out);
    if (rc) return rc;
    h->lid_cursor = is_lidar_end ? 0 : begin + taken;                             // :638, :643-646
    if (n_taken) *n_taken = taken;
    return FLB_OK;
}

int flb_visual_candidates(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* world_xyz, int n, int stride,
                          int grid_size, int border, float* map_value, int* winner) {
    FLB_CHECK_H(h);
    if (!Rcw || !Pcw || n < 0 || (n > 0 && !world_xyz) || stride < 3 || grid_size < 1 || border < 0 || !map_value || !winner)
        return fail(h, FLB_ERR_INVALID, "flb_visual_candidates: bad arguments");
    { int rc = vio_image_check(h, "flb_visual_candidates"); if (rc) return rc; }
    const int gw = h->img_w / grid_size, gh = h->img_h / grid_size, ncell = gw * gh;      // :55-57
    if (ncell < 1) return fail(h, FLB_ERR_INVALID, "flb_visual_candidates: grid_size larger than the image");
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }                           // the image upload has landed
    const size_t n1 = (size_t)std::max(n, 1);
    FLB_CUDA(h, h->vm_key.reserve((size_t)ncell));
    FLB_CUDA(h, h->vm_val.reserve((size_t)ncell));
    FLB_CUDA(h, h->vm_win.reserve((size_t)ncell));
    FLB_CUDA(h, h->vm_pts.reserve(n1 * 3));
    FLB_CUDA(h, h->vm_pose.reserve(12));
    void* stv = nullptr;
    const size_t st_bytes = n1 * 3 * sizeof(float) + (size_t)ncell * sizeof(float) + 12 * sizeof(double);
    FLB_CUDA(h, h->st_scan.acquire(st_bytes, &stv));
    double* st_pose = static_cast<double*>(stv);
    std::memcpy(st_pose, Rcw, 9 * sizeof(double));
    std::memcpy(st_pose + 9, Pcw, 3 * sizeof(double));
    float* st_val = reinterpret_cast<float*>(st_pose + 12);
    std::memcpy(st_val, map_value, (size_t)ncell * sizeof(float));
    float* st_pts = st_val + ncell;
    pack_points(st_pts, world_xyz, n, stride);
    FLB_CUDA(h, cudaMemcpyAsync(h->vm_pose.p, st_pose, 12 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(h->vm_val.p, st_val, (size_t)ncell * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    if (n > 0) FLB_CUDA(h, cudaMemcpyAsync(h->vm_pts.p, st_pts, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_scan.mark(h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vmap_seed<<<(ncell + 255) / 256, 256, 0, h->stream>>>(h->vm_val.p, ncell, h->vm_key.p);
        if (n > 0)
            k_vmap_candidates<<<(n + 127) / 128, 128, 0, h->stream>>>(h->cam, h->vm_pose.p, h->img.p, h->vm_pts.p, n, grid_size, gh, border,
                                                                      h->vm_key.p);
        k_vmap_resolve<<<(ncell + 255) / 256, 256, 0, h->stream>>>(h->vm_key.p, ncell, h->vm_val.p, h->vm_win.p);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 2;
    }
    FLB_CUDA(h, h->pin_out.reserve((size_t)ncell * (sizeof(float) + sizeof(int))));
    char* po = static_cast<char*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(po, h->vm_val.p, (size_t)ncell * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + (size_t)ncell * sizeof(float), h->vm_win.p, (size_t)ncell * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    std::memcpy(map_value, po, (size_t)ncell * sizeof(float));
    std::memcpy(winner, po + (size_t)ncell * sizeof(float), (size_t)ncell * sizeof(int));
    return FLB_OK;
}

// pcl::VoxelGrid of n >= 1 finite points already on the device (xyz, packed): k_bbox -> k_vg_keys -> radix sort ->
// k_vg_heads -> scan -> k_vg_centroids, enqueued on `stream`, nothing read back.  The centroids go to `out` in ascending
// leaf index; s.box[0..5] = the box, s.box[6] = PCL's index-overflow flag, s.box[7] = the leaf count.  flb_voxel_grid
// runs it on the scan slot's scratch, flb_vmap_select_cloud on buffers of its own.
struct VgScratch {
    unsigned *keys, *keys_sorted;
    int *vals, *vals_sorted, *head, *rank, *box;
};
static int voxel_grid_dev(flb_handle* h, const float* xyz, int n, float leaf, const VgScratch& s, float* out) {
    const int init[8] = {0x7fffffff, 0x7fffffff, 0x7fffffff, (int)0x80000000, (int)0x80000000, (int)0x80000000, 0, 0};
    FLB_CUDA(h, cudaMemcpyAsync(s.box, init, sizeof(init), cudaMemcpyHostToDevice, h->stream));
    const float inv_leaf = 1.0f / leaf;                              // inverse_leaf_size_ = Array4f::Ones() / leaf_size_
    const int g = (n + 255) / 256;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_bbox<<<std::min(g, 4 * std::max(h->num_sms, 1)), 256, 0, h->stream>>>(xyz, n, s.box);
        k_vg_keys<<<g, 256, 0, h->stream>>>(xyz, n, s.box, inv_leaf, s.keys, s.vals, s.box + 6);
        FLB_CUDA(h, cudaGetLastError());
    }
    size_t t1 = 0, t2 = 0;
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, t1, s.keys, s.keys_sorted, s.vals, s.vals_sorted, n, 0, 31, h->stream));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, t2, s.head, s.rank, n, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(std::max(t1, t2)));
    FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->cub_tmp.p, t1, s.keys, s.keys_sorted, s.vals, s.vals_sorted, n, 0, 31, h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vg_heads<<<g, 256, 0, h->stream>>>(s.keys_sorted, n, s.head);
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(h->cub_tmp.p, t2, s.head, s.rank, n, h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vg_centroids<<<g, 256, 0, h->stream>>>(xyz, s.keys_sorted, s.vals_sorted, s.head, s.rank, n, out, s.box + 7);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 8;
    }
    return FLB_OK;
}

int flb_voxel_grid(flb_handle* h, const float* xyz, int n, int stride, float leaf, float* out_xyz, int capacity, int* n_out) {
    FLB_CHECK_H(h);
    if (n < 0 || (n > 0 && !xyz) || stride < 3 || !(leaf > 0) || !n_out || capacity < 0 || (capacity > 0 && !out_xyz))
        return fail(h, FLB_ERR_INVALID, "flb_voxel_grid: bad arguments");
    *n_out = 0;
    if (n == 0) return FLB_OK;
    void* stv = nullptr;
    FLB_CUDA(h, h->st_scan.acquire((size_t)n * 3 * sizeof(float), &stv));
    float* st = static_cast<float*>(stv);
    pack_points(st, xyz, n, stride);
    float lo[3];
    if (fold_points<false>(st, n, lo, nullptr))
        return fail(h, FLB_ERR_INVALID, "flb_voxel_grid: non-finite coordinate at point %d", first_bad_point(st, n, INFINITY));
    FLB_CUDA(h, h->scan_raw.reserve((size_t)n * 3));
    FLB_CUDA(h, h->skeys.reserve(n));
    FLB_CUDA(h, h->skeys_sorted.reserve(n));
    FLB_CUDA(h, h->svals.reserve(n));
    FLB_CUDA(h, h->svals_sorted.reserve(n));
    FLB_CUDA(h, h->dead_before.reserve((size_t)2 * n + 2));      // head flags | ranks
    FLB_CUDA(h, h->map_comb.reserve((size_t)n * 3));             // centroids
    FLB_CUDA(h, h->bbox_dev.reserve(8));
    FLB_CUDA(h, cudaMemcpyAsync(h->scan_raw.p, st, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_scan.mark(h->stream));
    const VgScratch vs{h->skeys.p, h->skeys_sorted.p, h->svals.p, h->svals_sorted.p, h->dead_before.p, h->dead_before.p + n, h->bbox_dev.p};
    { int rcv = voxel_grid_dev(h, h->scan_raw.p, n, leaf, vs, h->map_comb.p); if (rcv) return rcv; }
    int tail[2] = {0, 0};
    FLB_CUDA(h, cudaMemcpyAsync(tail, h->bbox_dev.p + 6, sizeof(tail), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (tail[0]) return fail(h, FLB_ERR_INVALID, "flb_voxel_grid: leaf size too small for the cloud's extent (index overflow, as PCL warns)");
    *n_out = tail[1];
    const int m = std::min(tail[1], capacity);
    if (m > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(out_xyz, h->map_comb.p, (size_t)m * 3 * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    h->N = 0;                                    // the scan slot was used as scratch
    h->scan_valid = false;
    h->last_pass_valid = false;
    if (h->ef_state == flb_handle::kEfPending) h->ef_state = flb_handle::kEfLost;
    return FLB_OK;
}

// The device half of flb_scan_upload, shared with flb_scan_from_undistorted: N finite packed points at xyz (on the
// device, complete before anything enqueued on `scan_stream` from here on runs), lo = their per-axis minimum.  Orders
// them into the idle set of the double-buffered scan, resets its per-point caches and swaps it in.
// The ordering runs on `scan_stream` into the slot that is NOT being read: updates of the previous frame still queued or
// running on `stream` keep their scan, and -- because the persistent kernels leave one SM free and the ordering is one
// block (k_scan_sort_block) -- this frame's upload overlaps them instead of queueing behind them.
static int scan_install_dev(flb_handle* h, const float* xyz, int N, const float lo[3]) {
    const size_t n1 = (size_t)std::max(N, 1);
    const int cur = h->scan_slot, alt = cur ^ 1;
    cudaStream_t ss = h->scan_stream;
    FLB_CUDA(h, cudaEventRecord(h->ev_scan_free[cur], h->stream));     // all readers of the current slot are enqueued before this
    h->scan_free_valid[cur] = true;
    if (h->scan_free_valid[alt]) FLB_CUDA(h, cudaStreamWaitEvent(ss, h->ev_scan_free[alt], 0));
    FLB_CUDA(h, h->scan_alt.reserve(n1));
    FLB_CUDA(h, h->sel_alt.reserve(n1));
    FLB_CUDA(h, h->plane_ok_alt.reserve(n1));
    FLB_CUDA(h, h->plane_alt.reserve(n1));
    const size_t nb = (n1 + kLioBlock - 1) / kLioBlock;
    FLB_CUDA(h, h->partials.reserve(std::max<size_t>(nb * lio_packed(12), h->partials.cap)));
    bool flags_done = false;
    if (N > 0) {
        // Morton order in the body frame (cell = twice the map grid's cell): spatially coherent warps at any pose
        const float inv_cell = 0.5f / (float)h->cfg.cell_size;
        // One-block ordering vs keys + device-wide radix sort + gather (identical order).  Measured on an idle H100
        // (profiles/scan_upload_probe.py, copy included): 8 k points 42 vs 77 us, 16 k 100 vs 89, 24 k 129 vs 99 -- but the
        // one-block kernel runs on the SM the persistent kernels leave free, so when an update is still running on
        // `stream` (a pipelined caller) it costs nothing, while the device-wide kernels would queue behind the update.
        // So: one block up to 16 896 points always, up to 25 600 when `stream` is busy; FLB_BLOCK_SORT=0 / 2 or
        // flb_debug_set_scan_sort force the device-wide / one-block path.
        static const int env_block_sort = [] { const char* e = getenv("FLB_BLOCK_SORT"); return e ? atoi(e) : 1; }();
        const int mode = h->scan_sort_mode ? h->scan_sort_mode : (env_block_sort == 0 ? 2 : (env_block_sort == 2 ? 1 : 0));
        bool use_block = N <= 1024 * 25 && mode != 2;
        if (use_block && mode == 0 && N > 512 * 33) {
            const cudaError_t q = cudaStreamQuery(h->stream);
            (void)cudaGetLastError();
            use_block = (q == cudaErrorNotReady);
        }
        if (use_block) {
            LaunchScope ls(h, FAM_OTHER);
            int rcs = N <= 512 * 17   ? launch_scan_sort_block<512, 17>(h, ss, xyz, N, lo, inv_cell)
                      : N <= 512 * 33 ? launch_scan_sort_block<512, 33>(h, ss, xyz, N, lo, inv_cell)
                                      : launch_scan_sort_block<1024, 25>(h, ss, xyz, N, lo, inv_cell);
            if (rcs) return rcs;
            flags_done = true;
        } else {
            FLB_CUDA(h, h->skeys.reserve(n1));
            FLB_CUDA(h, h->skeys_sorted.reserve(n1));
            FLB_CUDA(h, h->svals.reserve(n1));
            FLB_CUDA(h, h->svals_sorted.reserve(n1));
            const int g = (N + 255) / 256;
            {
                LaunchScope ls(h, FAM_OTHER);
                k_scan_keys<<<g, 256, 0, ss>>>(xyz, N, lo[0], lo[1], lo[2], inv_cell, h->skeys.p, h->svals.p);
                FLB_CUDA(h, cudaGetLastError());
            }
            size_t tmp_bytes = 0;
            FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, h->skeys.p, h->skeys_sorted.p, h->svals.p,
                                                        h->svals_sorted.p, N, 0, 24, ss));
            FLB_CUDA(h, h->scan_cub_tmp.reserve(tmp_bytes));
            FLB_CUDA(h, cub::DeviceRadixSort::SortPairs(h->scan_cub_tmp.p, tmp_bytes, h->skeys.p, h->skeys_sorted.p, h->svals.p,
                                                        h->svals_sorted.p, N, 0, 24, ss));
            h->launches += 3;
            {
                LaunchScope ls(h, FAM_OTHER);
                k_scan_gather<<<g, 256, 0, ss>>>(xyz, N, h->svals_sorted.p, h->scan_alt.p);
                FLB_CUDA(h, cudaGetLastError());
            }
        }
    }
    if (!flags_done) {
        // point_selected_surf.resize(N, true) (src/laserMapping.cpp:1469)
        FLB_CUDA(h, cudaMemsetAsync(h->sel_alt.p, 1, n1, ss));
        FLB_CUDA(h, cudaMemsetAsync(h->plane_ok_alt.p, 0, n1, ss));
    }
    FLB_CUDA(h, cudaEventRecord(h->ev_scan_ready, ss));
    FLB_CUDA(h, cudaStreamWaitEvent(h->stream, h->ev_scan_ready, 0));
    std::swap(h->scan, h->scan_alt);
    std::swap(h->sel, h->sel_alt);
    std::swap(h->plane_ok, h->plane_ok_alt);
    std::swap(h->plane, h->plane_alt);
    h->scan_slot = alt;
    h->N = N;     // enqueue-only: everything later on this handle's stream is ordered after the upload
    h->scan_valid = true;
    h->scan_gen++;
    h->last_pass_valid = false;
    return FLB_OK;
}

int flb_scan_upload(flb_handle* h, const float* body_xyz, int N, int stride) {
    FLB_CHECK_H(h);
    if ((!body_xyz && N != 0) || N < 0 || stride < 3) return fail(h, FLB_ERR_INVALID, "flb_scan_upload: bad arguments");
    const size_t n1 = (size_t)std::max(N, 1);
    void* stv = nullptr;
    FLB_CUDA(h, h->st_scan.acquire(n1 * 3 * sizeof(float), &stv));
    float* st = static_cast<float*>(stv);
    const bool direct = N > 0 && stride == 3 && is_pinned(body_xyz);      // page-locked packed source: no staging copy
    if (direct) st = const_cast<float*>(body_xyz);
    else pack_points(st, body_xyz, N, stride);
    float lo[3];
    if (fold_points<false>(st, N, lo, nullptr)) return fail(h, FLB_ERR_INVALID, "flb_scan_upload: non-finite coordinate");
    // The copy runs on `scan_stream`, ahead of the ordering that reads it (the previous upload's ordering, which read
    // scan_raw too, is earlier on the same stream).  scan_raw / skeys / svals double as flb_voxel_grid's scratch on
    // `stream`; that call ends with a stream synchronise.
    FLB_CUDA(h, h->scan_raw.reserve(n1 * 3));
    if (N > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(h->scan_raw.p, st, (size_t)N * 3 * sizeof(float), cudaMemcpyHostToDevice, h->scan_stream));
        if (!direct) FLB_CUDA(h, h->st_scan.mark(h->scan_stream));
    }
    return scan_install_dev(h, h->scan_raw.p, N, lo);
}

// downSizeFilterSurf.setInputCloud(feats_undistort); downSizeFilterSurf.filter(*feats_down_body) (src/laserMapping.cpp:
// 1398-1399) followed by flb_scan_upload, on the device.  The undistortion output {x, y, z, offset} is packed into sf_xyz
// (k_cloud_pack, which also flags a non-finite point), filtered by voxel_grid_dev into sf_down in buffers of this call's
// own, and k_cloud_bounds folds the centroids' bounds into the record; one read of the record (non-finite flags, PCL's
// overflow flag, leaf count, the centroids' minimum = the Morton keys' origin) decides the errors, then the centroids are
// installed exactly as flb_scan_upload installs the host copy of the same floats.
//   Fences.  sf_down is the ordering's input on `scan_stream`.  Every install ends by making `stream` wait for its
// ordering (ev_scan_ready), so the filter of a later call, enqueued on `stream` after that, cannot overwrite sf_down
// under an ordering still reading it.  The other way round, the ordering of this call is enqueued on `scan_stream` only
// after the host has waited for the record read, which `stream` runs after the filter: the centroids are complete
// before the ordering can start, with no cross-stream wait.
int flb_scan_from_undistorted(flb_handle* h, float leaf, int* n_out) {
    FLB_CHECK_H(h);
    if (n_out) *n_out = 0;
    if (!(leaf > 0)) return fail(h, FLB_ERR_INVALID, "flb_scan_from_undistorted: bad arguments (leaf > 0)");
    if (h->comm || h->p2p.world > 0)
        return fail(h, FLB_ERR_STATE, "flb_scan_from_undistorted: single GPU only (each rank holds only its shard of the scan)");
    if (h->undist_n < 0)
        return fail(h, FLB_ERR_STATE, "flb_scan_from_undistorted: no flb_imu_undistort output (none yet, or the last call failed)");
    const int n = h->undist_n;
    float lo[3] = {0, 0, 0};
    int m = 0;
    if (n > 0) {
        FLB_CUDA(h, h->sf_xyz.reserve((size_t)n * 3));
        FLB_CUDA(h, h->sf_down.reserve((size_t)n * 3));
        FLB_CUDA(h, h->sf_keys.reserve(n));
        FLB_CUDA(h, h->sf_keys_sorted.reserve(n));
        FLB_CUDA(h, h->sf_vals.reserve(n));
        FLB_CUDA(h, h->sf_vals_sorted.reserve(n));
        FLB_CUDA(h, h->sf_heads.reserve((size_t)2 * n));
        FLB_CUDA(h, h->sf_rec.reserve(kSfRecWords));
        FLB_CUDA(h, h->pin_out.reserve(kSfRecWords * sizeof(unsigned)));
        unsigned* rec_in = h->sf_rec.p + kSfRecInput;
        unsigned* rec_c = h->sf_rec.p + kSfRecCentroids;
        int* box = reinterpret_cast<int*>(h->sf_rec.p + kSfRecBox);   // k_bbox box | overflow | leaf count
        FLB_CUDA(h, cudaMemsetAsync(h->sf_rec.p, 0, kSfRecBox * sizeof(unsigned), h->stream));
        {
            LaunchScope ls(h, FAM_OTHER);
            k_cloud_pack<false><<<(n + 255) / 256, 256, 0, h->stream>>>(h->undist_pts, n, h->sf_xyz.p, rec_in);
            FLB_CUDA(h, cudaGetLastError());
        }
        const VgScratch vs{h->sf_keys.p, h->sf_keys_sorted.p, h->sf_vals.p, h->sf_vals_sorted.p, h->sf_heads.p, h->sf_heads.p + n, box};
        { int rcv = voxel_grid_dev(h, h->sf_xyz.p, n, leaf, vs, h->sf_down.p); if (rcv) return rcv; }
        {
            LaunchScope ls(h, FAM_OTHER);
            k_cloud_bounds<<<(n + 255) / 256, 256, 0, h->stream>>>(h->sf_down.p, n, box + 7, rec_c);
            FLB_CUDA(h, cudaGetLastError());
        }
        unsigned* rec = static_cast<unsigned*>(h->pin_out.p);
        FLB_CUDA(h, cudaMemcpyAsync(rec, h->sf_rec.p, kSfRecWords * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        if (rec[kSfRecInput + kScanRecBad]) return fail(h, FLB_ERR_INVALID, "flb_scan_from_undistorted: non-finite coordinate");
        if (rec[kSfRecBox + 6])
            return fail(h, FLB_ERR_INVALID, "flb_scan_from_undistorted: leaf size too small for the cloud's extent (index overflow, as PCL warns)");
        if (rec[kSfRecCentroids + kScanRecBad]) return fail(h, FLB_ERR_INVALID, "flb_scan_from_undistorted: non-finite centroid");
        m = (int)rec[kSfRecBox + 7];
        float hi[3];
        scan_rec_bounds(rec + kSfRecCentroids, lo, hi);
    }
    { int rci = scan_install_dev(h, h->sf_down.p, m, lo); if (rci) return rci; }
    if (n_out) *n_out = m;
    return FLB_OK;
}

// ikdtree.Build(feats_down_body->points) of the first frame (src/laserMapping.cpp:1411-1419) from the scan on the device:
// k_cloud_pack scatters the ordered scan back to the caller's order into map_raw and folds its bounds, and the grid is
// built as flb_map_upload builds it from the same points.
int flb_map_upload_scan(flb_handle* h) {
    FLB_CHECK_H(h);
    if (h->comm || h->p2p.world > 0)
        return fail(h, FLB_ERR_STATE, "flb_map_upload_scan: single GPU only (each rank holds only its shard of the scan)");
    if (!h->scan_valid) return fail(h, FLB_ERR_STATE, "flb_map_upload_scan: no scan uploaded since the last flb_voxel_grid (or ever)");
    const int M = h->N;
    if (M < 1) return fail(h, FLB_ERR_INVALID, "flb_map_upload_scan: the scan is empty (M=%d)", M);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    FLB_CUDA(h, h->map_raw.reserve((size_t)M * 3));
    FLB_CUDA(h, h->add_rec.reserve(kScanRecWords));
    FLB_CUDA(h, h->pin_out.reserve(kScanRecWords * sizeof(unsigned)));
    FLB_CUDA(h, cudaMemsetAsync(h->add_rec.p, 0, kScanRecWords * sizeof(unsigned), h->stream));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_cloud_pack<true><<<(M + 255) / 256, 256, 0, h->stream>>>(h->scan.p, M, h->map_raw.p, h->add_rec.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    unsigned* rec = static_cast<unsigned*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(rec, h->add_rec.p, kScanRecWords * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    scan_rec_bounds(rec, h->map_lo, h->map_hi);      // (both installs refuse non-finite points: the record has no bad flag set)
    int rc = rebuild_grid(h, M);
    if (rc) return rc;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_knn(flb_handle* h, const float* q, int nq, int* idx, float* d2) {
    FLB_CHECK_H(h);
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_knn: no map uploaded");
    if (!q || !idx || !d2 || nq < 0) return fail(h, FLB_ERR_INVALID, "flb_knn: bad arguments");
    if (nq == 0) return FLB_OK;
    DevBuf<float> dq, dd;
    DevBuf<int> di;
    FLB_CUDA(h, dq.reserve((size_t)nq * 3));
    FLB_CUDA(h, dd.reserve((size_t)nq * kMatch));
    FLB_CUDA(h, di.reserve((size_t)nq * kMatch));
    FLB_CUDA(h, cudaMemcpyAsync(dq.p, q, (size_t)nq * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    {
        LaunchScope ls(h, FAM_LIO_KNN);
        if (h->sparse) k_knn<true><<<(nq + 127) / 128, 128, 0, h->stream>>>(h->grid, cell_index(h), h->map_pts.p, dq.p, nq, di.p, dd.p);
        else k_knn<false><<<(nq + 127) / 128, 128, 0, h->stream>>>(h->grid, h->cell_start.p, h->map_pts.p, dq.p, nq, di.p, dd.p);
    }
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(idx, di.p, (size_t)nq * kMatch * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d2, dd.p, (size_t)nq * kMatch * sizeof(float), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    dq.release(); dd.release(); di.release();
    if (e != cudaSuccess) return fail(h, FLB_ERR_CUDA, "flb_knn: %s", cudaGetErrorString(e));
    return FLB_OK;
}

// ---------------------------------------------------------------------------------------
int flb_lio_pass(flb_handle* h, const flb_lio_params* prm, const double R[9], const double p[3], int rematch, int width,
                 flb_normal_eq* out) {
    FLB_CHECK_H(h);
    if (!prm || !R || !p || !out || (width != 6 && width != 12)) return fail(h, FLB_ERR_INVALID, "flb_lio_pass: bad arguments");
    if (h->M <= 0 || h->N <= 0) return fail(h, FLB_ERR_STATE, "flb_lio_pass: map and scan must be uploaded first");
    const int N = h->N;
    FLB_CUDA(h, h->x_world.reserve((size_t)N * 3));
    FLB_CUDA(h, h->x_nn_idx.reserve((size_t)N * kMatch));
    FLB_CUDA(h, h->x_nn_d2.reserve((size_t)N * kMatch));
    FLB_CUDA(h, h->x_pd2.reserve(N));
    FLB_CUDA(h, h->x_pabcd.reserve((size_t)N * 4));
    FLB_CUDA(h, h->x_rowmask.reserve(N));
    FLB_CUDA(h, h->x_rows.reserve((size_t)N * 12));
    FLB_CUDA(h, h->x_meas.reserve(N));
    LioParamsDev d;
    to_dev_params(prm, d);
    { int rcp = upload_pose(h, h->pose12.p, R, p); if (rcp) return rcp; }
    LioArgs a = make_lio_args(h, d, handle_frame(h));
    a.force_rematch = rematch ? 1 : 0;
    a.pose_override = h->pose12.p;
    a.x_world = h->x_world.p;
    a.x_nn_idx = h->x_nn_idx.p;
    a.x_nn_d2 = h->x_nn_d2.p;
    a.x_pabcd = h->x_pabcd.p;
    a.x_pd2 = h->x_pd2.p;
    a.x_rowmask = h->x_rowmask.p;
    a.x_rows = h->x_rows.p;
    a.x_meas = h->x_meas.p;
    int rc = launch_lio_pass(h, a, width, rematch != 0);
    if (rc) return rc;
    note_lio_pass(h);
    const int K = lio_packed(width);
    if (h->comm) {
        rc = allreduce_packed(h, h->partials.p, lio_nblocks(h), K);
        if (rc) return rc;
    } else {
        LaunchScope ls(h, FAM_SOLVE);
        k_reduce_only<<<1, 32, 0, h->stream>>>(h->partials.p, lio_nblocks(h), K, h->packed.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    double* po = static_cast<double*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(po, h->packed.p, K * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    std::memset(out, 0, sizeof(*out));
    out->width = width;
    unpack_normal_eq(po, width, out->HTH, out->HTh);
    out->n_eff = (int)po[K - 2];
    out->sum_abs_res = po[K - 1];
    h->last_pass_width = width;
    h->last_pass_valid = true;
    return FLB_OK;
}

int flb_lio_export(flb_handle* h, float* world_xyz, int* nn_idx, float* nn_d2, float* pabcd, float* pd2, uint8_t* selected,
                   double* rows, double* meas, int* sel_idx, int* n_rows) {
    FLB_CHECK_H(h);
    if (!h->last_pass_valid) return fail(h, FLB_ERR_STATE, "flb_lio_export: no flb_lio_pass to export");
    const int N = h->N, W = h->last_pass_width;
    cudaStream_t s = h->stream;
    if (world_xyz) FLB_CUDA(h, cudaMemcpyAsync(world_xyz, h->x_world.p, (size_t)N * 3 * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (nn_idx) FLB_CUDA(h, cudaMemcpyAsync(nn_idx, h->x_nn_idx.p, (size_t)N * kMatch * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (nn_d2) FLB_CUDA(h, cudaMemcpyAsync(nn_d2, h->x_nn_d2.p, (size_t)N * kMatch * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (pabcd) FLB_CUDA(h, cudaMemcpyAsync(pabcd, h->x_pabcd.p, (size_t)N * 4 * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (pd2) FLB_CUDA(h, cudaMemcpyAsync(pd2, h->x_pd2.p, (size_t)N * sizeof(float), cudaMemcpyDeviceToHost, s));
    std::vector<unsigned char> mask(N);
    FLB_CUDA(h, cudaMemcpyAsync(mask.data(), h->x_rowmask.p, N, cudaMemcpyDeviceToHost, s));
    std::vector<double> hrows, hmeas;
    if (rows || meas) {
        hrows.resize((size_t)N * W);
        hmeas.resize(N);
        FLB_CUDA(h, cudaMemcpyAsync(hrows.data(), h->x_rows.p, (size_t)N * W * sizeof(double), cudaMemcpyDeviceToHost, s));
        FLB_CUDA(h, cudaMemcpyAsync(hmeas.data(), h->x_meas.p, (size_t)N * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    FLB_CUDA(h, cudaStreamSynchronize(s));
    // order-preserving compaction == laserCloudOri / corr_normvect (src/laserMapping.cpp:1588-1600)
    int n = 0;
    for (int i = 0; i < N; ++i) {
        if (selected) selected[i] = mask[i];
        if (!mask[i]) continue;
        if (rows) std::memcpy(rows + (size_t)n * W, hrows.data() + (size_t)i * W, W * sizeof(double));
        if (meas) meas[n] = hmeas[i];
        if (sel_idx) sel_idx[n] = i;
        ++n;
    }
    if (n_rows) *n_rows = n;
    return FLB_OK;
}

int flb_state_upload(flb_handle* h, const flb_state18* x, const flb_state18* x_prop) {
    FLB_CHECK_H(h);
    if (!x || !x_prop) return fail(h, FLB_ERR_INVALID, "flb_state_upload: null state");
    void* stv = nullptr;
    FLB_CUDA(h, h->st_state.acquire(2 * sizeof(State18), &stv));
    State18* st = static_cast<State18*>(stv);
    std::memcpy(&st[0], x, sizeof(State18));
    std::memcpy(&st[1], x_prop, sizeof(State18));
    {
        void* dsrc = nullptr;
        FLB_CUDA(h, cudaHostGetDevicePointer(&dsrc, st, 0));
        LaunchScope ls(h, FAM_OTHER);
        k_state_install<<<1, 256, 0, h->stream>>>(static_cast<const double*>(dsrc), h->states.p);   // [0..1] and the saved pair [3..4]
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, h->st_state.mark(h->stream));
    h->state_valid = true;
    h->reset_pending = h->prior_pending = false;     // both superseded by the upload
    return FLB_OK;
}

int flb_state_reset_enqueue(flb_handle* h) {
    FLB_CHECK_H(h);
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_state_reset_enqueue: no state uploaded");
    h->prior_pending = false;            // overwritten by the reset
    h->reset_pending = true;             // performed by the next LIO kernel (or flushed as a copy by any other consumer)
    return FLB_OK;
}

int flb_state_set_prior_enqueue(flb_handle* h) {
    FLB_CHECK_H(h);
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_state_set_prior_enqueue: no state uploaded");
    { int rcf = flush_state_ops(h); if (rcf) return rcf; }      // an earlier pending reset / prior comes first
    h->prior_pending = true;             // performed by the next VIO kernel (or flushed as a copy by any other consumer)
    return FLB_OK;
}

int flb_state_download(flb_handle* h, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio) {
    FLB_CHECK_H(h);
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_state_download: no state uploaded");
    { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    char* po = static_cast<char*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(po, &h->states.p[0], sizeof(State18), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + kResLio, h->lio_ctrl.p, sizeof(LioCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + kResVio, h->vio_ctrl.p, sizeof(VioCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + kResBarrier, h->barrier.p, sizeof(GridBarrier), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return read_result(h, po, x, lio, vio);
}

// Pipelined result read-back: enqueue the copy of (state, reports) of everything enqueued so far into result slot
// `slot`, return at once; flb_state_download_wait blocks on that slot only, so frame k's result can be collected while
// frame k+1 is already uploading / running.
int flb_state_download_enqueue(flb_handle* h, int slot) {
    FLB_CHECK_H(h);
    if (slot < 0 || slot > 1) return fail(h, FLB_ERR_INVALID, "flb_state_download_enqueue: slot must be 0 or 1");
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "flb_state_download_enqueue: no state uploaded");
    { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    FLB_CUDA(h, h->pin_res[slot].reserve(kResBytes));
    if (!h->ev_res[slot]) FLB_CUDA(h, cudaEventCreateWithFlags(&h->ev_res[slot], cudaEventDisableTiming));
    char* po = static_cast<char*>(h->pin_res[slot].p);
    {
        static_assert(sizeof(State18) % 4 == 0 && sizeof(LioCtrl) % 4 == 0 && sizeof(VioCtrl) % 4 == 0 && sizeof(GridBarrier) % 4 == 0, "word copies");
        void* dout = nullptr;
        FLB_CUDA(h, cudaHostGetDevicePointer(&dout, po, 0));
        LaunchScope ls(h, FAM_OTHER);
        k_pack_result<<<1, 256, 0, h->stream>>>(&h->states.p[0], reinterpret_cast<const unsigned*>(h->lio_ctrl.p), (int)(sizeof(LioCtrl) / 4),
                                                reinterpret_cast<const unsigned*>(h->vio_ctrl.p), (int)(sizeof(VioCtrl) / 4),
                                                reinterpret_cast<const unsigned*>(h->barrier.p), (int)(sizeof(GridBarrier) / 4),
                                                static_cast<unsigned*>(dout));
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, cudaEventRecord(h->ev_res[slot], h->stream));
    h->res_pending[slot] = true;
    return FLB_OK;
}

int flb_state_download_wait(flb_handle* h, int slot, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio) {
    FLB_CHECK_H(h);
    if (slot < 0 || slot > 1 || !h->res_pending[slot]) return fail(h, FLB_ERR_STATE, "flb_state_download_wait: nothing enqueued in this slot");
    FLB_CUDA(h, cudaEventSynchronize(h->ev_res[slot]));
    h->res_pending[slot] = false;
    return read_result(h, static_cast<const char*>(h->pin_res[slot].p), x, lio, vio);
}

int flb_lio_update_enqueue(flb_handle* h, const flb_lio_params* prm) {
    FLB_CHECK_H(h);
    if (!prm) return fail(h, FLB_ERR_INVALID, "null params");
    return enqueue_lio_update(h, prm);
}

int flb_vio_update_enqueue(flb_handle* h, const flb_vio_params* prm) {
    FLB_CHECK_H(h);
    if (!prm) return fail(h, FLB_ERR_INVALID, "null params");
    return enqueue_vio_update(h, prm);
}

// One frame in one call: uploads + both updates enqueued + (optionally) the pipelined read-back.
int flb_frame_enqueue(flb_handle* h, const flb_frame_inputs* in, const flb_lio_params* lprm, const flb_vio_params* vprm, int result_slot) {
    FLB_CHECK_H(h);
    if (!in || !lprm || !in->x || !in->x_prop) return fail(h, FLB_ERR_INVALID, "flb_frame_enqueue: null argument");
    int rc = flb_scan_upload(h, in->scan_xyz, in->n_scan, in->scan_stride);
    if (rc) return rc;
    rc = flb_state_upload(h, in->x, in->x_prop);
    if (rc) return rc;
    rc = enqueue_lio_update(h, lprm);
    if (rc) return rc;
    if (vprm) {
        if (in->gray) { rc = flb_image_upload(h, in->gray, in->width, in->height, in->stride_bytes); if (rc) return rc; }
        if (in->patch_pos) { rc = flb_patches_upload(h, in->patch_pos, in->patch, in->search_level, in->Pn); if (rc) return rc; }
        rc = flb_state_set_prior_enqueue(h);          // state_propagat = state (src/laserMapping.cpp:1292), zero-motion propagation
        if (rc) return rc;
        rc = enqueue_vio_update(h, vprm);
        if (rc) return rc;
    }
    if (result_slot >= 0) return flb_state_download_enqueue(h, result_slot);
    return FLB_OK;
}

int flb_lio_update(flb_handle* h, const flb_lio_params* prm, flb_state18* x, const flb_state18* x_prop, flb_lio_report* rep) {
    FLB_CHECK_H(h);
    if (!prm || !x || !x_prop) return fail(h, FLB_ERR_INVALID, "flb_lio_update: null argument");
    int rc = flb_state_upload(h, x, x_prop);
    if (rc) return rc;
    rc = enqueue_lio_update(h, prm);
    if (rc) return rc;
    flb_lio_report r{};
    rc = flb_state_download(h, x, &r, nullptr);
    if (rc) return rc;
    if (rep) *rep = r;
    if (r.status != 0) return fail(h, r.status, "flb_lio_update: device reported status %d (singular normal matrix?)", r.status);
    return FLB_OK;
}

// ---------------------------------------------------------------------------------------
int flb_lio_update_ikfom(flb_handle* h, const flb_ikfom_params* prm, flb_state_ikfom* x, flb_ikfom_report* rep) {
    FLB_CHECK_H(h);
    if (!prm || !x) return fail(h, FLB_ERR_INVALID, "flb_lio_update_ikfom: null argument");
    if (prm->max_iteration < 0) return fail(h, FLB_ERR_INVALID, "max_iteration < 0");
    if (h->M <= 0 || h->N <= 0) return fail(h, FLB_ERR_STATE, "flb_lio_update_ikfom: map and scan must be uploaded first");
    if (h->comm || h->p2p.world > 1) return fail(h, FLB_ERR_STATE, "flb_lio_update_ikfom: single-GPU only");
    void* stv = nullptr;
    FLB_CUDA(h, h->st_state.acquire(sizeof(StateIkfom), &stv));
    std::memcpy(stv, x, sizeof(StateIkfom));
    FLB_CUDA(h, cudaMemcpyAsync(&h->ik_states.p[0], stv, sizeof(StateIkfom), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_state.mark(h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(&h->ik_states.p[1], &h->ik_states.p[0], sizeof(StateIkfom), cudaMemcpyDeviceToDevice, h->stream));
    LioParamsDev d{};            // the extrinsic comes from the state every pass; only plane_thr / grid matter here
    LioArgs a = make_lio_args(h, d, handle_frame(h));
    IkfomSolveArgs s{};
    s.state = &h->ik_states.p[0];
    s.state_prop = &h->ik_states.p[1];
    s.ctrl = h->ik_ctrl.p;
    s.prm.R = prm->laser_point_cov;
    s.prm.max_iteration = prm->max_iteration;
    std::memcpy(s.prm.limit, prm->limit, sizeof(s.prm.limit));
    const int occ_ik = h->sparse ? h->occ_ik_sparse : h->occ_ik;
    const int cap = std::max(1, occ_ik * h->num_sms);
    const int want = std::min(cap, std::max(h->num_sms, std::min(2, occ_ik) * h->num_sms));
    const int grid = std::max(1, std::min((h->N + 31) / 32, want));
    FLB_CUDA(h, h->partials.reserve(std::max<size_t>((size_t)grid * lio_packed(12), h->partials.cap)));
    a.partials = h->partials.p;
    s.partials = h->partials.p;
    s.nblocks = grid;
    GridBarrier* bar = h->barrier.p;
    void* args[] = {&a, &s, &bar};
    {
        LaunchScope ls(h, FAM_LIO_KNN);
        void* kern = h->sparse ? (void*)k_lio_update_ikfom_persistent<kLioBlock, true> : (void*)k_lio_update_ikfom_persistent<kLioBlock, false>;
        FLB_CUDA(h, cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kLioBlock), args, 0,
                                                h->stream));
    }
    h->last_pass_valid = false;
    note_lio_pass(h);                    // the last h_share_model evaluation's sel bytes
    FLB_CUDA(h, h->pin_out.reserve(sizeof(StateIkfom) + sizeof(IkfomCtrl) + sizeof(GridBarrier)));
    char* po = static_cast<char*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(po, &h->ik_states.p[0], sizeof(StateIkfom), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + sizeof(StateIkfom), h->ik_ctrl.p, sizeof(IkfomCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(po + sizeof(StateIkfom) + sizeof(IkfomCtrl), h->barrier.p, sizeof(GridBarrier), cudaMemcpyDeviceToHost,
                                h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    { int rcw = watchdog_check(h, po + sizeof(StateIkfom) + sizeof(IkfomCtrl)); if (rcw) return rcw; }
    std::memcpy(x, po, sizeof(StateIkfom));
    IkfomCtrl c;
    std::memcpy(&c, po + sizeof(StateIkfom), sizeof(c));
    if (rep) {
        rep->passes = c.passes; rep->knn_passes = c.knn_passes; rep->n_eff_last = c.n_eff_last;
        rep->converged_last = c.converged_last; rep->res_mean_last = c.res_mean_last; rep->rows_total = c.rows_total;
        rep->status = c.status;
    }
    if (c.status != 0) return fail(h, c.status, "flb_lio_update_ikfom: device reported status %d", c.status);
    return FLB_OK;
}

// ---------------------------------------------------------------------------------------
int flb_image_upload(flb_handle* h, const uint8_t* gray, int width, int height, int stride) {
    FLB_CHECK_H(h);
    if (!gray || width < 16 || height < 16 || stride < width) return fail(h, FLB_ERR_INVALID, "flb_image_upload: bad arguments");
    FLB_CUDA(h, h->img_alt.reserve((size_t)width * height));
    const unsigned char* src = gray;
    const bool direct = (stride == width) && is_pinned(gray);     // page-locked caller buffer: no staging copy
    if (!direct) {
        void* stv = nullptr;
        FLB_CUDA(h, h->st_img.acquire((size_t)width * height, &stv));
        unsigned char* st = static_cast<unsigned char*>(stv);
        if (stride == width) std::memcpy(st, gray, (size_t)width * height);
        else for (int r = 0; r < height; ++r) std::memcpy(st + (size_t)r * width, gray + (size_t)r * stride, width);
        src = st;
    }
    { int rcq = vio_copy_begin(h, h->img_slot); if (rcq) return rcq; }
    FLB_CUDA(h, cudaMemcpyAsync(h->img_alt.p, src, (size_t)width * height, cudaMemcpyHostToDevice, h->copy_stream));
    if (!direct) FLB_CUDA(h, h->st_img.mark(h->copy_stream));
    { int rcq = vio_copy_end(h); if (rcq) return rcq; }
    std::swap(h->img, h->img_alt);
    std::swap(h->img_bgr, h->img_bgr_alt);
    h->img_bgr_valid = false;
    h->img_slot.slot ^= 1;
    h->img_w = width;
    h->img_h = height;
    h->last_vio_valid = false;
    return FLB_OK;
}

int flb_image_upload_bgr(flb_handle* h, const uint8_t* bgr, int width, int height, int stride_bytes, int gray_rule) {
    FLB_CHECK_H(h);
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_image_upload_bgr: flb_camera_set first");
    const int W = h->cam.width, H = h->cam.height;
    const bool halve = (width == 2 * W && height == 2 * H);
    if (!bgr || !(halve || (width == W && height == H)) || stride_bytes < 3 * width || (gray_rule != kGrayCv4 && gray_rule != kGrayCv3))
        return fail(h, FLB_ERR_INVALID, "flb_image_upload_bgr: bad arguments (%dx%d, stride %d, rule %d; camera %dx%d)", width, height,
                    stride_bytes, gray_rule, W, H);
    return image_upload_frame(h, bgr, width, height, stride_bytes, kEncBgr8, gray_rule);
}

int flb_image_upload_msg(flb_handle* h, const uint8_t* data, int width, int height, int step_bytes, int encoding, int gray_rule) {
    FLB_CHECK_H(h);
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_image_upload_msg: flb_camera_set first");
    const int W = h->cam.width, H = h->cam.height;
    const bool known = encoding >= kEncBgr8 && encoding <= kEncBayerGrbg8;
    const bool same = (width == W && height == H);
    // detect() resizes to (int)(cols * 0.5) x (int)(rows * 0.5): any other size leaves the camera's size behind
    const bool resized = !same && (width == 2 * W || width == 2 * W + 1) && (height == 2 * H || height == 2 * H + 1);
    const bool linear = resized && !(width == 2 * W && height == 2 * H);
    if (!data || !known || !(same || resized) || (gray_rule != kGrayCv4 && gray_rule != kGrayCv3) ||
        (linear && gray_rule == kGrayCv3) || (known && (int64_t)step_bytes < (int64_t)enc_bpp(encoding) * width))
        return fail(h, FLB_ERR_INVALID, "flb_image_upload_msg: bad arguments (%dx%d, step %d, encoding %d, rule %d; camera %dx%d)", width,
                    height, step_bytes, encoding, gray_rule, W, H);
    return image_upload_frame(h, data, width, height, step_bytes, encoding, gray_rule);
}

int flb_image_download(flb_handle* h, uint8_t* gray, uint8_t* bgr, int capacity_pixels, int* width, int* height) {
    FLB_CHECK_H(h);
    if (h->img_w <= 0) return fail(h, FLB_ERR_STATE, "flb_image_download: no image uploaded");
    if (bgr && !h->img_bgr_valid) return fail(h, FLB_ERR_STATE, "flb_image_download: the current image has no colour frame (flb_image_upload)");
    const size_t px = (size_t)h->img_w * h->img_h;
    if ((gray || bgr) && (capacity_pixels < 0 || (size_t)capacity_pixels < px))
        return fail(h, FLB_ERR_INVALID, "flb_image_download: capacity %d < %zu pixels", capacity_pixels, px);
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    if (gray) FLB_CUDA(h, cudaMemcpyAsync(gray, h->img.p, px, cudaMemcpyDeviceToHost, h->stream));
    if (bgr) FLB_CUDA(h, cudaMemcpyAsync(bgr, h->img_bgr.p, px * 3, cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (width) *width = h->img_w;
    if (height) *height = h->img_h;
    return FLB_OK;
}

int flb_patches_upload(flb_handle* h, const double* pos, const float* patch, const int* search_level, int Pn) {
    FLB_CHECK_H(h);
    if (Pn < 0 || (Pn > 0 && (!pos || !patch || !search_level))) return fail(h, FLB_ERR_INVALID, "flb_patches_upload: bad arguments");
    for (int i = 0; i < Pn; ++i)
        if (search_level[i] < 0 || search_level[i] > 2) return fail(h, FLB_ERR_INVALID, "search_level[%d] = %d outside [0,2]", i, search_level[i]);
    const size_t n = (size_t)std::max(Pn, 1);
    FLB_CUDA(h, h->patch_pos_alt.reserve(n * 3));
    FLB_CUDA(h, h->patch_ref_alt.reserve(n * 192));
    FLB_CUDA(h, h->patch_level_alt.reserve(n));
    FLB_CUDA(h, h->errors.reserve(2 * n));
    h->err_stride = (int)n;
    const int nb = (Pn + 7) / 8;
    FLB_CUDA(h, h->partials.reserve(std::max<size_t>((size_t)std::max(nb, 1) * kVioPacked, h->partials.cap)));
    const size_t bytes = n * (3 * sizeof(double) + 192 * sizeof(float) + sizeof(int)) + 16;
    if (Pn > 0) {
        const bool direct = is_pinned(pos) && is_pinned(patch) && is_pinned(search_level);
        { int rcq = vio_copy_begin(h, h->patch_slot); if (rcq) return rcq; }
        if (direct) {
            FLB_CUDA(h, cudaMemcpyAsync(h->patch_pos_alt.p, pos, (size_t)Pn * 3 * sizeof(double), cudaMemcpyHostToDevice, h->copy_stream));
            FLB_CUDA(h, cudaMemcpyAsync(h->patch_ref_alt.p, patch, (size_t)Pn * 192 * sizeof(float), cudaMemcpyHostToDevice, h->copy_stream));
            FLB_CUDA(h, cudaMemcpyAsync(h->patch_level_alt.p, search_level, (size_t)Pn * sizeof(int), cudaMemcpyHostToDevice, h->copy_stream));
        } else {
            // pageable caller buffers: pack into pinned staging and hand each piece to the copy engine as soon
            // as it is packed, the reference patches (96 % of the bytes) in four slices, so that the transfer
            // runs behind the host memcpy instead of after it
            void* stv = nullptr;
            FLB_CUDA(h, h->st_patch.acquire(bytes, &stv));
            char* b = static_cast<char*>(stv);
            std::memcpy(b, pos, (size_t)Pn * 3 * sizeof(double));
            FLB_CUDA(h, cudaMemcpyAsync(h->patch_pos_alt.p, b, (size_t)Pn * 3 * sizeof(double), cudaMemcpyHostToDevice, h->copy_stream));
            char* b3 = b + (size_t)Pn * 3 * sizeof(double);
            std::memcpy(b3, search_level, (size_t)Pn * sizeof(int));
            FLB_CUDA(h, cudaMemcpyAsync(h->patch_level_alt.p, b3, (size_t)Pn * sizeof(int), cudaMemcpyHostToDevice, h->copy_stream));
            char* b2 = b3 + (((size_t)Pn * sizeof(int) + 15) & ~(size_t)15);
            const size_t total = (size_t)Pn * 192, slice = (total + 3) / 4;
            for (size_t o = 0; o < total; o += slice) {
                const size_t cnt = std::min(slice, total - o);
                std::memcpy(b2 + o * sizeof(float), patch + o, cnt * sizeof(float));
                FLB_CUDA(h, cudaMemcpyAsync(h->patch_ref_alt.p + o, b2 + o * sizeof(float), cnt * sizeof(float), cudaMemcpyHostToDevice, h->copy_stream));
            }
        }
        if (!direct) FLB_CUDA(h, h->st_patch.mark(h->copy_stream));
        { int rcq = vio_copy_end(h); if (rcq) return rcq; }
    }
    std::swap(h->patch_pos, h->patch_pos_alt);
    std::swap(h->patch_ref, h->patch_ref_alt);
    std::swap(h->patch_level, h->patch_level_alt);
    h->patch_slot.slot ^= 1;
    if (h->comm) {
        // agree on the largest shard so every rank contributes an equal-size block to ncclAllGather;
        // the padding entries stay 0.0f, and adding 0.0f to the sequential float sum is exact.
        int* dmax = reinterpret_cast<int*>(h->packed.p);
        FLB_CUDA(h, cudaMemcpyAsync(dmax, &Pn, sizeof(int), cudaMemcpyHostToDevice, h->stream));
        int r = g_nccl.AllReduce(dmax, dmax, 1, kNcclInt32, kNcclMax, h->comm, h->stream);
        if (r != 0) return fail(h, FLB_ERR_COMM, "ncclAllReduce(max Pn) failed");
        int shard = 0;
        FLB_CUDA(h, cudaMemcpyAsync(&shard, dmax, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        h->err_shard = std::max(shard, 1);
        h->err_stride = std::max(h->err_stride, h->err_shard);
        FLB_CUDA(h, h->errors.reserve(2 * (size_t)h->err_stride));
        FLB_CUDA(h, h->errors_all.reserve((size_t)h->err_shard * (size_t)h->world));
    }
    FLB_CUDA(h, cudaMemsetAsync(h->errors.p, 0, h->errors.cap * sizeof(float), h->stream));
    h->Pn = Pn;
    h->pn_on_device = false;
    h->patches_set = true;
    h->err_from_sel = false;
    h->last_vio_valid = false;
    return FLB_OK;
}

int flb_camera_set(flb_handle* h, const flb_camera* cam) {
    FLB_CHECK_H(h);
    if (!cam || cam->width < 16 || cam->height < 16 || !(std::fabs(cam->fx) > 0) || !(std::fabs(cam->fy) > 0))
        return fail(h, FLB_ERR_INVALID, "flb_camera_set: bad camera");
    CamModel c{};
    c.width = cam->width;
    c.height = cam->height;
    c.fx = cam->fx; c.fy = cam->fy; c.cx = cam->cx; c.cy = cam->cy;
    for (int i = 0; i < 5; ++i) c.d[i] = cam->d[i];
    // vikit PinholeCamera::errorMultiplier2() = |fx|, errorMultiplier() = |4 fx fy| (src/lidar_selection.cpp:58-59)
    c.jfx = std::fabs(cam->fx);
    c.jfy = std::fabs(4.0 * cam->fx * cam->fy) / (4. * c.jfx);
    h->cam = c;
    h->cam_set = true;
    return FLB_OK;
}

int flb_vio_pass(flb_handle* h, const flb_vio_params* prm, const double R[9], const double p[3], int level, flb_vio_eq* out) {
    FLB_CHECK_H(h);
    if (!prm || !R || !p || !out || level < 0 || level > 2) return fail(h, FLB_ERR_INVALID, "flb_vio_pass: bad arguments");
    { int rc = vio_image_check(h, "flb_vio_pass"); if (rc) return rc; }
    std::memset(out, 0, sizeof(*out));
    { int rcp = resolve_pn(h); if (rcp) return rcp; }
    if (h->Pn == 0) return FLB_OK;
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    const size_t Pn = h->Pn;
    FLB_CUDA(h, h->x_z.reserve(Pn * 64));
    FLB_CUDA(h, h->x_H.reserve(Pn * 64 * 6));
    VioParamsDev d;
    to_dev_params(prm, d);
    { int rcp = upload_pose(h, h->pose12.p, R, p); if (rcp) return rcp; }
    VioArgs a = make_vio_args(h, d, handle_frame(h));
    a.pose_override = h->pose12.p;
    a.force_level = level;
    a.x_z = h->x_z.p;
    a.x_H = h->x_H.p;
    const int nb = vio_nblocks(h);
    {
        LaunchScope ls(h, FAM_VIO);
        k_vio_pass<kVioBlock><<<nb, kVioBlock, 0, h->stream>>>(a);
        FLB_CUDA(h, cudaGetLastError());
    }
    {
        LaunchScope ls(h, FAM_SOLVE);
        k_reduce_only<<<1, 32, 0, h->stream>>>(h->partials.p, nb, kVioPacked, h->packed.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, h->pin_out.reserve(kVioPacked * sizeof(double) + Pn * sizeof(float)));
    double* po = static_cast<double*>(h->pin_out.p);
    float* pe = reinterpret_cast<float*>(po + kVioPacked);
    FLB_CUDA(h, cudaMemcpyAsync(po, h->packed.p, kVioPacked * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(pe, h->errors.p, Pn * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    unpack_normal_eq(po, 6, out->HTH, out->HTz);
    out->n_meas = (int64_t)po[27];
    out->skipped = (int)po[28];
    // error = sum_i errors[i] (float, patch order) / n_meas  (src/lidar_selection.cpp:852,857)
    float e = 0.0f;
    for (size_t i = 0; i < Pn; ++i) e = e + pe[i];
    out->error = e / (float)(size_t)out->n_meas;
    h->last_vio_valid = true;
    h->err_from_sel = false;
    return FLB_OK;
}

int flb_vio_export(flb_handle* h, double* z, double* H_sub, float* errors) {
    FLB_CHECK_H(h);
    if (!h->last_vio_valid) return fail(h, FLB_ERR_STATE, "flb_vio_export: no flb_vio_pass to export");
    const size_t Pn = h->Pn;
    if (z) FLB_CUDA(h, cudaMemcpyAsync(z, h->x_z.p, Pn * 64 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (H_sub) FLB_CUDA(h, cudaMemcpyAsync(H_sub, h->x_H.p, Pn * 64 * 6 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (errors) FLB_CUDA(h, cudaMemcpyAsync(errors, h->errors.p, Pn * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_vio_errors(flb_handle* h, float* errors, int capacity) {
    FLB_CHECK_H(h);
    if (!errors || capacity < 0) return fail(h, FLB_ERR_INVALID, "flb_vio_errors: bad arguments");
    { int rcp = resolve_pn(h); if (rcp) return rcp; }
    const int n = std::min(capacity, h->Pn);
    if (n == 0) return FLB_OK;
    // which half the last executed pass of the last update wrote is part of the device control block
    VioCtrl c;
    FLB_CUDA(h, cudaMemcpyAsync(&c, h->vio_ctrl.p, sizeof(VioCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    const int buf = (c.err_buf == 1) ? 1 : 0;
    FLB_CUDA(h, cudaMemcpyAsync(errors, h->errors.p + (size_t)buf * h->err_stride, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_vio_update_level(flb_handle* h, const flb_vio_params* prm, int level, float total_residual, flb_state18* x,
                         const flb_state18* x_prop, float* last_error, double* G18x6, flb_vio_report* rep) {
    FLB_CHECK_H(h);
    if (!prm || !x || !x_prop || level < 0 || level > 2) return fail(h, FLB_ERR_INVALID, "flb_vio_update_level: bad arguments");
    { int rcc = vio_image_check(h, "flb_vio_update_level"); if (rcc) return rcc; }
    if (h->comm || h->p2p.world > 1) return fail(h, FLB_ERR_STATE, "flb_vio_update_level: single GPU");
    { int rcp = resolve_pn(h); if (rcp) return rcp; }
    if (last_error) *last_error = 0.f;                               // :746 (total_points == 0 returns 0.)
    flb_vio_report r{};
    if (h->Pn == 0) { if (rep) *rep = r; return FLB_OK; }
    int rc = flb_state_upload(h, x, x_prop);
    if (rc) return rc;
    VioParamsDev d;
    to_dev_params(prm, d);
    d.single_level = 1;
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    const FrameBufs fb = handle_frame(h);
    const VioSolveArgs s = make_vio_solve_args(h, d, fb);
    const VioArgs a = make_vio_args(h, d, fb);
    {
        LaunchScope ls(h, FAM_SOLVE);
        k_vio_begin_level<<<1, 32, 0, h->stream>>>(h->vio_ctrl.p, h->Pn, level, total_residual);
        FLB_CUDA(h, cudaGetLastError());
    }
    if (prm->max_iteration > 0) h->err_from_sel = false;
    // later passes return at once when the level has ended
    { int rcl = vio_pass_loop(h, a, s, std::max(prm->max_iteration, 0)); if (rcl) return rcl; }
    if (G18x6) {
        LaunchScope ls(h, FAM_SOLVE);
        k_vio_export_gain<<<1, kLeaderBlock, 0, h->stream>>>(s, h->packed.p);
        FLB_CUDA(h, cudaGetLastError());
        FLB_CUDA(h, cudaMemcpyAsync(G18x6, h->packed.p, 108 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    }
    h->last_vio_valid = false;
    rc = flb_state_download(h, x, nullptr, &r);
    if (rc) return rc;
    if (rep) *rep = r;
    if (last_error) *last_error = r.last_error[level];               // return last_error (:901)
    if (r.status != 0) return fail(h, r.status, "flb_vio_update_level: device reported status %d", r.status);
    return FLB_OK;
}

int flb_vio_update(flb_handle* h, const flb_vio_params* prm, flb_state18* x, const flb_state18* x_prop, flb_vio_report* rep) {
    FLB_CHECK_H(h);
    if (!prm || !x || !x_prop) return fail(h, FLB_ERR_INVALID, "flb_vio_update: null argument");
    if (h->cam_set && (h->cam.width != h->img_w || h->cam.height != h->img_h))
        return fail(h, FLB_ERR_STATE, "camera / image size mismatch");
    int rc = flb_state_upload(h, x, x_prop);
    if (rc) return rc;
    rc = enqueue_vio_update(h, prm);
    if (rc) return rc;
    flb_vio_report r{};
    rc = flb_state_download(h, x, nullptr, &r);
    if (rc) return rc;
    if (rep) *rep = r;
    if (r.status != 0) return fail(h, r.status, "flb_vio_update: device reported status %d", r.status);
    return FLB_OK;
}

// ---------------------------------------------------------------------------------------
int flb_profile_start(flb_handle* h) {
    FLB_CHECK_H(h);
    for (auto& ev : h->evs) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    h->evs.clear();
    h->profiling = true;
    return FLB_OK;
}

int flb_profile_stop(flb_handle* h, double ms[4], int64_t launches[4]) {
    FLB_CHECK_H(h);
    h->profiling = false;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < 4; ++i) { if (ms) ms[i] = 0.0; if (launches) launches[i] = 0; }
    for (auto& ev : h->evs) {
        float t = 0.f;
        cudaEventElapsedTime(&t, ev.a, ev.b);
        if (ev.fam < 4) {
            if (ms) ms[ev.fam] += t;
            if (launches) launches[ev.fam] += 1;
        }
        cudaEventDestroy(ev.a);
        cudaEventDestroy(ev.b);
    }
    h->evs.clear();
    return FLB_OK;
}

int flb_trace_enable(flb_handle* h, int on) {
    FLB_CHECK_H(h);
    h->tracing = on != 0;
    FLB_CUDA(h, cudaMemsetAsync(h->trace.p, 0, 2 * kTraceLen * sizeof(unsigned long long), h->stream));
    return FLB_OK;
}

// Test aid (not part of the public header): move the pose-packet flag base, e.g. next to its wrap-around point
// (the base advances by 4096 per persistent launch and is re-based, with the packet cleared, before it overflows).
int flb_debug_set_packet_epoch(flb_handle* h, unsigned epoch) {
    FLB_CHECK_H(h);
    h->pkt_epoch = epoch;
    return FLB_OK;
}

// Tracing aid (not part of the public header): per-block / per-warp stamps of the last VIO pass,
// kVioDbg words per block.
int flb_debug_vio_stamps(flb_handle* h, unsigned long long* out, int max_blocks, int* nblocks, int* words_per_block) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    const int n = std::min(h->dbg_vio_blocks, max_blocks);
    if (n > 0) FLB_CUDA(h, cudaMemcpy(out, h->dbg_vio.p, (size_t)n * kVioDbg * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    *nblocks = n;
    *words_per_block = kVioDbg;
    return FLB_OK;
}

// Test aid: force the scan ordering path of the following uploads (0 automatic, 1 one-block kernel, 2 device-wide sort).
int flb_debug_set_scan_sort(flb_handle* h, int mode) {
    FLB_CHECK_H(h);
    if (mode < 0 || mode > 2) return fail(h, FLB_ERR_INVALID, "flb_debug_set_scan_sort: mode 0, 1 or 2");
    h->scan_sort_mode = mode;
    return FLB_OK;
}

// Test aid: cell index of the following map rebuilds (flb_map_upload, flb_map_delete_boxes, an Add_Points that leaves the
// dense grid's box) -- 0 automatic (the dense table, see rebuild_grid), 1 dense always, 2 sparse always.
int flb_debug_set_map_index(flb_handle* h, int mode) {
    FLB_CHECK_H(h);
    if (mode < 0 || mode > 2) return fail(h, FLB_ERR_INVALID, "flb_debug_set_map_index: mode 0, 1 or 2");
    h->map_index_mode = mode;
    return FLB_OK;
}

// Test aid: the uploaded scan's order -- src_index[i] = index (in the caller's array) of the point at sorted position i.
int flb_debug_scan_order(flb_handle* h, int* src_index, int capacity) {
    FLB_CHECK_H(h);
    if (!src_index || capacity < h->N) return fail(h, FLB_ERR_INVALID, "flb_debug_scan_order: bad arguments");
    if (h->N == 0) return FLB_OK;
    std::vector<float4> tmp((size_t)h->N);
    FLB_CUDA(h, cudaMemcpyAsync(tmp.data(), h->scan.p, (size_t)h->N * sizeof(float4), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < h->N; ++i) std::memcpy(&src_index[i], &tmp[(size_t)i].w, sizeof(int));
    return FLB_OK;
}

int flb_debug_block_stamps(flb_handle* h, unsigned long long* out, int max_blocks, int* nblocks) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    const int n = std::min(h->dbg_blocks, max_blocks);     // 16 words per block: 4 block stamps, 8 warp stamps
    if (n > 0) FLB_CUDA(h, cudaMemcpy(out, h->dbg.p, (size_t)n * 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    *nblocks = n;
    return FLB_OK;
}

int flb_trace_download(flb_handle* h, int which, double* us, int max_entries, int* n_entries) {
    FLB_CHECK_H(h);
    if (!us || !n_entries || (which != 0 && which != 1)) return fail(h, FLB_ERR_INVALID, "flb_trace_download: bad arguments");
    unsigned long long t[kTraceLen];
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    FLB_CUDA(h, cudaMemcpy(t, h->trace.p + which * kTraceLen, sizeof(t), cudaMemcpyDeviceToHost));
    int n = 0;
    for (int i = 1; i < kTraceLen && i - 1 < max_entries; ++i) {
        if (t[i] == 0 && i < 64) { if (max_entries < kTraceLen - 1) break; us[n++] = 0.0; continue; }
        us[n++] = t[i] ? (double)(t[i] - t[0]) * 1e-3 : 0.0;
    }
    *n_entries = n;
    return FLB_OK;
}

// ---------------------------------------------------------------------------------------
int flb_comm_unique_id(void* unique_id_128b) {
    if (!unique_id_128b) return FLB_ERR_INVALID;
    if (!g_nccl.load()) return fail(nullptr, FLB_ERR_COMM, "libnccl.so.2 not found");
    ncclUniqueId id;
    int r = g_nccl.GetUniqueId(&id);
    if (r != 0) return fail(nullptr, FLB_ERR_COMM, "ncclGetUniqueId failed (%d)", r);
    std::memcpy(unique_id_128b, &id, 128);
    return FLB_OK;
}

int flb_comm_init(flb_handle* h, const void* unique_id_128b, int rank, int world_size) {
    FLB_CHECK_H(h);
    if (!unique_id_128b || world_size < 1 || rank < 0 || rank >= world_size) return fail(h, FLB_ERR_INVALID, "flb_comm_init: bad arguments");
    if (!g_nccl.load()) return fail(h, FLB_ERR_COMM, "libnccl.so.2 not found");
    if (h->comm) { g_nccl.CommDestroy(h->comm); h->comm = nullptr; }
    ncclUniqueId id;
    std::memcpy(&id, unique_id_128b, 128);
    int r = g_nccl.CommInitRank(&h->comm, world_size, id, rank);
    if (r != 0) { h->comm = nullptr; return fail(h, FLB_ERR_COMM, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"); }
    h->rank = rank;
    h->world = world_size;
    return FLB_OK;
}

// ---- fused NVLink exchange -------------------------------------------------------------------
int flb_p2p_export(flb_handle* h, void* handle_64b) {
    FLB_CHECK_H(h);
    if (!handle_64b) return fail(h, FLB_ERR_INVALID, "flb_p2p_export: null handle buffer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    FLB_CUDA(h, h->mailbox.reserve(1));
    FLB_CUDA(h, h->p2p_seq.reserve(1));
    FLB_CUDA(h, cudaMemset(h->mailbox.p, 0, sizeof(P2PMailbox)));
    FLB_CUDA(h, cudaMemset(h->p2p_seq.p, 0, sizeof(unsigned long long)));
    cudaIpcMemHandle_t ih;
    FLB_CUDA(h, cudaIpcGetMemHandle(&ih, h->mailbox.p));
    std::memcpy(handle_64b, &ih, 64);
    return FLB_OK;
}

int flb_p2p_attach(flb_handle* h, int rank, int world_size, const void* handles) {
    FLB_CHECK_H(h);
    if (!handles || world_size < 1 || world_size > kP2PMaxWorld || rank < 0 || rank >= world_size)
        return fail(h, FLB_ERR_INVALID, "flb_p2p_attach: bad arguments (world <= %d)", kP2PMaxWorld);
    if (!h->mailbox.p) return fail(h, FLB_ERR_STATE, "flb_p2p_attach: call flb_p2p_export first");
    P2PArgs a{};
    a.world = world_size;
    a.rank = rank;
    a.seq = h->p2p_seq.p;
    for (int r = 0; r < world_size; ++r) {
        if (r == rank) { a.mail[r] = h->mailbox.p; continue; }
        cudaIpcMemHandle_t ih;
        std::memcpy(&ih, static_cast<const char*>(handles) + 64 * (size_t)r, 64);
        void* ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, ih, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail(h, FLB_ERR_COMM, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
        h->p2p_peer_ptr[r] = ptr;
        a.mail[r] = static_cast<P2PMailbox*>(ptr);
    }
    h->p2p = a;
    h->rank = rank;
    h->world = world_size;
    return FLB_OK;
}

int flb_p2p_detach(flb_handle* h) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    for (int r = 0; r < kP2PMaxWorld; ++r)
        if (h->p2p_peer_ptr[r]) { cudaIpcCloseMemHandle(h->p2p_peer_ptr[r]); h->p2p_peer_ptr[r] = nullptr; }
    h->p2p = P2PArgs{};
    return FLB_OK;
}

int flb_comm_destroy(flb_handle* h) {
    FLB_CHECK_H(h);
    if (h->comm) { g_nccl.CommDestroy(h->comm); h->comm = nullptr; }
    h->world = 1;
    h->rank = 0;
    return FLB_OK;
}

}  // extern "C"

// =======================================================================================
// Batched frames (SURVEY.md section 7 H2(iv)): B independent frames per launch
// =======================================================================================
extern "C" {

int flb_batch_begin(flb_handle* h, int B, int max_points_per_frame) {
    FLB_CHECK_H(h);
    if (B < 1 || B > 4096 || max_points_per_frame < 1) return fail(h, FLB_ERR_INVALID, "flb_batch_begin: bad arguments");
    if (h->M <= 0) return fail(h, FLB_ERR_STATE, "flb_batch_begin: upload the map first");
    auto& b = h->batch;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    b.B = B;
    b.n_cap = (max_points_per_frame + kLioBlock - 1) / kLioBlock * kLioBlock;
    b.N.assign(B, 0);
    const size_t tot = (size_t)B * b.n_cap;
    FLB_CUDA(h, b.scan.reserve(tot));
    FLB_CUDA(h, b.plane.reserve(tot));
    FLB_CUDA(h, b.sel.reserve(tot));
    FLB_CUDA(h, b.plane_ok.reserve(tot));
    FLB_CUDA(h, b.states.reserve((size_t)B * 5));
    FLB_CUDA(h, b.lio_ctrl.reserve(B));
    FLB_CUDA(h, b.vio_ctrl.reserve(B));
    FLB_CUDA(h, b.prior.reserve(B));
    FLB_CUDA(h, b.G_last.reserve((size_t)B * 108));
    FLB_CUDA(h, b.lio_args.reserve(B));
    FLB_CUDA(h, b.lio_solve.reserve(B));
    FLB_CUDA(h, b.vio_args.reserve(B));
    FLB_CUDA(h, b.vio_solve.reserve(B));
    FLB_CUDA(h, b.lio_ctrl_ptrs.reserve(B));
    FLB_CUDA(h, b.vio_ctrl_ptrs.reserve(B));
    std::vector<LioCtrl*> lp(B);
    std::vector<VioCtrl*> vp(B);
    for (int i = 0; i < B; ++i) { lp[i] = b.lio_ctrl.p + i; vp[i] = b.vio_ctrl.p + i; }
    FLB_CUDA(h, cudaMemcpy(b.lio_ctrl_ptrs.p, lp.data(), B * sizeof(LioCtrl*), cudaMemcpyHostToDevice));
    FLB_CUDA(h, cudaMemcpy(b.vio_ctrl_ptrs.p, vp.data(), B * sizeof(VioCtrl*), cudaMemcpyHostToDevice));
    FLB_CUDA(h, cudaMemset(b.lio_ctrl.p, 0, B * sizeof(LioCtrl)));
    FLB_CUDA(h, cudaMemset(b.vio_ctrl.p, 0, B * sizeof(VioCtrl)));
    return FLB_OK;
}

int flb_batch_set_frame(flb_handle* h, int frame, const float* body_xyz, int N, int stride, const flb_state18* x, const flb_state18* x_prop) {
    FLB_CHECK_H(h);
    auto& b = h->batch;
    if (frame < 0 || frame >= b.B || !x || !x_prop || N < 1 || N > b.n_cap) return fail(h, FLB_ERR_INVALID, "flb_batch_set_frame: bad arguments");
    int rc = flb_scan_upload(h, body_xyz, N, stride);      // validates, Morton-sorts into h->scan
    if (rc) return rc;
    const size_t off = (size_t)frame * b.n_cap;
    FLB_CUDA(h, cudaMemcpyAsync(b.scan.p + off, h->scan.p, (size_t)N * sizeof(float4), cudaMemcpyDeviceToDevice, h->stream));
    FLB_CUDA(h, cudaMemsetAsync(b.sel.p + off, 1, N, h->stream));
    FLB_CUDA(h, cudaMemsetAsync(b.plane_ok.p + off, 0, N, h->stream));
    rc = flb_state_upload(h, x, x_prop);                   // through the handle's staging, then into the frame's slots
    if (rc) return rc;
    State18* st = b.states.p + (size_t)frame * 5;
    FLB_CUDA(h, cudaMemcpyAsync(st, &h->states.p[0], 2 * sizeof(State18), cudaMemcpyDeviceToDevice, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(st + 3, &h->states.p[0], 2 * sizeof(State18), cudaMemcpyDeviceToDevice, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    b.N[frame] = N;
    b.n_max = *std::max_element(b.N.begin(), b.N.end());
    return FLB_OK;
}

/* restore every frame's x / x_prop to what flb_batch_set_frame gave it (benchmark loop) */
int flb_batch_state_reset_enqueue(flb_handle* h) {
    FLB_CHECK_H(h);
    auto& b = h->batch;
    if (b.B < 1) return fail(h, FLB_ERR_STATE, "flb_batch_state_reset_enqueue: no batch");
    FLB_CUDA(h, cudaMemcpy2DAsync(b.states.p, 5 * sizeof(State18), b.states.p + 3, 5 * sizeof(State18), 2 * sizeof(State18), b.B,
                                  cudaMemcpyDeviceToDevice, h->stream));
    return FLB_OK;
}

int flb_batch_update_enqueue(flb_handle* h, const flb_lio_params* lprm, const flb_vio_params* vprm) {
    FLB_CHECK_H(h);
    auto& b = h->batch;
    if (b.B < 1 || b.n_max < 1) return fail(h, FLB_ERR_STATE, "flb_batch_update_enqueue: flb_batch_begin / flb_batch_set_frame first");
    if (!lprm) return fail(h, FLB_ERR_INVALID, "flb_batch_update_enqueue: null LIO params");
    if (h->comm || h->p2p.world > 1) return fail(h, FLB_ERR_STATE, "batched frames: single GPU");
    for (int i = 0; i < b.B; ++i)
        if (b.N[i] < 1) return fail(h, FLB_ERR_STATE, "flb_batch_update_enqueue: frame %d not set", i);
    const int B = b.B;
    const bool vio = vprm != nullptr && h->Pn > 0 && vprm->max_iteration > 0;
    if (vio) {
        { int rc = vio_image_check(h, "flb_batch_update_enqueue"); if (rc) return rc; }
        if (h->pn_on_device) { int rc = resolve_pn(h); if (rc) return rc; }
    }
    const int nb_lio = (b.n_max + kLioBlock - 1) / kLioBlock;
    const int nb_vio = (h->Pn + (kVioBlock / 32) - 1) / (kVioBlock / 32);
    b.partials_per = (size_t)std::max(nb_lio * lio_packed(6), nb_vio * kVioPacked);
    FLB_CUDA(h, b.partials.reserve((size_t)B * b.partials_per));
    const int estride = std::max(h->Pn, 1);
    FLB_CUDA(h, b.errors.reserve((size_t)B * 2 * estride));
    // frame i's slice of the batch buffers
    auto frame = [&](int i) -> FrameBufs {
        const size_t off = (size_t)i * b.n_cap;
        return {b.scan.p + off, b.N[i], b.states.p + (size_t)i * 5, b.lio_ctrl.p + i, b.vio_ctrl.p + i, b.prior.p + i, b.sel.p + off,
                b.plane.p + off, b.plane_ok.p + off, b.partials.p + (size_t)i * b.partials_per, b.errors.p + (size_t)i * 2 * estride,
                estride, b.G_last.p + (size_t)i * 108};
    };
    LioParamsDev ld;
    to_dev_params(lprm, ld);
    std::vector<LioArgs> la(B);
    std::vector<LioSolveArgs> ls(B);
    for (int i = 0; i < B; ++i) {
        la[i] = make_lio_args(h, ld, frame(i));
        ls[i] = make_lio_solve_args(h, ld, frame(i));
    }
    // argument tables: pageable -> device through the stream (small; ordered before the launches that read them)
    FLB_CUDA(h, cudaMemcpyAsync(b.lio_args.p, la.data(), B * sizeof(LioArgs), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(b.lio_solve.p, ls.data(), B * sizeof(LioSolveArgs), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));          // la / ls are stack-owned
    {
        LaunchScope lsx(h, FAM_SOLVE);
        k_lio_begin_batched<<<(B + 127) / 128, 128, 0, h->stream>>>(b.lio_ctrl_ptrs.p, B);
        FLB_CUDA(h, cudaGetLastError());
    }
    const int T = lprm->max_iteration;
    for (int it = -1; it < T; ++it) {
        {
            // family tag: with early stop disabled the rematch passes are the first and the last (Appendix A)
            LaunchScope lsx(h, (it == -1 || it == T - 1) ? FAM_LIO_KNN : FAM_LIO_PLAIN);
            if (h->sparse) k_lio_pass_batched<6, kLioBlock, true><<<dim3(nb_lio, B), kLioBlock, 0, h->stream>>>(b.lio_args.p);
            else k_lio_pass_batched<6, kLioBlock, false><<<dim3(nb_lio, B), kLioBlock, 0, h->stream>>>(b.lio_args.p);
            FLB_CUDA(h, cudaGetLastError());
        }
        LaunchScope lsx(h, FAM_SOLVE);
        k_lio_finalize_batched<<<B, kLeaderBlock, 0, h->stream>>>(b.lio_solve.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    if (!vio) return FLB_OK;
    // state_propagat := the LIO posterior (zero-motion propagation between the two updates), per frame
    FLB_CUDA(h, cudaMemcpy2DAsync(b.states.p + 1, 5 * sizeof(State18), b.states.p, 5 * sizeof(State18), sizeof(State18), B,
                                  cudaMemcpyDeviceToDevice, h->stream));
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    VioParamsDev vd;
    to_dev_params(vprm, vd);
    std::vector<VioArgs> va(B);
    std::vector<VioSolveArgs> vs(B);
    for (int i = 0; i < B; ++i) {
        va[i] = make_vio_args(h, vd, frame(i));
        vs[i] = make_vio_solve_args(h, vd, frame(i));
    }
    FLB_CUDA(h, cudaMemcpyAsync(b.vio_args.p, va.data(), B * sizeof(VioArgs), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(b.vio_solve.p, vs.data(), B * sizeof(VioSolveArgs), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    {
        LaunchScope lsx(h, FAM_SOLVE);
        k_vio_begin_batched<<<(B + 127) / 128, 128, 0, h->stream>>>(b.vio_ctrl_ptrs.p, B, h->Pn);
        FLB_CUDA(h, cudaGetLastError());
    }
    const int total = 3 * vprm->max_iteration;
    for (int it = 0; it < total; ++it) {
        {
            LaunchScope lsx(h, FAM_VIO);
            k_vio_pass_batched<kVioBlock><<<dim3(nb_vio, B), kVioBlock, 0, h->stream>>>(b.vio_args.p);
            FLB_CUDA(h, cudaGetLastError());
        }
        LaunchScope lsx(h, FAM_SOLVE);
        k_vio_finalize_batched<<<B, kLeaderBlock, 0, h->stream>>>(b.vio_solve.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    return FLB_OK;
}

int flb_batch_state_download(flb_handle* h, int frame, flb_state18* x, flb_lio_report* lio, flb_vio_report* vio) {
    FLB_CHECK_H(h);
    auto& b = h->batch;
    if (frame < 0 || frame >= b.B) return fail(h, FLB_ERR_INVALID, "flb_batch_state_download: bad frame");
    State18 xs;
    LioCtrl lc;
    VioCtrl vc;
    FLB_CUDA(h, cudaMemcpyAsync(&xs, b.states.p + (size_t)frame * 5, sizeof(State18), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(&lc, b.lio_ctrl.p + frame, sizeof(LioCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaMemcpyAsync(&vc, b.vio_ctrl.p + frame, sizeof(VioCtrl), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (x) std::memcpy(x, &xs, sizeof(State18));
    if (lio) fill_lio_report(lc, lio);
    if (vio) fill_vio_report(vc, vio);
    return FLB_OK;
}

}  // extern "C"

// =======================================================================================
// Device-resident visual map (SURVEY.md section 8 rows f2 / f4)
// =======================================================================================
namespace {

int vm_check(flb_handle* h, const char* who) {
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "%s: flb_vmap_reset first", who);
    return vio_image_check(h, who);
}

// Upload (or derive from the device state) T_f_w of the current frame into vm.pose.
int vm_set_pose(flb_handle* h, const double* Rcw, const double* Pcw) {
    if (Rcw && Pcw) return upload_pose(h, h->vm.pose.p, Rcw, Pcw);
    if (!h->state_valid) return fail(h, FLB_ERR_STATE, "visual map: no pose given and no device state");
    { int rcf = flush_state_ops(h); if (rcf) return rcf; }
    LaunchScope ls(h, FAM_OTHER);
    k_vm_pose_from_state<<<1, 32, 0, h->stream>>>(&h->states.p[0], h->vm.rci.p, h->vm.pose.p);
    FLB_CUDA(h, cudaGetLastError());
    return FLB_OK;
}

// points of this call -> vm.pg (packed xyz)
int vm_upload_points(flb_handle* h, const float* xyz, int n, int stride) {
    const size_t n1 = (size_t)std::max(n, 1);
    FLB_CUDA(h, h->vm.pg.reserve(n1 * 3));
    if (n == 0) return FLB_OK;
    void* stv = nullptr;
    FLB_CUDA(h, h->vm.st_pg.acquire(n1 * 3 * sizeof(float), &stv));
    float* st = static_cast<float*>(stv);
    pack_points(st, xyz, n, stride);
    float lo[3], hi[3];
    bool bad = fold_points<true>(st, n, lo, hi);
    for (int k = 0; k < 3; ++k) bad = bad || lo[k] < -kVmapCoordLimit || hi[k] > kVmapCoordLimit;
    if (bad)
        return fail(h, FLB_ERR_INVALID, "visual map: coordinate %d non-finite or beyond 2^20 voxels", first_bad_point(st, n, kVmapCoordLimit));
    FLB_CUDA(h, cudaMemcpyAsync(h->vm.pg.p, st, (size_t)n * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->vm.st_pg.mark(h->stream));
    return FLB_OK;
}

template <typename T>
int vm_grow_buf(flb_handle* h, DevBuf<T>& b, size_t used_ub, size_t need) {
    if (need <= b.cap) return FLB_OK;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    DevBuf<T> nb;
    FLB_CUDA(h, nb.reserve(std::max(need, b.cap * 2)));
    if (b.p && used_ub) FLB_CUDA(h, cudaMemcpy(nb.p, b.p, std::min(used_ub, b.cap) * sizeof(T), cudaMemcpyDeviceToDevice));
    b.release();
    b = nb;
    return FLB_OK;
}

// flb_vmap_reclaim's buffers shadow the feature array and the pool.  The first reclaim allocates them; afterwards
// vm_ensure_capacity grows them together with those arrays (it has synchronised by then), so a reclaim neither frees
// memory nor waits for the device.  Nothing in them outlives a reclaim except the free-slot stack, and the pool only
// grows when every slot is in use, i.e. with that stack empty: none of them needs its contents copied.
int vm_reclaim_reserve(flb_handle* h) {
    auto& vm = h->vm;
    const size_t slots = (size_t)std::max(vm.pool_slots, 1);
    FLB_CUDA(h, vm.fts_alt.reserve(vm.fts.cap));
    FLB_CUDA(h, vm.rc_rank.reserve(vm.fts.cap + 1));
    FLB_CUDA(h, vm.free_slots.reserve(slots));
    FLB_CUDA(h, vm.rc_slot.reserve(3 * slots));
    size_t bytes = 0;                        // the scan's scratch only grows with its length: size it for the largest one
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, bytes, vm.rc_rank.p, vm.rc_rank.p, (int)(vm.fts.cap + 1), h->stream));
    FLB_CUDA(h, vm.rc_cub.reserve(std::max<size_t>(bytes, 1)));
    vm.rc_cub_bytes = std::max(vm.rc_cub_bytes, bytes);
    return FLB_OK;
}

// Make room for `add_p` more points, `add_f` more features and one more keyframe image.  The host only keeps upper
// bounds of the device counters; when a bound hits the capacity it is refreshed from the device before anything grows.
// The image bound counts slots in use: after a reclaim, slots on the free-slot stack are room, and the pool grows only
// when none is left (then the slots in use are exactly the pool's tail).
int vm_ensure_capacity(flb_handle* h, int add_p, int add_f) {
    auto& vm = h->vm;
    const size_t img_bytes = (size_t)h->img_w * h->img_h;
    const size_t fts_cap = vm.fts.cap;
    const int pool_slots = vm.pool_slots;
    if ((size_t)(vm.pts_ub + add_p) > vm.pts.cap || (size_t)(vm.fts_ub + add_f) > vm.fts.cap || vm.img_ub + 1 > vm.pool_slots) {
        int c[VM_COUNTERS];
        FLB_CUDA(h, cudaMemcpyAsync(c, vm.counters.p, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        vm.pts_ub = c[VM_N_POINTS];
        vm.fts_ub = c[VM_N_FEATS];
        vm.img_ub = c[VM_N_IMAGES] - c[VM_N_FREE];
    }
    { int rc = vm_grow_buf(h, vm.pts, (size_t)vm.pts_ub, (size_t)(vm.pts_ub + add_p)); if (rc) return rc; }
    { int rc = vm_grow_buf(h, vm.fts, (size_t)vm.fts_ub, (size_t)(vm.fts_ub + add_f)); if (rc) return rc; }
    if (vm.img_ub + 1 > vm.pool_slots) {
        const int slots = std::max(vm.pool_slots * 2, 16);
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
        DevBuf<unsigned char> nb;
        FLB_CUDA(h, nb.reserve((size_t)slots * img_bytes));
        if (vm.pool.p && vm.img_ub) FLB_CUDA(h, cudaMemcpy(nb.p, vm.pool.p, (size_t)vm.img_ub * img_bytes, cudaMemcpyDeviceToDevice));
        vm.pool.release();
        vm.pool = nb;
        vm.pool_slots = slots;
    }
    if (vm.fts_alt.p && (vm.fts.cap != fts_cap || vm.pool_slots != pool_slots)) return vm_reclaim_reserve(h);
    return FLB_OK;
}

}  // namespace

extern "C" {

int flb_vmap_reset(flb_handle* h, const flb_vmap_params* p) {
    FLB_CHECK_H(h);
    if (!p || p->grid_size < 1) return fail(h, FLB_ERR_INVALID, "flb_vmap_reset: bad parameters");
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_vmap_reset: flb_camera_set first");
    auto& vm = h->vm;
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    VmParams q{};
    q.grid_size = p->grid_size;
    q.grid_n_width = h->cam.width / p->grid_size;                  // :55-57
    q.grid_n_height = h->cam.height / p->grid_size;
    q.length = q.grid_n_width * q.grid_n_height;
    q.halfpatch = 4;
    q.ncc_en = p->ncc_en;
    q.outlier_threshold = p->outlier_threshold;
    q.ncc_thre = p->ncc_thre;
    if (q.length < 1) return fail(h, FLB_ERR_INVALID, "flb_vmap_reset: grid_size larger than the image");
    vm.prm = q;
    {   // Rci / Pci (LidarSelector::init :44-45, set_extrinsic :35-39)
        double Rli[9], Pli[3], t[3];
        m3_T(p->R_LI, Rli);
        m3_vec(Rli, p->t_LI, t);
        for (int i = 0; i < 3; ++i) Pli[i] = -t[i];
        m3_mul(p->Rcl, Rli, vm.Rci_Pci);
        m3_vec(p->Rcl, Pli, t);
        for (int i = 0; i < 3; ++i) vm.Rci_Pci[9 + i] = t[i] + p->Pcl[i];
    }
    const size_t L = (size_t)q.length, npix = (size_t)h->cam.width * h->cam.height;
    FLB_CUDA(h, vm.counters.reserve(VM_COUNTERS));
    FLB_CUDA(h, vm.pose.reserve(12));
    FLB_CUDA(h, vm.rci.reserve(12));
    FLB_CUDA(h, vm.depth.reserve(npix));
    FLB_CUDA(h, vm.cell_best.reserve(L));
    FLB_CUDA(h, vm.cand_key.reserve(L));
    FLB_CUDA(h, vm.cell_type.reserve(L));
    FLB_CUDA(h, vm.map_value.reserve(L));
    FLB_CUDA(h, vm.cell_err.reserve(L));
    FLB_CUDA(h, vm.cell_patch.reserve(L * 192));
    FLB_CUDA(h, vm.sel_error.reserve(L));
    FLB_CUDA(h, vm.cell_flag.reserve(L));
    FLB_CUDA(h, vm.cell_rank.reserve(L));
    FLB_CUDA(h, vm.cell_level.reserve(L));
    FLB_CUDA(h, vm.cell_point.reserve(L));
    FLB_CUDA(h, vm.sel_index.reserve(L));
    FLB_CUDA(h, vm.sel_point.reserve(L));
    FLB_CUDA(h, vm.winner.reserve(L));
    FLB_CUDA(h, vm.scan_tmp.reserve(2 * L));
    FLB_CUDA(h, vm.pts.reserve(std::max<size_t>(4 * L, 1024)));
    FLB_CUDA(h, vm.fts.reserve(std::max<size_t>(8 * L, 2048)));
    // the VIO kernel's inputs are the selection's outputs: one patch per grid cell at most
    FLB_CUDA(h, h->patch_pos.reserve(L * 3));
    FLB_CUDA(h, h->patch_ref.reserve(L * 192));
    FLB_CUDA(h, h->patch_level.reserve(L));
    int c[VM_COUNTERS] = {0};
    c[VM_IMG_FRAME] = -1;
    c[VM_IMG_SLOT] = -1;
    FLB_CUDA(h, cudaMemcpy(vm.counters.p, c, sizeof(c), cudaMemcpyHostToDevice));
    FLB_CUDA(h, cudaMemcpy(vm.rci.p, vm.Rci_Pci, sizeof(vm.Rci_Pci), cudaMemcpyHostToDevice));
    FLB_CUDA(h, cudaMemset(vm.map_value.p, 0, L * sizeof(float)));   // init(), :66
    vm.pts_ub = vm.fts_ub = vm.img_ub = 0;
    vm.on = true;
    return FLB_OK;
}

}  // extern "C"

namespace {

// addFromSparseMap once the pose is set: pg_down = n device points, or -- n_dev non-null -- *n_dev (on the device) of at
// most n.  flb_vmap_select and flb_vmap_select_cloud differ only in how pg_down gets to the device.
int vm_select_dev(flb_handle* h, const float* pg_down, int n, const int* n_dev, int* n_selected) {
    auto& vm = h->vm;
    const int L = vm.prm.length, border = (vm.prm.halfpatch + 1) * 8;
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }                 // the current image has landed
    size_t nkeys = 1024;
    while (nkeys < 2 * (size_t)std::max(n, 1)) nkeys <<= 1;
    FLB_CUDA(h, vm.keyset.reserve(nkeys));
    vm.key_mask = (unsigned)(nkeys - 1);
    const size_t npix = (size_t)h->cam.width * h->cam.height;
    // per-patch error buffers of the VIO update that follows: capacity = one patch per grid cell
    FLB_CUDA(h, h->errors.reserve(2 * (size_t)L));
    h->err_stride = std::max(h->err_stride, L);
    FLB_CUDA(h, h->errors.reserve(2 * (size_t)h->err_stride));
    FLB_CUDA(h, h->partials.reserve(std::max<size_t>((size_t)(L / 8 + 2) * kVioPacked, h->partials.cap)));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_clear<<<h->num_sms * 2, 256, 0, h->stream>>>(vm.depth.p, npix, vm.keyset.p, nkeys, vm.cell_best.p, vm.cell_type.p, vm.map_value.p,
                                                          vm.cell_flag.p, L, vm.counters.p);
        if (n > 0)
            k_vm_scan<<<(n + 255) / 256, 256, 0, h->stream>>>(h->cam, vm.pose.p, pg_down, n, n_dev, border, vm.keyset.p, vm.key_mask,
                                                              vm.depth.p, vm.counters.p);
        const int np = std::max(vm.pts_ub, 1);
        k_vm_candidates<<<(np + 255) / 256, 256, 0, h->stream>>>(h->cam, vm.prm, vm.pose.p, vm.pts.p, vm.counters.p, vm.keyset.p, vm.key_mask,
                                                                 border, vm.cell_best.p, vm.cell_type.p,
                                                                 reinterpret_cast<int*>(vm.map_value.p));
        k_vm_build<<<(L + kVmBuildWarps - 1) / kVmBuildWarps, kVmBuildWarps * 32, 0, h->stream>>>(
            h->cam, vm.prm, vm.pose.p, vm.pts.p, vm.fts.p, vm.pool.p, h->img.p, vm.depth.p, vm.cell_best.p, vm.cell_type.p, vm.counters.p,
            vm.cell_flag.p, vm.cell_level.p, vm.cell_point.p, vm.cell_err.p, vm.cell_patch.p);
        k_vm_rank<<<1, 1024, 0, h->stream>>>(vm.cell_flag.p, L, vm.cell_rank.p, vm.counters.p);
        k_vm_scatter<<<(L + 7) / 8, 256, 0, h->stream>>>(L, vm.cell_flag.p, vm.cell_rank.p, vm.cell_level.p, vm.cell_point.p, vm.cell_err.p,
                                                         vm.cell_patch.p, vm.pts.p, h->patch_pos.p, h->patch_ref.p, h->patch_level.p,
                                                         vm.sel_index.p, vm.sel_point.p, vm.sel_error.p);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 5;
    }
    h->pn_on_device = true;
    h->patches_set = true;
    h->err_from_sel = true;
    h->Pn = L;
    h->last_vio_valid = false;
    if (n_selected) {
        int rc = resolve_pn(h);
        if (rc) return rc;
        *n_selected = h->Pn;
    }
    return FLB_OK;
}

// The world cloud's consumers (flb_*_cloud) need one: FLB_ERR_STATE until a flb_world_cloud succeeds.
int wc_check(flb_handle* h, const char* who) {
    if (h->wc_n < 0) return fail(h, FLB_ERR_STATE, "%s: no world cloud (flb_world_cloud first, or it failed)", who);
    return FLB_OK;
}

}  // namespace

extern "C" {

int flb_vmap_select(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* pg_down, int n, int stride, int* n_selected) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_select"); if (rc) return rc; }
    if (n < 0 || (n > 0 && !pg_down) || stride < 3) return fail(h, FLB_ERR_INVALID, "flb_vmap_select: bad arguments");
    { int rc = vm_set_pose(h, Rcw, Pcw); if (rc) return rc; }
    { int rc = vm_upload_points(h, pg_down, n, stride); if (rc) return rc; }
    return vm_select_dev(h, h->vm.pg.p, n, nullptr, n_selected);
}

// LidarSelector::detect's addFromSparseMap(img, pg_down) with pg_down = downSizeFilter(pcl_wait_pub) (src/lidar_selection.cpp:
// 351-353) on the device: flb_voxel_grid's chain on the world cloud into buffers of this call's own (the scan slot is not
// touched), then the selection with the leaf count left on the device (k_vm_scan runs over the cloud's size as its bound).
int flb_vmap_select_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], float leaf, int* n_selected) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_select_cloud"); if (rc) return rc; }
    { int rc = wc_check(h, "flb_vmap_select_cloud"); if (rc) return rc; }
    if (!(leaf > 0)) return fail(h, FLB_ERR_INVALID, "flb_vmap_select_cloud: bad arguments (leaf > 0)");
    const int n = h->wc_n;
    if (n > 0) {
        // PCL's index-overflow test from the bounds flb_world_cloud read (k_vg_keys' float expressions on k_bbox's
        // box, which equals them): decided here, so the leaf count never has to come back
        const float inv_leaf = 1.0f / leaf;
        double cells = 1.0;
        for (int k = 0; k < 3; ++k) {
            const float d = (h->wc_hi[k] - h->wc_lo[k]) * inv_leaf;
            cells *= d < 9.0e18f ? (double)((long long)d + 1) : 9.2e18;
        }
        if (cells > 2147483647.0)
            return fail(h, FLB_ERR_INVALID, "flb_vmap_select_cloud: leaf size too small for the cloud's extent (index overflow, as PCL warns)");
    }
    { int rc = vm_set_pose(h, Rcw, Pcw); if (rc) return rc; }
    if (n == 0) return vm_select_dev(h, h->wc_down.p, 0, nullptr, n_selected);
    FLB_CUDA(h, h->wc_down.reserve((size_t)n * 3));
    FLB_CUDA(h, h->wc_keys.reserve(n));
    FLB_CUDA(h, h->wc_keys_sorted.reserve(n));
    FLB_CUDA(h, h->wc_vals.reserve(n));
    FLB_CUDA(h, h->wc_vals_sorted.reserve(n));
    FLB_CUDA(h, h->wc_heads.reserve((size_t)2 * n));
    FLB_CUDA(h, h->wc_box.reserve(8));
    const VgScratch vs{h->wc_keys.p, h->wc_keys_sorted.p, h->wc_vals.p, h->wc_vals_sorted.p, h->wc_heads.p, h->wc_heads.p + n, h->wc_box.p};
    { int rcv = voxel_grid_dev(h, h->wc_xyz.p, n, leaf, vs, h->wc_down.p); if (rcv) return rcv; }
    return vm_select_dev(h, h->wc_down.p, n, h->wc_box.p + 7, n_selected);
}

int flb_vmap_selected(flb_handle* h, int capacity, int* n_out, int* index, int* point, int* search_level, float* error, double* pos,
                      float* patch) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_selected"); if (rc) return rc; }
    auto& vm = h->vm;
    int n = 0;
    FLB_CUDA(h, cudaMemcpyAsync(&n, vm.counters.p + VM_N_SEL, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (n_out) *n_out = n;
    const size_t m = (size_t)std::min(std::max(capacity, 0), n);
    if (m == 0) return FLB_OK;
    cudaStream_t s = h->stream;
    if (index) FLB_CUDA(h, cudaMemcpyAsync(index, vm.sel_index.p, m * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (point) FLB_CUDA(h, cudaMemcpyAsync(point, vm.sel_point.p, m * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (search_level) FLB_CUDA(h, cudaMemcpyAsync(search_level, h->patch_level.p, m * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (error) FLB_CUDA(h, cudaMemcpyAsync(error, vm.sel_error.p, m * sizeof(float), cudaMemcpyDeviceToHost, s));
    if (pos) FLB_CUDA(h, cudaMemcpyAsync(pos, h->patch_pos.p, m * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    if (patch) FLB_CUDA(h, cudaMemcpyAsync(patch, h->patch_ref.p, m * 192 * sizeof(float), cudaMemcpyDeviceToHost, s));
    FLB_CUDA(h, cudaStreamSynchronize(s));
    return FLB_OK;
}

}  // extern "C"

namespace {

// addSparseMap once the capacity and the pose are set, over n device points pg (flb_vmap_grow / flb_vmap_grow_cloud).
int vm_grow_dev(flb_handle* h, const float* pg, int n, int frame_id) {
    auto& vm = h->vm;
    const int L = vm.prm.length, border = (vm.prm.halfpatch + 1) * 8;
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    const size_t img_bytes = (size_t)h->img_w * h->img_h;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_store_image<<<h->num_sms, 256, 0, h->stream>>>(h->img.p, img_bytes, vm.pool.p, vm.counters.p, vm.free_slots.p, frame_id);
        k_vmap_seed<<<(L + 255) / 256, 256, 0, h->stream>>>(vm.map_value.p, L, vm.cand_key.p);
        if (n > 0)
            k_vmap_candidates<<<(n + 127) / 128, 128, 0, h->stream>>>(h->cam, vm.pose.p, h->img.p, pg, n, vm.prm.grid_size, vm.prm.grid_n_height,
                                                                      border, vm.cand_key.p);
        k_vmap_resolve<<<(L + 255) / 256, 256, 0, h->stream>>>(vm.cand_key.p, L, vm.map_value.p, vm.winner.p);
        k_vm_materialise<<<1, 1024, 0, h->stream>>>(h->cam, L, vm.pose.p, pg, vm.winner.p, vm.map_value.p, vm.scan_tmp.p, vm.pts.p, vm.fts.p,
                                                    vm.counters.p, vm.free_slots.p, frame_id, (int)vm.pts.cap, (int)vm.fts.cap);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 4;
    }
    vm.pts_ub += L;
    vm.fts_ub += L;
    vm.img_ub += 1;
    return FLB_OK;
}

}  // namespace

extern "C" {

int flb_vmap_grow(flb_handle* h, const double Rcw[9], const double Pcw[3], const float* pg, int n, int stride, int frame_id) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_grow"); if (rc) return rc; }
    if (n < 0 || (n > 0 && !pg) || stride < 3 || frame_id < 0) return fail(h, FLB_ERR_INVALID, "flb_vmap_grow: bad arguments");
    const int L = h->vm.prm.length;
    { int rc = vm_ensure_capacity(h, L, L); if (rc) return rc; }
    { int rc = vm_set_pose(h, Rcw, Pcw); if (rc) return rc; }
    { int rc = vm_upload_points(h, pg, n, stride); if (rc) return rc; }
    return vm_grow_dev(h, h->vm.pg.p, n, frame_id);
}

// addSparseMap(img, pcl_wait_pub) (src/lidar_selection.cpp:142-202) over the world cloud on the device.
int flb_vmap_grow_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], int frame_id) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_grow_cloud"); if (rc) return rc; }
    { int rc = wc_check(h, "flb_vmap_grow_cloud"); if (rc) return rc; }
    if (frame_id < 0) return fail(h, FLB_ERR_INVALID, "flb_vmap_grow_cloud: bad arguments");
    const int L = h->vm.prm.length;
    { int rc = vm_ensure_capacity(h, L, L); if (rc) return rc; }
    { int rc = vm_set_pose(h, Rcw, Pcw); if (rc) return rc; }
    return vm_grow_dev(h, h->wc_xyz.p, h->wc_n, frame_id);
}

int flb_vmap_add_observations(flb_handle* h, const double Rcw[9], const double Pcw[3], int frame_id) {
    FLB_CHECK_H(h);
    { int rc = vm_check(h, "flb_vmap_add_observations"); if (rc) return rc; }
    if (frame_id < 0) return fail(h, FLB_ERR_INVALID, "flb_vmap_add_observations: bad arguments");
    auto& vm = h->vm;
    const int L = vm.prm.length;
    { int rc = vm_ensure_capacity(h, 0, L); if (rc) return rc; }
    { int rc = vm_set_pose(h, Rcw, Pcw); if (rc) return rc; }
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }
    const size_t img_bytes = (size_t)h->img_w * h->img_h;
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_store_image<<<h->num_sms, 256, 0, h->stream>>>(h->img.p, img_bytes, vm.pool.p, vm.counters.p, vm.free_slots.p, frame_id);
        k_vm_observe<<<1, 1024, 0, h->stream>>>(h->cam, vm.pose.p, h->img.p, vm.sel_point.p, h->patch_level.p, vm.scan_tmp.p, L, vm.pts.p,
                                                vm.fts.p, vm.counters.p, vm.free_slots.p, frame_id, (int)vm.fts.cap);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 1;
    }
    vm.fts_ub += L;
    vm.img_ub += 1;
    return FLB_OK;
}

}  // extern "C"

namespace {

int colorize_pose(flb_handle* h, const char* who, const double* Rcw, const double* Pcw) {
    auto& vm = h->vm;
    FLB_CUDA(h, vm.pose.reserve(12));
    FLB_CUDA(h, vm.rci.reserve(12));
    if (!(Rcw && Pcw) && !vm.on) return fail(h, FLB_ERR_STATE, "%s: no pose given and no flb_vmap_reset (extrinsics)", who);
    return vm_set_pose(h, Rcw, Pcw);
}

// The colour frame the colouring reads, into *d_img: the caller's bgr, packed and uploaded on `stream` into dst
// (W x H x 3 bytes); bgr == NULL: the current image set's colour frame (flb_image_upload_bgr), read in place once its
// upload has landed.
int colorize_image(flb_handle* h, const uint8_t* bgr, int stride_bytes, unsigned char* dst, const unsigned char** d_img) {
    if (!bgr) {
        *d_img = h->img_bgr.p;
        return vio_inputs_acquire(h);
    }
    const int W = h->cam.width, H = h->cam.height;
    const size_t img_bytes = (size_t)W * H * 3;
    void* stv = nullptr;
    FLB_CUDA(h, h->st_img.acquire(img_bytes, &stv));
    unsigned char* st = static_cast<unsigned char*>(stv);
    for (int r = 0; r < H; ++r) std::memcpy(st + (size_t)r * W * 3, bgr + (size_t)r * stride_bytes, (size_t)W * 3);
    FLB_CUDA(h, cudaMemcpyAsync(dst, st, img_bytes, cudaMemcpyHostToDevice, h->stream));
    FLB_CUDA(h, h->st_img.mark(h->stream));
    *d_img = dst;
    return FLB_OK;
}

// The per-point kernel and the download of rgb / valid for n >= 1 device points xyz, the colour image (colorize_image)
// uploaded ahead of rgb / valid.
int colorize_dev(flb_handle* h, const uint8_t* bgr, int stride_bytes, const float* xyz, int n, uint8_t* rgb, uint8_t* valid) {
    auto& vm = h->vm;
    const int W = h->cam.width, H = h->cam.height;
    const size_t img_bytes = bgr ? (size_t)W * H * 3 : 0;
    FLB_CUDA(h, h->x_rowmask.reserve(img_bytes + (size_t)n * 4));     // [colour image |] rgb | valid
    const unsigned char* d_img = nullptr;
    unsigned char* d_rgb = h->x_rowmask.p + img_bytes;
    unsigned char* d_val = d_rgb + (size_t)n * 3;
    { int rci = colorize_image(h, bgr, stride_bytes, h->x_rowmask.p, &d_img); if (rci) return rci; }
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_colorize<<<(n + 255) / 256, 256, 0, h->stream>>>(h->cam, vm.pose.p, d_img, xyz, n, d_rgb, d_val);
        FLB_CUDA(h, cudaGetLastError());
    }
    FLB_CUDA(h, h->pin_out.reserve((size_t)n * 4));
    FLB_CUDA(h, cudaMemcpyAsync(h->pin_out.p, d_rgb, (size_t)n * 4, cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    std::memcpy(rgb, h->pin_out.p, (size_t)n * 3);
    std::memcpy(valid, static_cast<unsigned char*>(h->pin_out.p) + (size_t)n * 3, n);
    h->last_pass_valid = false;                       // the row-mask export buffer was reused
    return FLB_OK;
}

// bgr == NULL needs a colour frame of the camera's size in the current image set
int colorize_frame_check(flb_handle* h, const char* who, const uint8_t* bgr) {
    if (!bgr && !(h->img_bgr_valid && h->img_w == h->cam.width && h->img_h == h->cam.height))
        return fail(h, FLB_ERR_STATE, "%s: bgr == NULL needs the current image from flb_image_upload_bgr at the camera's size", who);
    return FLB_OK;
}

// Chunks for `need` save records, their pointers uploaded to rs_table on `stream` (a table that grows is reallocated:
// cudaFree waits for the scatters reading the old one).  *ok = false when the device has no memory for one more chunk:
// the frame is then dropped like one beyond the cap; the chunks that were allocated stay for later frames.
int rgb_save_reserve(flb_handle* h, long long need, bool* ok) {
    const size_t want = (size_t)((need + (1LL << kRgbChunkLog2) - 1) >> kRgbChunkLog2);
    while (h->rs_chunks.size() < want) {
        uint4* c = nullptr;
        if (cudaMalloc(&c, ((size_t)1 << kRgbChunkLog2) * sizeof(uint4)) != cudaSuccess) {
            cudaGetLastError();                       // an allocation failure is not sticky: clear it
            break;
        }
        h->rs_chunks.push_back(c);
    }
    if (h->rs_chunks.size() > h->rs_table_n) {
        FLB_CUDA(h, h->rs_table.reserve(h->rs_chunks.size()));
        FLB_CUDA(h, cudaMemcpyAsync(h->rs_table.p, h->rs_chunks.data(), h->rs_chunks.size() * sizeof(uint4*), cudaMemcpyHostToDevice,
                                    h->stream));
        h->rs_table_n = h->rs_chunks.size();
    }
    *ok = h->rs_chunks.size() >= want;
    return FLB_OK;
}

}  // namespace

extern "C" {

int flb_colorize(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, const float* world_xyz, int n,
                 int stride, uint8_t* rgb, uint8_t* valid) {
    FLB_CHECK_H(h);
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_colorize: flb_camera_set first");
    const int W = h->cam.width;
    if ((bgr && stride_bytes < 3 * W) || n < 0 || (n > 0 && (!world_xyz || !rgb || !valid)) || stride < 3)
        return fail(h, FLB_ERR_INVALID, "flb_colorize: bad arguments");
    { int rc = colorize_frame_check(h, "flb_colorize", bgr); if (rc) return rc; }
    if (n == 0) return FLB_OK;
    { int rc = colorize_pose(h, "flb_colorize", Rcw, Pcw); if (rc) return rc; }
    { int rc = vm_upload_points(h, world_xyz, n, stride); if (rc) return rc; }
    return colorize_dev(h, bgr, stride_bytes, h->vm.pg.p, n, rgb, valid);
}

// publish_frame_world_rgb of pcl_wait_pub (src/laserMapping.cpp:710-745) with the world cloud on the device.
int flb_colorize_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, uint8_t* rgb,
                       uint8_t* valid) {
    FLB_CHECK_H(h);
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_colorize_cloud: flb_camera_set first");
    { int rc = wc_check(h, "flb_colorize_cloud"); if (rc) return rc; }
    const int n = h->wc_n;
    if ((bgr && stride_bytes < 3 * h->cam.width) || (n > 0 && (!rgb || !valid))) return fail(h, FLB_ERR_INVALID, "flb_colorize_cloud: bad arguments");
    { int rc = colorize_frame_check(h, "flb_colorize_cloud", bgr); if (rc) return rc; }
    if (n == 0) return FLB_OK;
    { int rc = colorize_pose(h, "flb_colorize_cloud", Rcw, Pcw); if (rc) return rc; }
    return colorize_dev(h, bgr, stride_bytes, h->wc_xyz.p, n, rgb, valid);
}

// publish_frame_world_rgb's laserCloudWorldRGB (src/laserMapping.cpp:726-747) as 32-byte records on the device:
// k_rgb_flags colours every world point, cub's exclusive sum ranks the kept ones, the count is read back, and
// k_rgb_scatter writes each kept point's record (and, with the save on and room under its cap, its save record).
int flb_rgb_cloud(flb_handle* h, const double Rcw[9], const double Pcw[3], const uint8_t* bgr, int stride_bytes, int* n_out) {
    FLB_CHECK_H(h);
    h->rc_n = -1;                                     // on any error below, no cloud is held
    if (n_out) *n_out = 0;
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_rgb_cloud: flb_camera_set first");
    { int rc = wc_check(h, "flb_rgb_cloud"); if (rc) return rc; }
    const int n = h->wc_n;
    if (bgr && stride_bytes < 3 * h->cam.width) return fail(h, FLB_ERR_INVALID, "flb_rgb_cloud: bad arguments");
    { int rc = colorize_frame_check(h, "flb_rgb_cloud", bgr); if (rc) return rc; }
    if (n == 0) {
        h->rc_n = 0;
        return FLB_OK;
    }
    { int rc = colorize_pose(h, "flb_rgb_cloud", Rcw, Pcw); if (rc) return rc; }
    if (bgr) FLB_CUDA(h, h->rc_img.reserve((size_t)h->cam.width * h->cam.height * 3));
    FLB_CUDA(h, h->rc_bgra.reserve(n));
    FLB_CUDA(h, h->rc_flag.reserve((size_t)n + 1));
    FLB_CUDA(h, h->rc_pos.reserve((size_t)n + 1));
    const unsigned char* d_img = nullptr;
    { int rci = colorize_image(h, bgr, stride_bytes, h->rc_img.p, &d_img); if (rci) return rci; }
    {
        LaunchScope ls(h, FAM_OTHER);
        k_rgb_flags<<<(n + 1 + 255) / 256, 256, 0, h->stream>>>(h->cam, h->vm.pose.p, d_img, h->wc_xyz.p, n, h->rc_bgra.p, h->rc_flag.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    size_t tmp_bytes = 0;
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, h->rc_flag.p, h->rc_pos.p, n + 1, h->stream));
    FLB_CUDA(h, h->cub_tmp.reserve(tmp_bytes));
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(h->cub_tmp.p, tmp_bytes, h->rc_flag.p, h->rc_pos.p, n + 1, h->stream));
    h->launches++;
    FLB_CUDA(h, h->pin_out.reserve(sizeof(int)));
    int* cnt = static_cast<int*>(h->pin_out.p);
    FLB_CUDA(h, cudaMemcpyAsync(cnt, h->rc_pos.p + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    const int m = *cnt;
    uint4* const* table = nullptr;
    if (h->rs_on && m > 0) {
        bool ok = m <= h->rs_max - h->rs_n;
        if (ok) { int rcs = rgb_save_reserve(h, h->rs_n + m, &ok); if (rcs) return rcs; }
        if (ok) table = h->rs_table.p;
        else h->rs_dropped += m;                      // the frame's cloud is still built: saving never stops publishing
    }
    if (m > 0) {
        FLB_CUDA(h, h->rc_out.reserve(2 * (size_t)m));
        LaunchScope ls(h, FAM_OTHER);
        k_rgb_scatter<<<(n + 255) / 256, 256, 0, h->stream>>>(h->wc_xyz.p, h->rc_bgra.p, h->rc_flag.p, h->rc_pos.p, n, h->rc_out.p, table,
                                                              h->rs_n);
        FLB_CUDA(h, cudaGetLastError());
    }
    if (table) h->rs_n += m;
    h->rc_n = m;
    if (n_out) *n_out = m;
    return FLB_OK;
}

int flb_rgb_cloud_download(flb_handle* h, void* points32, int capacity, int* n_out) {
    FLB_CHECK_H(h);
    if (capacity < 0 || (capacity > 0 && !points32)) return fail(h, FLB_ERR_INVALID, "flb_rgb_cloud_download: bad arguments");
    if (h->rc_n < 0) return fail(h, FLB_ERR_STATE, "flb_rgb_cloud_download: no coloured cloud (flb_rgb_cloud first, or it failed)");
    if (n_out) *n_out = h->rc_n;
    const int m = std::min(capacity, h->rc_n);
    if (m > 0) {
        FLB_CUDA(h, cudaMemcpyAsync(points32, h->rc_out.p, (size_t)m * 2 * sizeof(uint4), cudaMemcpyDeviceToHost, h->stream));
        FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    return FLB_OK;
}

int flb_rgb_save_begin(flb_handle* h, int64_t max_points) {
    FLB_CHECK_H(h);
    if (max_points < 1) return fail(h, FLB_ERR_INVALID, "flb_rgb_save_begin: max_points %lld < 1", (long long)max_points);
    if (h->rs_on) return fail(h, FLB_ERR_STATE, "flb_rgb_save_begin: a save is open (flb_rgb_save_end first)");
    h->rs_on = true;
    h->rs_max = max_points;
    h->rs_n = h->rs_dropped = 0;
    return FLB_OK;
}

int flb_rgb_save_size(flb_handle* h, int64_t* n, int64_t* dropped, int64_t* device_bytes) {
    FLB_CHECK_H(h);
    if (!h->rs_on) return fail(h, FLB_ERR_STATE, "flb_rgb_save_size: no save open (flb_rgb_save_begin first)");
    if (n) *n = h->rs_n;
    if (dropped) *dropped = h->rs_dropped;
    if (device_bytes)
        *device_bytes = (int64_t)(h->rs_chunks.size() * ((size_t)1 << kRgbChunkLog2) * sizeof(uint4) + h->rs_table.cap * sizeof(uint4*) +
                                  h->rs_pack.cap * sizeof(uint4));
    return FLB_OK;
}

int flb_rgb_save_download(flb_handle* h, int64_t first, int64_t count, void* points32) {
    FLB_CHECK_H(h);
    if (!h->rs_on) return fail(h, FLB_ERR_STATE, "flb_rgb_save_download: no save open (flb_rgb_save_begin first)");
    if (first < 0 || count < 0 || count > h->rs_n - first || (count > 0 && !points32))
        return fail(h, FLB_ERR_INVALID, "flb_rgb_save_download: bad arguments (records %lld + %lld of %lld)", (long long)first,
                    (long long)count, h->rs_n);
    if (count == 0) return FLB_OK;
    // One bounded slice at a time: k_rgb_save_pack expands it into rs_pack, the copy takes it out; stream order keeps
    // the next slice's pack behind the copy.
    constexpr long long kSlice = 1LL << 18;
    FLB_CUDA(h, h->rs_pack.reserve(2 * (size_t)std::min<long long>(count, kSlice)));
    char* dst = static_cast<char*>(points32);
    for (long long done = 0; done < count; done += kSlice) {
        const int k = (int)std::min<long long>(count - done, kSlice);
        {
            LaunchScope ls(h, FAM_OTHER);
            k_rgb_save_pack<<<(k + 255) / 256, 256, 0, h->stream>>>(h->rs_table.p, first + done, k, h->rs_pack.p);
            FLB_CUDA(h, cudaGetLastError());
        }
        FLB_CUDA(h, cudaMemcpyAsync(dst + done * 2 * (long long)sizeof(uint4), h->rs_pack.p, (size_t)k * 2 * sizeof(uint4),
                                    cudaMemcpyDeviceToHost, h->stream));
    }
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_rgb_save_end(flb_handle* h) {
    FLB_CHECK_H(h);
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    rgb_save_free(h);
    return FLB_OK;
}

// LidarSelector::display_keypatch (src/lidar_selection.cpp:985-1005) without its text, into a copy of the current colour
// frame: k_kp_stamp marks each pixel with the highest patch index whose disk covers it, k_kp_compose colours it.
int flb_keypatch_image(flb_handle* h, const double Rcw[9], const double Pcw[3], uint8_t* bgr_out, int stride_bytes, int* n_patches) {
    FLB_CHECK_H(h);
    if (!bgr_out || (!Rcw != !Pcw)) return fail(h, FLB_ERR_INVALID, "flb_keypatch_image: bad arguments");
    if (!h->cam_set) return fail(h, FLB_ERR_STATE, "flb_keypatch_image: flb_camera_set first");
    const int W = h->cam.width, H = h->cam.height;
    if (stride_bytes < 3 * W) return fail(h, FLB_ERR_INVALID, "flb_keypatch_image: stride_bytes %d < 3 * %d", stride_bytes, W);
    { int rc = colorize_frame_check(h, "flb_keypatch_image", nullptr); if (rc) return rc; }
    if (h->comm || h->p2p.world > 1) return fail(h, FLB_ERR_STATE, "flb_keypatch_image: each rank holds only its shard of the patch list");
    if (!h->patches_set) return fail(h, FLB_ERR_STATE, "flb_keypatch_image: no patch list (flb_vmap_select* or flb_patches_upload)");
    { int rc = colorize_pose(h, "flb_keypatch_image", Rcw, Pcw); if (rc) return rc; }
    const size_t npix = (size_t)W * H;
    FLB_CUDA(h, h->kp_owner.reserve(npix));
    FLB_CUDA(h, h->kp_out.reserve(npix * 3));
    { int rcq = vio_inputs_acquire(h); if (rcq) return rcq; }                      // the colour frame and the patches have landed
    const int n = h->pn_on_device ? h->vm.prm.length : h->Pn;
    const int* n_dev = h->pn_on_device ? h->vm.counters.p + VM_N_SEL : nullptr;
    const float* errors = h->err_from_sel ? h->vm.sel_error.p : h->errors.p;
    const int* err_half = h->err_from_sel ? nullptr : &h->vio_ctrl.p->err_buf;
    {
        LaunchScope ls(h, FAM_OTHER);
        FLB_CUDA(h, cudaMemsetAsync(h->kp_owner.p, 0xff, npix * sizeof(int), h->stream));
        if (n > 0)
            k_kp_stamp<<<(unsigned)(((size_t)n * 32 + 255) / 256), 256, 0, h->stream>>>(h->cam, h->vm.pose.p, h->patch_pos.p, n, n_dev, W, H,
                                                                                   h->kp_owner.p);
        k_kp_compose<<<(unsigned)((npix + 255) / 256), 256, 0, h->stream>>>(h->img_bgr.p, h->kp_owner.p, errors, err_half, h->err_stride,
                                                                            (int)npix, h->kp_out.p);
        FLB_CUDA(h, cudaGetLastError());
        if (n > 0) h->launches++;
    }
    FLB_CUDA(h, cudaMemcpy2DAsync(bgr_out, stride_bytes, h->kp_out.p, (size_t)W * 3, (size_t)W * 3, H, cudaMemcpyDeviceToHost, h->stream));
    if (n_patches) {
        if (n_dev) FLB_CUDA(h, cudaMemcpyAsync(n_patches, n_dev, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        else *n_patches = h->Pn;
    }
    if (!is_pinned(bgr_out)) FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_vmap_counts(flb_handle* h, int* points, int* features, int* images, int* selected, int* last_added) {
    FLB_CHECK_H(h);
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "flb_vmap_counts: flb_vmap_reset first");
    int c[VM_COUNTERS];
    FLB_CUDA(h, cudaMemcpyAsync(c, h->vm.counters.p, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    h->vm.pts_ub = c[VM_N_POINTS];
    h->vm.fts_ub = c[VM_N_FEATS];
    h->vm.img_ub = c[VM_N_IMAGES] - c[VM_N_FREE];
    if (points) *points = c[VM_N_POINTS];
    if (features) *features = c[VM_N_FEATS];
    if (images) *images = c[VM_N_IMAGES] - c[VM_N_FREE];
    if (selected) *selected = c[VM_N_SEL];
    if (last_added) *last_added = c[VM_LAST_ADDED];
    if (c[VM_LAST_ADDED] < 0) return fail(h, FLB_ERR_STATE, "visual map: an append did not fit its buffers (internal capacity bound violated)");
    return FLB_OK;
}

int flb_vmap_map_value(flb_handle* h, float* out, int capacity) {
    FLB_CHECK_H(h);
    if (!h->vm.on || !out) return fail(h, FLB_ERR_STATE, "flb_vmap_map_value: flb_vmap_reset first");
    const size_t n = (size_t)std::min(capacity, h->vm.prm.length);
    FLB_CUDA(h, cudaMemcpyAsync(out, h->vm.map_value.p, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    return FLB_OK;
}

int flb_vmap_dump(flb_handle* h, int cap_points, int cap_features, double* pos, float* value, int* n_obs, int* obs20, double* ft_geo17,
                  float* ft_score, int* ft_level_id_img) {
    FLB_CHECK_H(h);
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "flb_vmap_dump: flb_vmap_reset first");
    int np = 0, nf = 0;
    { int rc = flb_vmap_counts(h, &np, &nf, nullptr, nullptr, nullptr); if (rc) return rc; }
    np = std::min(np, cap_points);
    nf = std::min(nf, cap_features);
    std::vector<VmPoint> P((size_t)np);
    std::vector<VmFeature> F((size_t)nf);
    if (np) FLB_CUDA(h, cudaMemcpy(P.data(), h->vm.pts.p, (size_t)np * sizeof(VmPoint), cudaMemcpyDeviceToHost));
    if (nf) FLB_CUDA(h, cudaMemcpy(F.data(), h->vm.fts.p, (size_t)nf * sizeof(VmFeature), cudaMemcpyDeviceToHost));
    for (int j = 0; j < np; ++j) {
        if (pos) std::memcpy(pos + 3 * (size_t)j, P[j].pos, 3 * sizeof(double));
        if (value) value[j] = P[j].value;
        if (n_obs) n_obs[j] = P[j].n_obs;
        if (obs20) for (int q = 0; q < 20; ++q) obs20[20 * (size_t)j + q] = q < P[j].n_obs ? P[j].obs[q] : -1;
    }
    for (int j = 0; j < nf; ++j) {
        if (ft_geo17) {
            double* g = ft_geo17 + 17 * (size_t)j;
            g[0] = F[j].px[0]; g[1] = F[j].px[1];
            std::memcpy(g + 2, F[j].f, 3 * sizeof(double));
            std::memcpy(g + 5, F[j].R, 9 * sizeof(double));
            std::memcpy(g + 14, F[j].t, 3 * sizeof(double));
        }
        if (ft_score) ft_score[j] = F[j].score;
        if (ft_level_id_img) { ft_level_id_img[3 * (size_t)j] = F[j].level; ft_level_id_img[3 * (size_t)j + 1] = F[j].id; ft_level_id_img[3 * (size_t)j + 2] = F[j].img; }
    }
    return FLB_OK;
}

int flb_vmap_reclaim(flb_handle* h) {
    FLB_CHECK_H(h);
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "flb_vmap_reclaim: flb_vmap_reset first");
    auto& vm = h->vm;
    { int rc = vm_reclaim_reserve(h); if (rc) return rc; }
    // The host bounds size the grids and the scan; the kernels stop at the device counts.  Features between the device
    // count and the bound are never named, so their flags stay 0 and rank[M] is the number of live features.
    const int M = vm.fts_ub;
    const size_t point_words = (size_t)std::max(vm.pts_ub, 1) * kVmPointWords, feat_words = (size_t)std::max(M, 1) * kVmFeatWords;
    auto blocks = [h](size_t words) { return (int)std::min<size_t>((words + 255) / 256, (size_t)h->num_sms * 8); };
    cudaStream_t s = h->stream;
    FLB_CUDA(h, cudaMemsetAsync(vm.rc_rank.p, 0, (size_t)(M + 1) * sizeof(int), s));
    FLB_CUDA(h, cudaMemsetAsync(vm.rc_slot.p, 0, (size_t)vm.pool_slots * sizeof(int), s));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_rc_mark<<<blocks(point_words), 256, 0, s>>>(vm.pts.p, vm.counters.p, vm.rc_rank.p);
        FLB_CUDA(h, cudaGetLastError());
    }
    size_t bytes = vm.rc_cub_bytes;
    FLB_CUDA(h, cub::DeviceScan::ExclusiveSum(vm.rc_cub.p, bytes, vm.rc_rank.p, vm.rc_rank.p, M + 1, s));
    {
        LaunchScope ls(h, FAM_OTHER);
        k_vm_rc_compact<<<blocks(feat_words), 256, 0, s>>>(vm.fts.p, vm.fts_alt.p, vm.rc_rank.p, vm.counters.p, vm.rc_slot.p);
        k_vm_rc_remap<<<blocks(point_words), 256, 0, s>>>(vm.pts.p, vm.rc_rank.p, vm.counters.p);
        k_vm_rc_slots<<<1, 1024, 0, s>>>(vm.counters.p, vm.rc_rank.p + M, vm.rc_slot.p, std::max(vm.pool_slots, 1), vm.free_slots.p);
        FLB_CUDA(h, cudaGetLastError());
        h->launches += 4;                   // + the scan's two kernels
    }
    std::swap(vm.fts, vm.fts_alt);
    return FLB_OK;
}

int flb_vmap_usage(flb_handle* h, int* points, int* features, int* dead_features, int* feature_capacity, int* slots_in_use, int* free_slots,
                   int* pool_slots, int64_t* device_bytes) {
    FLB_CHECK_H(h);
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "flb_vmap_usage: flb_vmap_reset first");
    auto& vm = h->vm;
    int c[VM_COUNTERS];
    FLB_CUDA(h, cudaMemcpyAsync(c, vm.counters.p, sizeof(c), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    vm.pts_ub = c[VM_N_POINTS];
    vm.fts_ub = c[VM_N_FEATS];
    vm.img_ub = c[VM_N_IMAGES] - c[VM_N_FREE];
    if (dead_features) {
        std::vector<VmPoint> P((size_t)c[VM_N_POINTS]);
        if (!P.empty()) FLB_CUDA(h, cudaMemcpy(P.data(), vm.pts.p, P.size() * sizeof(VmPoint), cudaMemcpyDeviceToHost));
        std::vector<unsigned char> named((size_t)c[VM_N_FEATS], 0);
        for (const VmPoint& p : P)
            for (int q = 0; q < p.n_obs; ++q) named[p.obs[q]] = 1;
        *dead_features = c[VM_N_FEATS] - (int)std::count(named.begin(), named.end(), 1);
    }
    if (points) *points = c[VM_N_POINTS];
    if (features) *features = c[VM_N_FEATS];
    if (feature_capacity) *feature_capacity = (int)vm.fts.cap;
    if (slots_in_use) *slots_in_use = c[VM_N_IMAGES] - c[VM_N_FREE];
    if (free_slots) *free_slots = c[VM_N_FREE];
    if (pool_slots) *pool_slots = vm.pool_slots;
    if (device_bytes) {
        int64_t b = 0;
        auto add = [&b](const auto& buf) { b += (int64_t)(buf.cap * sizeof(*buf.p)); };
        add(vm.pts); add(vm.fts); add(vm.fts_alt); add(vm.pool); add(vm.counters); add(vm.pose); add(vm.rci); add(vm.pg);
        add(vm.depth); add(vm.keyset); add(vm.cell_best); add(vm.cand_key); add(vm.cell_type); add(vm.map_value); add(vm.cell_err);
        add(vm.cell_patch); add(vm.sel_error); add(vm.cell_flag); add(vm.cell_rank); add(vm.cell_level); add(vm.cell_point);
        add(vm.sel_index); add(vm.sel_point); add(vm.winner); add(vm.scan_tmp); add(vm.free_slots); add(vm.rc_rank); add(vm.rc_slot);
        add(vm.rc_cub);
        *device_bytes = b;
    }
    return FLB_OK;
}

int flb_vmap_keyframe(flb_handle* h, int slot, uint8_t* gray, int capacity) {
    FLB_CHECK_H(h);
    if (!h->vm.on) return fail(h, FLB_ERR_STATE, "flb_vmap_keyframe: flb_vmap_reset first");
    const size_t img_bytes = (size_t)h->img_w * h->img_h;
    if (!gray || capacity < 0 || (size_t)capacity < img_bytes) return fail(h, FLB_ERR_INVALID, "flb_vmap_keyframe: bad arguments");
    int tail = 0;
    FLB_CUDA(h, cudaMemcpyAsync(&tail, h->vm.counters.p + VM_N_IMAGES, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    FLB_CUDA(h, cudaStreamSynchronize(h->stream));
    if (slot < 0 || slot >= tail) return fail(h, FLB_ERR_INVALID, "flb_vmap_keyframe: slot %d outside the pool's %d slots", slot, tail);
    FLB_CUDA(h, cudaMemcpy(gray, h->vm.pool.p + (size_t)slot * img_bytes, img_bytes, cudaMemcpyDeviceToHost));
    return FLB_OK;
}

}  // extern "C"
