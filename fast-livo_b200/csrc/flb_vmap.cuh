// flb_vmap.cuh -- device-resident visual map (SURVEY.md section 8 rows f2 and f4) for sm_90a.
//
//   select   LidarSelector::addFromSparseMap (src/lidar_selection.cpp:346-587): scan-voxel set + sparse depth image,
//            per-grid-cell closest visible map point, depth-continuity test, closest-view observation
//            (src/point.cpp:141-178), affine warp of the reference patch at three pyramid levels (:232-296), NCC / SSD
//            gates -- the patch list lands in the VIO kernel's input buffers, in place, on the device
//   grow     LidarSelector::addSparseMap (:142-202): Shi-Tomasi candidate per grid cell (k_vmap_* in flb_kernels.cuh),
//            then one new Point + Feature per won cell
//   observe  LidarSelector::addObservation (:913-965): new observations of the selected points, oldest-view eviction
//
// The map is three flat arrays (VmPoint, VmFeature, keyframe images) that only ever grow at the tail, so ids are
// stable and equal to the reference's creation order.  Every per-element function lives in flb_device.cuh and is
// checked bit for bit against the oracle on the CPU (tests/hostemu); the kernels below only distribute the work:
// per-point kernels use 64-bit atomics whose winner is order-independent ({distance bits : ~index} minimum,
// {index : depth bits} maximum), per-cell work is one warp per cell, appends are ordered by a block-wide scan.
#pragma once

#include <cuda_runtime.h>
#include "flb_device.cuh"

namespace flb {

// counters (device-resident; mirrored on the host only when a caller asks)
enum { VM_N_POINTS = 0, VM_N_FEATS = 1, VM_N_SEL = 2, VM_N_IMAGES = 3, VM_IMG_FRAME = 4, VM_IMG_SLOT = 5, VM_LAST_ADDED = 6, VM_COUNTERS = 8 };

constexpr unsigned long long kVmEmpty = ~0ull;

struct VmWarpCtx {
    int lane, n;
    __device__ __forceinline__ void sync() const { __syncwarp(); }
    __device__ __forceinline__ bool any(bool b) const { return __any_sync(0xffffffffu, b); }
};

// T_f_w of the current frame from the device state (LidarSelector::updateFrameState, :905-911):
// Rcw = Rci * Rwi^T, Pcw = -Rci * Rwi^T * Pwi + Pci
__global__ void __launch_bounds__(32) k_vm_pose_from_state(const State18* x, const double* Rci_Pci, double* pose12) {
    if (threadIdx.x != 0) return;
    double Rt[9], t[3];
    m3_T(x->rot, Rt);
    m3_mul(Rci_Pci, Rt, pose12);
    m3_vec(pose12, x->pos, t);
    for (int i = 0; i < 3; ++i) pose12[9 + i] = -t[i] + Rci_Pci[9 + i];
}

// One pass over everything a selection starts from: depth image, scan-voxel set, per-cell claims.
__global__ void k_vm_clear(unsigned long long* depth, size_t n_depth, unsigned long long* keyset, size_t n_keys, unsigned long long* cell_best,
                           unsigned char* cell_type, float* map_value, int* cell_flag, int length, int* counters) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = i; e < n_depth; e += stride) depth[e] = 0ull;
    for (size_t e = i; e < n_keys; e += stride) keyset[e] = kVmEmpty;
    for (size_t e = i; e < (size_t)length; e += stride) {
        cell_best[e] = kVmEmpty;
        cell_type[e] = 0;
        map_value[e] = 0.0f;                                                      // :356
        cell_flag[e] = 0;
    }
    if (i == 0) counters[VM_N_SEL] = 0;
}

__device__ __forceinline__ unsigned vm_hash(unsigned long long k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (unsigned)k;
}

// First loop (:378-418): every voxel-filtered scan point marks its 0.5 m voxel and writes its depth into the pixel
// it projects to (the LAST point of the cloud wins a pixel: maximum over {index + 1 : depth bits}).
__global__ void k_vm_scan(CamModel cam, const double* __restrict__ pose12, const float* __restrict__ pg_down, int n, int border,
                          unsigned long long* __restrict__ keyset, unsigned key_mask, unsigned long long* __restrict__ depth,
                          const int* __restrict__ counters) {
    if (counters[VM_N_POINTS] <= 0) return;                                       // :348
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float p[3] = {pg_down[3 * (size_t)i], pg_down[3 * (size_t)i + 1], pg_down[3 * (size_t)i + 2]};
    const unsigned long long key = vm_scan_key(p);
    unsigned slot = vm_hash(key) & key_mask;
    for (;;) {
        const unsigned long long prev = atomicCAS(keyset + slot, kVmEmpty, key);
        if (prev == kVmEmpty || prev == key) break;
        slot = (slot + 1) & key_mask;
    }
    double Rcw[9], Pcw[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) Rcw[k] = pose12[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) Pcw[k] = pose12[9 + k];
    const double pt_w[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double pt_c[3];
    se3_apply(Rcw, Pcw, pt_w, pt_c);
    if (pt_c[2] > 0) {
        const double px0 = cam.jfx * pt_c[0] / pt_c[2] + cam.cx, px1 = cam.jfy * pt_c[1] / pt_c[2] + cam.cy;   // :399-400
        if (vm_in_frame(cam, px0, px1, border)) {
            const float d = (float)pt_c[2];
            atomicMax(depth + (size_t)cam.width * (int)px1 + (int)px0, ((unsigned long long)(i + 1) << 32) | float_as_u32(d));
        }
    }
}

__device__ __forceinline__ bool vm_key_present(const unsigned long long* keyset, unsigned key_mask, unsigned long long key) {
    unsigned slot = vm_hash(key) & key_mask;
    for (;;) {
        const unsigned long long v = keyset[slot];
        if (v == key) return true;
        if (v == kVmEmpty) return false;
        slot = (slot + 1) & key_mask;
    }
}

// Second loop (:430-470): every map point whose voxel was touched by the scan claims its grid cell; per cell the
// closest point wins (`cur_dist <= map_dist`, later visited wins a tie: here the higher point id), the cell's value is
// the maximum point value.
__global__ void k_vm_candidates(CamModel cam, VmParams prm, const double* __restrict__ pose12, const VmPoint* __restrict__ pts,
                                const int* __restrict__ counters, const unsigned long long* __restrict__ keyset, unsigned key_mask,
                                int border, unsigned long long* __restrict__ cell_best, unsigned char* __restrict__ cell_type,
                                int* __restrict__ map_value_bits) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= counters[VM_N_POINTS]) return;
    const VmPoint& pt = pts[j];
    if (!vm_key_present(keyset, key_mask, vm_pack_key(pt.key[0], pt.key[1], pt.key[2]))) return;
    double Rcw[9], Pcw[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) Rcw[k] = pose12[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) Pcw[k] = pose12[9 + k];
    double pt_cam[3], pc[2], frame_pos[3];
    se3_apply(Rcw, Pcw, pt.pos, pt_cam);
    if (pt_cam[2] < 0) return;
    world2cam(cam, pt_cam, pc);
    if (!vm_in_frame(cam, pc[0], pc[1], border)) return;
    const int index = (int)(pc[0] / prm.grid_size) * prm.grid_n_height + (int)(pc[1] / prm.grid_size);
    cell_type[index] = 1;                                                         // TYPE_MAP
    se3_pos(Rcw, Pcw, frame_pos);
    const double ov[3] = {frame_pos[0] - pt.pos[0], frame_pos[1] - pt.pos[1], frame_pos[2] - pt.pos[2]};
    const float cur_dist = (float)norm3(ov);
    if (cur_dist <= 10000.0f)
        atomicMin(cell_best + index, ((unsigned long long)float_as_u32(cur_dist) << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)j));
    // cur_value >= map_value[index] (values are >= 0 or tiny negatives: as signed ints, float order is preserved
    // for non-negative values and every negative value stays below the initial 0)
    atomicMax(map_value_bits + index, (int)float_as_u32(pt.value));
}

// Third loop (:479-580): one warp per grid cell.
constexpr int kVmBuildWarps = 8;
__global__ void __launch_bounds__(kVmBuildWarps * 32) k_vm_build(CamModel cam, VmParams prm, const double* __restrict__ pose12,
                                                                 const VmPoint* __restrict__ pts, const VmFeature* __restrict__ feats,
                                                                 const unsigned char* __restrict__ img_pool,
                                                                 const unsigned char* __restrict__ img_cur,
                                                                 const unsigned long long* __restrict__ depth,
                                                                 const unsigned long long* __restrict__ cell_best,
                                                                 const unsigned char* __restrict__ cell_type, const int* __restrict__ counters,
                                                                 int* __restrict__ cell_flag, int* __restrict__ cell_level,
                                                                 int* __restrict__ cell_point, float* __restrict__ cell_err,
                                                                 float* __restrict__ cell_patch) {
    __shared__ float s_wrap[kVmBuildWarps][192];
    __shared__ float s_cur[kVmBuildWarps][64];
    __shared__ double s_sh[kVmBuildWarps][8];
    if (counters[VM_N_POINTS] <= 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kVmBuildWarps + warp;
    if (i >= prm.length) return;
    if (!cell_type[i] || cell_best[i] == kVmEmpty) return;
    const int pj = (int)(0xFFFFFFFFu - (unsigned)(cell_best[i] & 0xFFFFFFFFull));
    double Rcw[9], Pcw[3], frame_pos[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) Rcw[k] = pose12[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) Pcw[k] = pose12[9 + k];
    se3_pos(Rcw, Pcw, frame_pos);
    VmWarpCtx cx{lane, 32};
    int level = 0;
    float error = 0.0f;
    const bool keep = vm_build_cell(cx, cam, prm, Rcw, Pcw, frame_pos, pts[pj], feats, img_pool, img_cur, depth, s_wrap[warp], s_cur[warp],
                                    s_sh[warp], &level, &error);
    if (!keep) return;
    for (int e = lane; e < 192; e += 32) cell_patch[(size_t)i * 192 + e] = s_wrap[warp][e];
    if (lane == 0) {
        cell_flag[i] = 1;
        cell_level[i] = level;
        cell_point[i] = pj;
        cell_err[i] = error;
    }
}

// Block-wide exclusive scan of flags[0..n) (n arbitrary) by ONE block of 1024 threads; rank[i] = number of set flags
// before i, *total = their count.  Order-preserving: this is what makes every append deterministic.
__device__ __forceinline__ void vm_block_scan(const int* __restrict__ flags, int n, int* __restrict__ rank, int* total_out) {
    __shared__ int s_part[1024];
    __shared__ int s_total;
    const int tid = threadIdx.x;
    const int per = (n + 1023) / 1024;
    const int a = min(n, tid * per), b = min(n, a + per);
    int c = 0;
    for (int i = a; i < b; ++i) c += flags[i] ? 1 : 0;
    s_part[tid] = c;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
        const int v = tid >= off ? s_part[tid - off] : 0;
        __syncthreads();
        s_part[tid] += v;
        __syncthreads();
    }
    int run = s_part[tid] - c;
    for (int i = a; i < b; ++i) {
        rank[i] = run;
        run += flags[i] ? 1 : 0;
    }
    if (tid == 1023) s_total = s_part[1023];
    __syncthreads();
    *total_out = s_total;
}

__global__ void __launch_bounds__(1024) k_vm_rank(const int* __restrict__ cell_flag, int length, int* __restrict__ cell_rank, int* counters) {
    int total;
    vm_block_scan(cell_flag, length, cell_rank, &total);
    if (threadIdx.x == 0) counters[VM_N_SEL] = total;
}

// sub_sparse_map, in cell order (:566-571): straight into the VIO kernel's inputs.
__global__ void __launch_bounds__(256) k_vm_scatter(int length, const int* __restrict__ cell_flag, const int* __restrict__ cell_rank,
                                                    const int* __restrict__ cell_level, const int* __restrict__ cell_point,
                                                    const float* __restrict__ cell_err, const float* __restrict__ cell_patch,
                                                    const VmPoint* __restrict__ pts, double* __restrict__ patch_pos,
                                                    float* __restrict__ patch_ref, int* __restrict__ patch_level, int* __restrict__ sel_index,
                                                    int* __restrict__ sel_point, float* __restrict__ sel_error) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * 8 + warp;
    if (i >= length || !cell_flag[i]) return;
    const int k = cell_rank[i];
    for (int e = lane; e < 192; e += 32) patch_ref[(size_t)k * 192 + e] = cell_patch[(size_t)i * 192 + e];
    if (lane < 3) patch_pos[3 * (size_t)k + lane] = pts[cell_point[i]].pos[lane];
    if (lane == 3) patch_level[k] = cell_level[i];
    if (lane == 4) sel_index[k] = i;
    if (lane == 5) sel_point[k] = cell_point[i];
    if (lane == 6) sel_error[k] = cell_err[i];
}

// The keyframe image of the current frame goes into the next free pool slot unless this frame already has one.  The
// slot only becomes part of the map when a feature referencing it is appended (k_vm_materialise / k_vm_observe).
__global__ void k_vm_store_image(const unsigned char* __restrict__ img, size_t bytes, unsigned char* __restrict__ pool, const int* counters,
                                 int frame_id) {
    if (counters[VM_IMG_FRAME] == frame_id && counters[VM_IMG_SLOT] >= 0) return;
    unsigned char* dst = pool + (size_t)counters[VM_N_IMAGES] * bytes;
    const size_t n16 = bytes / 16;
    const uint4* s4 = reinterpret_cast<const uint4*>(img);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = i; e < n16; e += stride) d4[e] = s4[e];
    for (size_t e = n16 * 16 + i; e < bytes; e += stride) dst[e] = img[e];
}

__device__ __forceinline__ int vm_commit_image(int* counters, int frame_id) {     // thread 0 only
    if (!(counters[VM_IMG_FRAME] == frame_id && counters[VM_IMG_SLOT] >= 0)) {
        counters[VM_IMG_SLOT] = counters[VM_N_IMAGES];
        counters[VM_N_IMAGES] += 1;
        counters[VM_IMG_FRAME] = frame_id;
    }
    return counters[VM_IMG_SLOT];
}

__device__ __forceinline__ void vm_write_feature(const CamModel& cam, VmFeature& ft, const double* pc, const double* pose12, float score,
                                                 int level, int id, int img) {
    ft.px[0] = pc[0]; ft.px[1] = pc[1];
    cam2world(cam, pc[0], pc[1], ft.f);
    for (int k = 0; k < 9; ++k) ft.R[k] = pose12[k];
    for (int k = 0; k < 3; ++k) ft.t[k] = pose12[9 + k];
    ft.score = score; ft.level = level; ft.id = id; ft.img = img;
}

// addSparseMap's second loop (:171-195) + AddPoint (:204-230): one new Point with one Feature per won cell, cell order.
__global__ void __launch_bounds__(1024) k_vm_materialise(CamModel cam, int length, const double* __restrict__ pose12,
                                                         const float* __restrict__ pg, const int* __restrict__ winner,
                                                         const float* __restrict__ map_value, int* __restrict__ rank_tmp,
                                                         VmPoint* __restrict__ pts, VmFeature* __restrict__ feats, int* counters,
                                                         int frame_id, int pts_cap, int fts_cap) {
    __shared__ int s_slot, s_base_p, s_base_f;
    // flags = winner >= 0 (rank_tmp doubles as the flag array first)
    for (int i = threadIdx.x; i < length; i += 1024) rank_tmp[length + i] = winner[i] >= 0 ? 1 : 0;
    __syncthreads();
    int total;
    vm_block_scan(rank_tmp + length, length, rank_tmp, &total);
    if (threadIdx.x == 0) {
        s_base_p = counters[VM_N_POINTS];
        s_base_f = counters[VM_N_FEATS];
        const bool fits = s_base_p + total <= pts_cap && s_base_f + total <= fts_cap;
        s_slot = (total > 0 && fits) ? vm_commit_image(counters, frame_id) : -1;
        counters[VM_LAST_ADDED] = fits ? total : -1;
        if (fits) { counters[VM_N_POINTS] = s_base_p + total; counters[VM_N_FEATS] = s_base_f + total; }
    }
    __syncthreads();
    if (s_slot < 0) return;
    for (int i = threadIdx.x; i < length; i += 1024) {
        if (winner[i] < 0) continue;
        const int k = rank_tmp[i];
        const float* q = pg + 3 * (size_t)winner[i];
        const double pt[3] = {(double)q[0], (double)q[1], (double)q[2]};
        double pf[3], pc[2];
        se3_apply(pose12, pose12 + 9, pt, pf);
        world2cam(cam, pf, pc);
        VmPoint& p = pts[s_base_p + k];
        p.pos[0] = pt[0]; p.pos[1] = pt[1]; p.pos[2] = pt[2];
        p.value = map_value[i];
        p.n_obs = 1;
        vm_feat_key(pt, p.key);
        p.obs[0] = s_base_f + k;
        vm_write_feature(cam, feats[s_base_f + k], pc, pose12, map_value[i], 0, frame_id, s_slot);
    }
}

// addObservation (:913-965) over the sub_sparse_map of the last selection.  Each selected point belongs to one grid
// cell, so the per-point list updates are independent; the new features are appended in patch order.
__global__ void __launch_bounds__(1024) k_vm_observe(CamModel cam, const double* __restrict__ pose12, const unsigned char* __restrict__ img,
                                                     const int* __restrict__ sel_point, const int* __restrict__ patch_level,
                                                     int* __restrict__ flag_rank /* 2 x cap */, int cap, VmPoint* __restrict__ pts,
                                                     VmFeature* __restrict__ feats, int* counters, int frame_id, int fts_cap) {
    __shared__ int s_slot, s_base_f;
    const int n = counters[VM_N_SEL];
    if (n <= 0) {
        if (threadIdx.x == 0) counters[VM_LAST_ADDED] = 0;
        return;
    }
    double cur_pos[3];
    se3_pos(pose12, pose12 + 9, cur_pos);
    int* flag = flag_rank + cap;
    for (int i = threadIdx.x; i < n; i += 1024) {
        VmPoint& pt = pts[sel_point[i]];
        double pc[2];
        int erase_slot;
        const bool add_flag = vm_observation_test(cam, pose12, pose12 + 9, cur_pos, pt, feats, pc, &erase_slot);
        if (erase_slot >= 0) {                                                    // deleteFeatureRef(getFurthestViewObs), :946-952
            for (int q = erase_slot; q + 1 < pt.n_obs; ++q) pt.obs[q] = pt.obs[q + 1];
            pt.n_obs--;
        }
        flag[i] = add_flag ? 1 : 0;
    }
    __syncthreads();
    int total;
    vm_block_scan(flag, n, flag_rank, &total);
    if (threadIdx.x == 0) {
        s_base_f = counters[VM_N_FEATS];
        const bool fits = s_base_f + total <= fts_cap;
        s_slot = (total > 0 && fits) ? vm_commit_image(counters, frame_id) : -1;
        counters[VM_LAST_ADDED] = fits ? total : -1;
        if (fits) counters[VM_N_FEATS] = s_base_f + total;
    }
    __syncthreads();
    if (s_slot < 0) return;
    for (int i = threadIdx.x; i < n; i += 1024) {
        if (!flag[i]) continue;
        VmPoint& pt = pts[sel_point[i]];
        double pf[3], pc[2];
        se3_apply(pose12, pose12 + 9, pt.pos, pf);
        world2cam(cam, pf, pc);
        pt.value = shi_tomasi_score(img, cam.width, cam.height, cam.width, (int)pc[0], (int)pc[1]);      // :955
        const int fi = s_base_f + flag_rank[i];
        vm_write_feature(cam, feats[fi], pc, pose12, pt.value, patch_level[i], frame_id, s_slot);         // :957
        for (int q = pt.n_obs; q > 0; --q) pt.obs[q] = pt.obs[q - 1];            // addFrameRef: push_front
        pt.obs[0] = fi;
        pt.n_obs++;
    }
}

// publish_frame_world_rgb (src/laserMapping.cpp:710-745): per point, r g b + a validity flag
__global__ void k_vm_colorize(CamModel cam, const double* __restrict__ pose12, const unsigned char* __restrict__ bgr,
                              const float* __restrict__ xyz, int n, unsigned char* __restrict__ rgb, unsigned char* __restrict__ valid) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double Rcw[9], Pcw[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) Rcw[k] = pose12[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) Pcw[k] = pose12[9 + k];
    unsigned char c[3] = {0, 0, 0};
    const float p[3] = {xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
    const bool ok = vm_colorize_point(cam, Rcw, Pcw, bgr, p, c);
    rgb[3 * (size_t)i] = c[0]; rgb[3 * (size_t)i + 1] = c[1]; rgb[3 * (size_t)i + 2] = c[2];
    valid[i] = ok ? 1 : 0;
}

}  // namespace flb
