// flb_device.cuh -- per-thread device math of the FAST-LIVO hot path (sm_90a).
//
// Everything here is a pure function of its arguments, compiled with
// -fmad=false so that every float/double expression rounds exactly as written
// (the reference's x86-64 build has no FMA contraction either).  The functions are
// FLB_HD so that tests/hostemu can compile the very same source with g++ and check
// it against the oracle without a GPU; the product library only ever calls them
// from __global__ kernels (kernels.cu).
//
// Reference citations are relative to hku-mars/FAST-LIVO @ dcebf84.
#pragma once

#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#if !defined(__CUDACC__)
#include <algorithm>
using std::max;
using std::min;
#endif

#if defined(__CUDACC__)
#define FLB_HD __host__ __device__ __forceinline__
#define FLB_UNROLL _Pragma("unroll")
#else
#define FLB_HD inline
#define FLB_UNROLL
#endif

namespace flb {

FLB_HD float u32_as_float(unsigned u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, sizeof(f));
    return f;
#endif
}
FLB_HD unsigned float_as_u32(float f) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(f);
#else
    unsigned u;
    memcpy(&u, &f, sizeof(u));
    return u;
#endif
}

constexpr int kMatch = 5;    // NUM_MATCH_POINTS, include/common_lib.h:39
constexpr int kDim = 18;     // DIM_STATE,        include/common_lib.h:34
constexpr int kPatch = 8;    // patch_size (every config), patch_size_total = 64

// ------------------------------------------------------------------ 3x3 helpers
FLB_HD void m3_mul(const double* A, const double* B, double* C) {
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        FLB_UNROLL
        for (int j = 0; j < 3; ++j)
            C[3 * i + j] = A[3 * i + 0] * B[0 + j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
    }
}
FLB_HD void m3_T(const double* A, double* T) {
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        FLB_UNROLL
        for (int j = 0; j < 3; ++j) T[3 * i + j] = A[3 * j + i];
    }
}
FLB_HD void m3_vec(const double* A, const double* v, double* o) {
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) o[i] = A[3 * i + 0] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
// SKEW_SYM_MATRX, include/so3_math.h:9
FLB_HD void skew3(const double* v, double* K) {
    K[0] = 0.0;   K[1] = -v[2]; K[2] = v[1];
    K[3] = v[2];  K[4] = 0.0;   K[5] = -v[0];
    K[6] = -v[1]; K[7] = v[0];  K[8] = 0.0;
}
FLB_HD double norm3(const double* v) { return sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

// include/so3_math.h:54-72  Exp(v1, v2, v3)
FLB_HD void so3_exp(const double* v, double* R) {
    const double nrm = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (nrm > 0.00001) {
        const double r[3] = {v[0] / nrm, v[1] / nrm, v[2] / nrm};
        double K[9], KK[9];
        skew3(r, K);
        m3_mul(K, K, KK);
        const double s = sin(nrm), c1 = 1.0 - cos(nrm);
        FLB_UNROLL
        for (int i = 0; i < 9; ++i) R[i] = R[i] + s * K[i] + c1 * KK[i];
    }
}

// include/so3_math.h:75-81  Log(R)
FLB_HD void so3_log(const double* R, double* out) {
    const double tr = R[0] + R[4] + R[8];
    const double theta = (tr > 3.0 - 1e-6) ? 0.0 : acos(0.5 * (tr - 1));
    const double K[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    if (fabs(theta) < 0.001) {
        FLB_UNROLL
        for (int i = 0; i < 3; ++i) out[i] = 0.5 * K[i];
    } else {
        const double f = 0.5 * theta / sin(theta);
        FLB_UNROLL
        for (int i = 0; i < 3; ++i) out[i] = f * K[i];
    }
}

// ------------------------------------------------------------------ plane fit
// esti_plane<float>, include/common_lib.h:448-493: least squares A(5x3) x = -1 by
// column-pivoted Householder QR in float32, then normalise and test the 5 points.
// Operation order is the oracle's (oracle/flo_oracle.cpp: flo_esti_plane); with
// -fmad=false this is bit-exact against it.  All array indices are compile-time
// after unrolling so qr[][] lives in registers.
FLB_HD bool plane_fit5(const float (&nb)[kMatch][3], float threshold, float (&pabcd)[4]) {
    constexpr int rows = kMatch, cols = 3;
    float qr[rows][cols];
    FLB_UNROLL
    for (int j = 0; j < rows; ++j) {
        FLB_UNROLL
        for (int c = 0; c < cols; ++c) qr[j][c] = nb[j][c];
    }
    float hcoef[cols];
    int colidx[cols] = {0, 1, 2};
    float nrmU[cols], nrmD[cols];
    FLB_UNROLL
    for (int c = 0; c < cols; ++c) {
        float s = 0.f;
        FLB_UNROLL
        for (int j = 0; j < rows; ++j) s = s + qr[j][c] * qr[j][c];
        nrmD[c] = nrmU[c] = sqrtf(s);
    }
    const float eps = 1.1920928955078125e-07f;  // FLT_EPSILON
    float maxnorm = nrmU[0];
    FLB_UNROLL
    for (int c = 1; c < cols; ++c)
        if (nrmU[c] > maxnorm) maxnorm = nrmU[c];
    const float th0 = maxnorm * eps;
    const float threshold_helper = (th0 * th0) / float(rows);
    const float downdate_thr = sqrtf(eps);
    int nonzero_pivots = cols;
    FLB_UNROLL
    for (int k = 0; k < cols; ++k) {
        int big = k;
        float bigv = nrmU[k];
        FLB_UNROLL
        for (int c = k + 1; c < cols; ++c)
            if (nrmU[c] > bigv) { bigv = nrmU[c]; big = c; }
        const float big_sq = bigv * bigv;
        if (nonzero_pivots == cols && big_sq < threshold_helper * float(rows - k)) nonzero_pivots = k;
        FLB_UNROLL
        for (int c = k + 1; c < cols; ++c) {
            if (c == big) {
                FLB_UNROLL
                for (int j = 0; j < rows; ++j) { const float t = qr[j][k]; qr[j][k] = qr[j][c]; qr[j][c] = t; }
                float t = nrmU[k]; nrmU[k] = nrmU[c]; nrmU[c] = t;
                t = nrmD[k]; nrmD[k] = nrmD[c]; nrmD[c] = t;
                const int ti = colidx[k]; colidx[k] = colidx[c]; colidx[c] = ti;
            }
        }
        float tailSq = 0.f;
        FLB_UNROLL
        for (int j = k + 1; j < rows; ++j) tailSq = tailSq + qr[j][k] * qr[j][k];
        const float c0 = qr[k][k];
        float beta, tau;
        if (tailSq <= 1.17549435082228750797e-38f) {  // FLT_MIN
            tau = 0.f;
            beta = c0;
            FLB_UNROLL
            for (int j = k + 1; j < rows; ++j) qr[j][k] = 0.f;
        } else {
            beta = sqrtf(c0 * c0 + tailSq);
            if (c0 >= 0.f) beta = -beta;
            const float den = c0 - beta;
            FLB_UNROLL
            for (int j = k + 1; j < rows; ++j) qr[j][k] = qr[j][k] / den;
            tau = (beta - c0) / beta;
        }
        qr[k][k] = beta;
        hcoef[k] = tau;
        if (tau != 0.f) {
            FLB_UNROLL
            for (int c = k + 1; c < cols; ++c) {
                float tmp = 0.f;
                FLB_UNROLL
                for (int j = k + 1; j < rows; ++j) tmp = tmp + qr[j][k] * qr[j][c];
                tmp = tmp + qr[k][c];
                qr[k][c] = qr[k][c] - tau * tmp;
                FLB_UNROLL
                for (int j = k + 1; j < rows; ++j) qr[j][c] = qr[j][c] - (tau * qr[j][k]) * tmp;
            }
        }
        FLB_UNROLL
        for (int c = k + 1; c < cols; ++c) {
            if (nrmU[c] != 0.f) {
                float temp = fabsf(qr[k][c]) / nrmU[c];
                temp = (1.f + temp) * (1.f - temp);
                temp = temp < 0.f ? 0.f : temp;
                const float ratio = nrmU[c] / nrmD[c];
                const float temp2 = temp * (ratio * ratio);
                if (temp2 <= downdate_thr) {
                    float s = 0.f;
                    FLB_UNROLL
                    for (int j = k + 1; j < rows; ++j) s = s + qr[j][c] * qr[j][c];
                    nrmD[c] = sqrtf(s);
                    nrmU[c] = nrmD[c];
                } else {
                    nrmU[c] = nrmU[c] * sqrtf(temp);
                }
            }
        }
    }
    float cv[rows];
    FLB_UNROLL
    for (int j = 0; j < rows; ++j) cv[j] = -1.0f;
    float x[3] = {0.f, 0.f, 0.f};
    FLB_UNROLL
    for (int k = 0; k < cols; ++k) {
        if (k < nonzero_pivots) {
            const float tau = hcoef[k];
            if (tau != 0.f) {
                float tmp = 0.f;
                FLB_UNROLL
                for (int j = k + 1; j < rows; ++j) tmp = tmp + qr[j][k] * cv[j];
                tmp = tmp + cv[k];
                cv[k] = cv[k] - tau * tmp;
                FLB_UNROLL
                for (int j = k + 1; j < rows; ++j) cv[j] = cv[j] - (tau * qr[j][k]) * tmp;
            }
        }
    }
    FLB_UNROLL
    for (int i = cols - 1; i >= 0; --i) {
        if (i < nonzero_pivots) {
            cv[i] = cv[i] / qr[i][i];
            FLB_UNROLL
            for (int r = 0; r < i; ++r) cv[r] = cv[r] - cv[i] * qr[r][i];
        }
    }
    FLB_UNROLL
    for (int i = 0; i < cols; ++i) {
        if (i < nonzero_pivots) {
            FLB_UNROLL
            for (int c = 0; c < cols; ++c)
                if (colidx[i] == c) x[c] = cv[i];
        }
    }
    const float n = sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    pabcd[0] = x[0] / n;
    pabcd[1] = x[1] / n;
    pabcd[2] = x[2] / n;
    pabcd[3] = (float)(1.0 / (double)n);
    bool ok = true;
    FLB_UNROLL
    for (int j = 0; j < rows; ++j) {
        const float v = pabcd[0] * nb[j][0] + pabcd[1] * nb[j][1] + pabcd[2] * nb[j][2] + pabcd[3];
        if (!(fabsf(v) <= threshold)) ok = false;
    }
    return ok;
}

// ------------------------------------------------------------------ LIO per-point
// Per-pass constants (uniform over the scan): pose, extrinsic and their transposes.
struct LioPose {
    double R[9], p[3];       // state.rot_end / pos_end
    double R_LI[9], t_LI[3]; // Lidar_rot_to_IMU / Lidar_offset_to_IMU
    double Rt[9], RLIt[9];   // transposes
};

// pointBodyToWorld, src/laserMapping.cpp:272-286: double math, float store.
FLB_HD void lio_body_to_world(const LioPose& c, const float* pb, double* pI, float* pw) {
    const double b[3] = {(double)pb[0], (double)pb[1], (double)pb[2]};
    m3_vec(c.R_LI, b, pI);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) pI[k] = pI[k] + c.t_LI[k];
    double w[3];
    m3_vec(c.R, pI, w);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) pw[k] = (float)(w[k] + c.p[k]);
}

// Residual + gate, src/laserMapping.cpp:1573-1576.  Returns s > 0.9.
FLB_HD bool lio_residual(const float* pabcd, const float* pw, const float* pb, float* pd2_out) {
    const float pd2 = pabcd[0] * pw[0] + pabcd[1] * pw[1] + pabcd[2] * pw[2] + pabcd[3];
    const double b[3] = {(double)pb[0], (double)pb[1], (double)pb[2]};
    const float s = (float)(1 - 0.9 * (double)fabsf(pd2) / sqrt(norm3(b)));
    *pd2_out = pd2;
    return (double)s > 0.9;
}

// The per-point byte a LIO pass leaves: bit 0 = point_selected_surf after the pass (:1570-1584), bit 1 = the point is a
// row of the pass (point_selected_surf[i] && res_last[i] <= 2.0, :1593), i.e. a member of laserCloudOri.  Bit 1 implies
// bit 0, so `byte != 0` still reads point_selected_surf.  The row test is not implied by s > 0.9: that gate admits
// |pd2| > 2 for points beyond 324 m (|pd2| < sqrt(|p_body|) / 9).
constexpr unsigned char kLioSel = 1, kLioRow = 3;
FLB_HD unsigned char lio_sel_byte(bool sel, float pd2) {
    return sel ? (((double)fabsf(pd2) <= 2.0) ? kLioRow : kLioSel) : (unsigned char)0;
}
FLB_HD bool lio_sel_is_row(unsigned char b) { return b == kLioRow; }

// Live-layout row [A, n], A = [p_I]x * R^T * n   (src/laserMapping.cpp:1611-1625)
FLB_HD void lio_row6(const LioPose& c, const double* pI, const float* pabcd, double* row) {
    double cross[9], M1[9], A[3];
    skew3(pI, cross);
    const double nv[3] = {(double)pabcd[0], (double)pabcd[1], (double)pabcd[2]};
    m3_mul(cross, c.Rt, M1);
    m3_vec(M1, nv, A);
    row[0] = A[0]; row[1] = A[1]; row[2] = A[2];
    row[3] = nv[0]; row[4] = nv[1]; row[5] = nv[2];
}

// IKFoM-layout row [n, A, B, C]  (src/laserMapping.cpp:1063-1082):
//   C = R^T n, A = [p_I]x C, B = [p_b]x R_LI^T C
FLB_HD void lio_row12(const LioPose& c, const double* pI, const float* pb, const float* pabcd, double* row) {
    const double nv[3] = {(double)pabcd[0], (double)pabcd[1], (double)pabcd[2]};
    const double b[3] = {(double)pb[0], (double)pb[1], (double)pb[2]};
    double C[3], A[3], B[3], cross[9], crossb[9], M2[9];
    m3_vec(c.Rt, nv, C);
    skew3(pI, cross);
    m3_vec(cross, C, A);
    skew3(b, crossb);
    m3_mul(crossb, c.RLIt, M2);
    m3_vec(M2, C, B);
    row[0] = nv[0]; row[1] = nv[1]; row[2] = nv[2];
    row[3] = A[0];  row[4] = A[1];  row[5] = A[2];
    row[6] = B[0];  row[7] = B[1];  row[8] = B[2];
    row[9] = C[0];  row[10] = C[1]; row[11] = C[2];
}

// ------------------------------------------------------------------ kNN over the uniform grid
// Two cell indexes over the same sorted point array (points ordered by cell, x fastest, then by insertion):
//  dense:  cell_start[(z*ny + y)*nx + x] = first point of the cell, one entry per cell of the grid box;
//  sparse: an open-addressing hash table of the OCCUPIED cells only, entries {key, start, end} (SparseCell), with the
//          cell key packing (z, y, x) + 2^20 in 21 bits each, x lowest, so that key order is dense cell-id order.
// Sparse mode keeps the GridDesc layout: nx holds the table's slot mask, ny / nz are unused, and the cell-table pointer
// points at the SparseCell array.
struct GridDesc {
    float ox, oy, oz;     // origin (min corner)
    float cell, inv_cell;
    int nx, ny, nz;       // cells per axis; cell id = (z*ny + y)*nx + x  (x fastest); sparse: nx = slot mask
    float max_d2;         // 5.0
    int max_ring;         // ceil(sqrt(max_d2)/cell) + 1
};

constexpr int kCellKeyBias = 1 << 20;                     // cells more than 2^20 from the origin have no key
constexpr unsigned long long kNoCell = ~0ull;             // empty hash slot; sorts behind every real key

struct alignas(16) SparseCell {
    unsigned long long key;
    int start, end;                                       // [start, end) in the sorted point array
};

FLB_HD bool cell_key_ok(int c) { return c >= -kCellKeyBias && c < kCellKeyBias; }
FLB_HD unsigned long long cell_key(int cx, int cy, int cz) {
    return ((unsigned long long)(cz + kCellKeyBias) << 42) | ((unsigned long long)(cy + kCellKeyBias) << 21) |
           (unsigned long long)(cx + kCellKeyBias);
}
FLB_HD unsigned cell_hash(unsigned long long key) { return (unsigned)((key * 0x9E3779B97F4A7C15ull) >> 32); }

// [start, end) of one cell (0, 0 when empty or out of key range); linear probing from the hashed slot
FLB_HD void sparse_find(const SparseCell* __restrict__ table, unsigned mask, int cx, int cy, int cz, int& s, int& e) {
    s = e = 0;
    if (!(cell_key_ok(cx) && cell_key_ok(cy) && cell_key_ok(cz))) return;
    const unsigned long long key = cell_key(cx, cy, cz);
    for (unsigned h = cell_hash(key) & mask;; h = (h + 1) & mask) {
#if defined(__CUDA_ARCH__)
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(table + h));
        const unsigned long long k = ((unsigned long long)v.y << 32) | v.x;
        if (k == key) { s = (int)v.z; e = (int)v.w; return; }
#else
        const SparseCell v = table[h];
        const unsigned long long k = v.key;
        if (k == key) { s = v.start; e = v.end; return; }
#endif
        if (k == kNoCell) return;
    }
}

struct Top5 {
    float d[kMatch];
    int i[kMatch];
};

FLB_HD void top5_init(Top5& t) {
    FLB_UNROLL
    for (int j = 0; j < kMatch; ++j) { t.d[j] = INFINITY; t.i[j] = -1; }
}

// Strict-< insertion (first visited wins a tie: ikd_Tree.cpp:860), ascending order.
FLB_HD void top5_insert(Top5& t, float d, int id) {
    if (d < t.d[4]) {
        if (d < t.d[3]) {
            t.d[4] = t.d[3]; t.i[4] = t.i[3];
            if (d < t.d[2]) {
                t.d[3] = t.d[2]; t.i[3] = t.i[2];
                if (d < t.d[1]) {
                    t.d[2] = t.d[1]; t.i[2] = t.i[1];
                    if (d < t.d[0]) {
                        t.d[1] = t.d[0]; t.i[1] = t.i[0];
                        t.d[0] = d; t.i[0] = id;
                    } else { t.d[1] = d; t.i[1] = id; }
                } else { t.d[2] = d; t.i[2] = id; }
            } else { t.d[3] = d; t.i[3] = id; }
        } else { t.d[4] = d; t.i[4] = id; }
    }
}

// calc_dist, include/ikd-Tree/ikd_Tree.cpp:1291-1295: (dx*dx + dy*dy) + dz*dz in float32.
FLB_HD float dist2f(float ax, float ay, float az, float bx, float by, float bz) {
    const float dx = ax - bx, dy = ay - by, dz = az - bz;
    return dx * dx + dy * dy + dz * dz;
}

#if defined(__CUDACC__)
typedef float4 map_pt;
#else
struct map_pt { float x, y, z, w; };
#endif
#if defined(__CUDA_ARCH__)
#define FLB_LDG4(ptr) __ldg(ptr)
#define FLB_LDGI(ptr) __ldg(ptr)
#else
#define FLB_LDG4(ptr) (*(ptr))
#define FLB_LDGI(ptr) (*(ptr))
#endif

// ------------------------------------------------------------------ map_incremental from the uploaded scan
// map_incremental (src/laserMapping.cpp:692-706), one point: the ordered scan entry `b` (body xyz, the caller's index in
// w) -> pointBodyToWorld of it (:272-286) in pw.  Returns the caller's index, where the world point goes.
FLB_HD int map_scan_point(const LioPose& c, const map_pt& b, float* pw) {
    const float pb[3] = {b.x, b.y, b.z};
    double pI[3];
    lio_body_to_world(c, pb, pI, pw);
    return (int)float_as_u32(b.w);
}

// publish_effect_world's capture (flb_effect_cloud), one point of the ordered scan: its row flag (lio_sel_byte) and its
// body point go to its caller's index (w), so that an order-preserving select over the flags yields laserCloudOri in
// scan-index order (src/laserMapping.cpp:1588-1600).
FLB_HD void effect_scatter_point(const map_pt& b, unsigned char sel_byte, unsigned char* flag, map_pt* body) {
    const int oi = (int)float_as_u32(b.w);
    flag[oi] = lio_sel_is_row(sel_byte) ? 1 : 0;
    body[oi] = b;
}

// Whether all three floats are finite (exponent field not all ones), as flb_map_add_points tests its input.
FLB_HD bool finite3(const float* v) {
    return ((float_as_u32(v[0]) & 0x7F800000u) != 0x7F800000u) && ((float_as_u32(v[1]) & 0x7F800000u) != 0x7F800000u) &&
           ((float_as_u32(v[2]) & 0x7F800000u) != 0x7F800000u);
}

// Bounds record of the new points: an unsigned key that orders like the float, so that an atomic maximum on a zeroed
// word yields the maximum (of key) and the minimum (of ~key).  -0.0 orders below +0.0; nothing downstream of the bounds
// tells the two apart.
enum { kScanRecMax = 0, kScanRecMin = 3, kScanRecBad = 6, kScanRecWords = 8 };
FLB_HD unsigned f32_order_key(float f) {
    const unsigned b = float_as_u32(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
FLB_HD float f32_from_order_key(unsigned k) { return u32_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// ------------------------------------------------------------------ local-map cube (lasermap_fov_segment)
// Box q = {min xyz, max xyz} contains p: the half-open test of Delete_by_range (ikd_Tree.cpp:650), min <= p < max.
FLB_HD bool box_contains(const float* q, float x, float y, float z) {
    return q[0] <= x && q[3] > x && q[1] <= y && q[4] > y && q[2] <= z && q[5] > z;
}

constexpr int kFovMaxBoxes = 3;   // at most one slab per axis (:398-411)
// LocalMap_Points (BoxPointType: float vertices) and Localmap_Initialized (src/laserMapping.cpp:361-362)
struct FovCube {
    float vmin[3], vmax[3];
    int initialized, pad;
};
// One call of lasermap_fov_segment: the cube it leaves, cub_needrm (n_boxes of them, {min xyz, max xyz}; the unused
// slots are the empty box, all zeros), and the number of map points inside them (the flagging kernel adds it up).
struct FovRecord {
    FovCube cube;
    int n_boxes, n_deleted;
    float boxes[6 * kFovMaxBoxes];
};

// lasermap_fov_segment (src/laserMapping.cpp:363-412) up to Delete_Point_Boxes, op for op with the reference's types:
// pos_LiD double, the cube's vertices float, dist_to_map_edge float of fabs(double - float), the threshold the float
// product MOV_THRESHOLD * DET_RANGE, mov_dist a double max stored as float.  `in` is the cube before the call.
FLB_HD void fov_segment_step(const FovCube& in, const double* pos, double cube_len, float det_range, float mov_threshold,
                             FovRecord& out) {
    out.cube = in;
    out.n_boxes = 0;
    out.n_deleted = 0;
    for (int k = 0; k < 6 * kFovMaxBoxes; ++k) out.boxes[k] = 0.0f;
    if (!in.initialized) {                                                     // :376-384
        for (int i = 0; i < 3; ++i) {
            out.cube.vmin[i] = (float)(pos[i] - cube_len / 2.0);
            out.cube.vmax[i] = (float)(pos[i] + cube_len / 2.0);
        }
        out.cube.initialized = 1;
        return;
    }
    const float thr = mov_threshold * det_range;
    float dist[3][2];
    bool need_move = false;
    for (int i = 0; i < 3; ++i) {                                              // :386-391
        dist[i][0] = (float)fabs(pos[i] - (double)in.vmin[i]);
        dist[i][1] = (float)fabs(pos[i] - (double)in.vmax[i]);
        if (dist[i][0] <= thr || dist[i][1] <= thr) need_move = true;
    }
    if (!need_move) return;
    const double a = (cube_len - 2.0 * (double)mov_threshold * (double)det_range) * 0.5 * 0.9;   // :396
    const double b = (double)(det_range * (mov_threshold - 1));
    const float mov_dist = (float)(a < b ? b : a);                             // std::max: the first unless it is less
    for (int i = 0; i < 3; ++i) {                                              // :397-411
        float tmp[6] = {in.vmin[0], in.vmin[1], in.vmin[2], in.vmax[0], in.vmax[1], in.vmax[2]};
        if (dist[i][0] <= thr) {
            out.cube.vmax[i] -= mov_dist;
            out.cube.vmin[i] -= mov_dist;
            tmp[i] = in.vmax[i] - mov_dist;
        } else if (dist[i][1] <= thr) {
            out.cube.vmax[i] += mov_dist;
            out.cube.vmin[i] += mov_dist;
            tmp[3 + i] = in.vmin[i] + mov_dist;
        } else {
            continue;
        }
        for (int k = 0; k < 6; ++k) out.boxes[6 * out.n_boxes + k] = tmp[k];
        ++out.n_boxes;
    }
}

// Row bounds, the one reader of a cell index: the points of cells [xa, xb] of row (z, y) are one contiguous run of the
// sorted array; returns its [start, end).  Dense: two table reads (the caller clips to the grid).  Sparse: start of the
// first occupied cell, end of the last; (0, 0) when none is occupied.
template <bool SPARSE>
FLB_HD void grid_row(const GridDesc& g, const int* __restrict__ cells, int z, int y, int xa, int xb, int& s, int& e) {
    if constexpr (!SPARSE) {
        const int rowbase = (z * g.ny + y) * g.nx;
        s = FLB_LDGI(cells + rowbase + xa);
        e = FLB_LDGI(cells + rowbase + xb + 1);
    } else {
        const SparseCell* table = reinterpret_cast<const SparseCell*>(cells);
        int x = xa, e0 = 0;
        s = 0;
        for (; x <= xb; ++x) {
            sparse_find(table, (unsigned)g.nx, x, y, z, s, e0);
            if (e0 > s) break;
        }
        e = e0;
        for (int x1 = xb; x1 > x; --x1) {
            int s1, e1;
            sparse_find(table, (unsigned)g.nx, x1, y, z, s1, e1);
            if (e1 > s1) { e = e1; break; }
        }
    }
}

// Walk `nruns` (<= 9) runs of sorted map points whose [start, end) bounds sit in the per-thread scratch (start of run k
// at rows[k * rstride], end at rows[(9 + k) * rstride]) as ONE candidate sequence, up to four points (independent 16-B
// loads) per step, in run order then index order.  A lane's trip count is its own candidate count / 4, so lanes whose
// non-empty runs differ do not wait on each other run by run.  The walk is one memory round trip per step (the insert
// needs the loaded points), so the loads of step s + 1 are issued BEFORE step s is consumed: two steps in flight.
struct KnnCursor {
    int k, m, e;
};
// next group of <= 4 consecutive candidates: returns their count (0: the sequence is exhausted) and the first index
FLB_HD int knn_cursor_next(KnnCursor& c, const int* rows, int rstride, int nruns, int& first) {
    while (c.m >= c.e) {
        if (++c.k >= nruns) return 0;
        c.m = rows[c.k * rstride];
        c.e = rows[(9 + c.k) * rstride];
    }
    const int left = c.e - c.m;
    const int n = left > 4 ? 4 : left;
    first = c.m;
    c.m += n;
    return n;
}
FLB_HD void knn_walk_runs(const map_pt* __restrict__ pts, const int* rows, int rstride, int nruns, float qx, float qy, float qz,
                          Top5& t) {
    KnnCursor c{-1, 0, 0};
    int m = 0;
    int n = knn_cursor_next(c, rows, rstride, nruns, m);
    if (n == 0) return;
    map_pt P0 = FLB_LDG4(pts + m);
    map_pt P1 = FLB_LDG4(pts + (n > 1 ? m + 1 : m));
    map_pt P2 = FLB_LDG4(pts + (n > 2 ? m + 2 : m));
    map_pt P3 = FLB_LDG4(pts + (n > 3 ? m + 3 : m));
    for (;;) {
        int m1 = m;
        const int n1 = knn_cursor_next(c, rows, rstride, nruns, m1);
        // (n1 == 0: harmless re-load of the current group's first point)
        const map_pt Q0 = FLB_LDG4(pts + m1);
        const map_pt Q1 = FLB_LDG4(pts + (n1 > 1 ? m1 + 1 : m1));
        const map_pt Q2 = FLB_LDG4(pts + (n1 > 2 ? m1 + 2 : m1));
        const map_pt Q3 = FLB_LDG4(pts + (n1 > 3 ? m1 + 3 : m1));
        top5_insert(t, dist2f(qx, qy, qz, P0.x, P0.y, P0.z), m);
        if (n > 1) top5_insert(t, dist2f(qx, qy, qz, P1.x, P1.y, P1.z), m + 1);
        if (n > 2) top5_insert(t, dist2f(qx, qy, qz, P2.x, P2.y, P2.z), m + 2);
        if (n > 3) top5_insert(t, dist2f(qx, qy, qz, P3.x, P3.y, P3.z), m + 3);
        if (n1 == 0) break;
        P0 = Q0; P1 = Q1; P2 = Q2; P3 = Q3;
        m = m1;
        n = n1;
    }
}

// Exact 5-NN restricted to d2 <= max_d2, by ring expansion over the sorted uniform grid.
// After all cells within Chebyshev radius r of the query's cell are scanned, every
// unscanned point is at least (r*cell + margin) away, margin = distance from the query
// to the nearest face of its own cell.  Terminate when the 5th best is inside that
// bound (minus a float slack that also covers points binned across a face by
// rounding), or when the bound passes sqrt(max_d2).  Returns sorted positions in t.i.
//
// Every ring is walked as x-runs of cells whose cell-table bounds are fetched nine runs at a time (18 independent
// loads: one memory round trip per batch instead of one per run): rings 0 and 1 (the 3x3x3 block, where a query next to
// a surface ends) are nine 3-cell rows; the shell of ring r >= 2 is (2r+1)-cell rows on its z / y faces and single cells
// at x = cx -+ r elsewhere.  (A query displaced from the surfaces by the prior's error -- the first pass of a frame --
// needs ring 2 or 3: round 1 walked those shells one run and one dependent round trip at a time.)
//
// SPARSE: `cells` is the SparseCell hash table (see GridDesc).  There is no grid box, so nothing is clipped and there is
// no early exit outside it; rings 0+1 are 27 independent cell probes (a row's run = first to last occupied cell), the
// shells r >= 2 probe cell by cell.  Runs, their order and the termination bounds are the dense ones, so on a shared
// cell geometry both indexes return bit-identical results.
template <bool SPARSE = false>
FLB_HD void knn5_grid(const GridDesc& g, const int* __restrict__ cell_start, const map_pt* __restrict__ pts,
                      float qx, float qy, float qz, Top5& t, int* rows, int rstride) {
    // rows: per-thread scratch for 18 ints, element k at rows[k * rstride] (shared memory on the device,
    // one column per thread, so a warp's accesses are conflict-free)
    top5_init(t);
    const float fx = (qx - g.ox) * g.inv_cell, fy = (qy - g.oy) * g.inv_cell, fz = (qz - g.oz) * g.inv_cell;
    if constexpr (SPARSE) {
        // beyond the key range (+ the rings): no cell there has a key
        const float lim = (float)(kCellKeyBias + g.max_ring + 2);
        if (!(fx > -lim && fy > -lim && fz > -lim && fx < lim && fy < lim && fz < lim)) return;
    } else {
        // far outside the grid: nothing within sqrt(max_d2)
        const float lim = (float)(g.max_ring + 2);
        if (!(fx > -lim && fy > -lim && fz > -lim && fx < (float)g.nx + lim && fy < (float)g.ny + lim &&
              fz < (float)g.nz + lim))
            return;
    }
    const int cx = (int)floorf(fx), cy = (int)floorf(fy), cz = (int)floorf(fz);
    float mx = fminf(fx - (float)cx, (float)(cx + 1) - fx);
    float my = fminf(fy - (float)cy, (float)(cy + 1) - fy);
    float mz = fminf(fz - (float)cz, (float)(cz + 1) - fz);
    const float margin = fmaxf(fminf(mx, fminf(my, mz)) * g.cell - 1e-3f * g.cell, 0.f);
    {
        if constexpr (SPARSE) {
            // rings 0+1: 27 independent probes, then each row's run from its first to its last occupied cell
            const SparseCell* table = reinterpret_cast<const SparseCell*>(cell_start);
            int cs[27], ce[27];
            FLB_UNROLL
            for (int k = 0; k < 27; ++k)
                sparse_find(table, (unsigned)g.nx, cx + k % 3 - 1, cy + (k / 3) % 3 - 1, cz + k / 9 - 1, cs[k], ce[k]);
            FLB_UNROLL
            for (int k = 0; k < 9; ++k) {
                const int* s3 = cs + 3 * k;
                const int* e3 = ce + 3 * k;
                rows[k * rstride] = e3[0] > s3[0] ? s3[0] : (e3[1] > s3[1] ? s3[1] : s3[2]);
                rows[(9 + k) * rstride] = e3[2] > s3[2] ? e3[2] : (e3[1] > s3[1] ? e3[1] : e3[0]);
            }
        } else {
            // rings 0+1: rows (dz, dy) in {-1,0,1}^2, x-range [cx-1, cx+1] clipped to the grid
            const int xa = cx - 1 < 0 ? 0 : cx - 1, xb = cx + 1 >= g.nx ? g.nx - 1 : cx + 1;
            FLB_UNROLL
            for (int k = 0; k < 9; ++k) {
                const int z = cz + k / 3 - 1, y = cy + k % 3 - 1;
                const bool in = (z >= 0 && z < g.nz && y >= 0 && y < g.ny && xa <= xb);
                const int rowbase = in ? (z * g.ny + y) * g.nx : 0;
                rows[k * rstride] = in ? FLB_LDGI(cell_start + rowbase + xa) : 0;
                rows[(9 + k) * rstride] = in ? FLB_LDGI(cell_start + rowbase + xb + 1) : 0;
            }
        }
        knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t);
        const float bound = g.cell + margin;
        const float b2 = bound * bound;
        if (t.d[4] <= b2) return;                 // 5th best is certainly final
        if (b2 > g.max_d2 * 1.0001f) return;      // everything unscanned is beyond max_d2
    }
    for (int r = 2; r <= g.max_ring; ++r) {
        const int z0 = cz - r, z1 = cz + r, y0 = cy - r, y1 = cy + r, x0 = cx - r, x1 = cx + r;
        int cnt = 0;
        if constexpr (!SPARSE) {
            const int xa = x0 < 0 ? 0 : x0, xb = x1 >= g.nx ? g.nx - 1 : x1;
            for (int z = (z0 < 0 ? 0 : z0); z <= (z1 >= g.nz ? g.nz - 1 : z1); ++z) {
                const bool zface = (z == z0) || (z == z1);
                for (int y = (y0 < 0 ? 0 : y0); y <= (y1 >= g.ny ? g.ny - 1 : y1); ++y) {
                    const int rowbase = (z * g.ny + y) * g.nx;
                    if (zface || y == y0 || y == y1) {
                        if (xa <= xb) {
                            rows[cnt * rstride] = FLB_LDGI(cell_start + rowbase + xa);
                            rows[(9 + cnt) * rstride] = FLB_LDGI(cell_start + rowbase + xb + 1);
                            if (++cnt == 9) { knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t); cnt = 0; }
                        }
                    } else {
                        if (x0 >= 0 && x0 < g.nx) {
                            rows[cnt * rstride] = FLB_LDGI(cell_start + rowbase + x0);
                            rows[(9 + cnt) * rstride] = FLB_LDGI(cell_start + rowbase + x0 + 1);
                            if (++cnt == 9) { knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t); cnt = 0; }
                        }
                        if (x1 >= 0 && x1 < g.nx) {
                            rows[cnt * rstride] = FLB_LDGI(cell_start + rowbase + x1);
                            rows[(9 + cnt) * rstride] = FLB_LDGI(cell_start + rowbase + x1 + 1);
                            if (++cnt == 9) { knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t); cnt = 0; }
                        }
                    }
                }
            }
        } else {
            // unclipped: z / y faces are (2r+1)-cell rows, elsewhere the cells x0 and x1; empty runs are not queued
            for (int z = z0; z <= z1; ++z) {
                const bool zface = (z == z0) || (z == z1);
                for (int y = y0; y <= y1; ++y) {
                    const bool full = zface || y == y0 || y == y1;
                    for (int part = 0; part < (full ? 1 : 2); ++part) {
                        int s, e;
                        if (full) grid_row<true>(g, cell_start, z, y, x0, x1, s, e);
                        else grid_row<true>(g, cell_start, z, y, part ? x1 : x0, part ? x1 : x0, s, e);
                        if (e > s) {
                            rows[cnt * rstride] = s;
                            rows[(9 + cnt) * rstride] = e;
                            if (++cnt == 9) { knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t); cnt = 0; }
                        }
                    }
                }
            }
        }
        if (cnt) knn_walk_runs(pts, rows, rstride, cnt, qx, qy, qz, t);
        const float bound = (float)r * g.cell + margin;
        const float b2 = bound * bound;
        if (t.d[4] <= b2) break;             // 5th best is certainly final
        if (b2 > g.max_d2 * 1.0001f) break;  // everything unscanned is beyond max_d2
    }
}

// ------------------------------------------------------------------ VIO per-patch / per-pixel
struct CamModel {
    int width, height;
    double fx, fy, cx, cy;   // projection (world2cam)
    double d[5];
    double jfx, jfy;         // dpi's fx, fy: |fx|, |4 fx fy| / (4 |fx|)  (src/lidar_selection.cpp:58-59)
};

// Per-pass constants of UpdateState, src/lidar_selection.cpp:776-782 + init() :41-52.
struct VioPose {
    double Rcw[9], Pcw[3];   // :780-781
    double Jdp_dt[9];        // :782  (= Rci * Rwi^T)
    double Jdphi_dR[9];      // = Rci
    double Jdp_dR[9];        // = -Rci * [Pic]x
};

// State-independent part (LidarSelector::init(), src/lidar_selection.cpp:44-52): Jdphi_dR = Rci,
// Jdp_dR = -Rci * [Pic]x with Pic = -Rci^T * Pci.  Computed once per update on the host.
FLB_HD void vio_pose_constants(const double* Rci, const double* Pci, double* Jdphi_dR, double* Jdp_dR) {
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) Jdphi_dR[i] = Rci[i];
    double RciT[9], Pic[3], sk[9], m[9];
    m3_T(Rci, RciT);
    m3_vec(RciT, Pci, Pic);
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) Pic[i] = -Pic[i];
    skew3(Pic, sk);
    m3_mul(Rci, sk, m);
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) Jdp_dR[i] = -m[i];
}

// State-dependent part, once per pass (src/lidar_selection.cpp:780-782).
FLB_HD void vio_make_pose(const double* Rci, const double* Pci, const double* Jdphi_dR, const double* Jdp_dR, const double* R,
                          const double* p, VioPose& o) {
    double Rt[9], t[3];
    m3_T(R, Rt);
    m3_mul(Rci, Rt, o.Rcw);
    m3_vec(o.Rcw, p, t);
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) o.Pcw[i] = -t[i] + Pci[i];
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) { o.Jdp_dt[i] = o.Rcw[i]; o.Jdphi_dR[i] = Jdphi_dR[i]; o.Jdp_dR[i] = Jdp_dR[i]; }
}

// vikit PinholeCamera::world2cam(Vector3d) (SURVEY.md Appendix C).
FLB_HD void world2cam(const CamModel& cam, const double* pf, double* px) {
    const double x = pf[0] / pf[2], y = pf[1] / pf[2];
    if (!(fabs(cam.d[0]) > 0.0000001)) {
        px[0] = cam.fx * x + cam.cx;
        px[1] = cam.fy * y + cam.cy;
    } else {
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
        const double cdist = 1 + cam.d[0] * r2 + cam.d[1] * r4 + cam.d[4] * r6;
        const double xd = x * cdist + cam.d[2] * a1 + cam.d[3] * a2;
        const double yd = y * cdist + cam.d[2] * a3 + cam.d[3] * a1;
        px[0] = xd * cam.fx + cam.cx;
        px[1] = yd * cam.fy + cam.cy;
    }
}

// Patch-level quantities of src/lidar_selection.cpp:792-816.
struct PatchGeom {
    double Ja, Jb, Jc, Jd;   // the non-zero entries of dpi(pf) (:92-103): [Ja 0 Jb; 0 Jc Jd]
    double pf[3];            // p_hat = skew(pf) (:805) is expanded where it is used
    float w_tl, w_tr, w_bl, w_br;
    int u_i, v_i;        // integer anchor
    int scale;
    bool valid;          // in front of the camera and tap footprint inside the image (our guard, SURVEY §7 H5)
};

FLB_HD void vio_patch_geom(const CamModel& cam, const VioPose& vp, const double* pos, int level, int search_level,
                           PatchGeom& g) {
    const int scale = 1 << (level + search_level);
    g.scale = scale;
    g.valid = false;
    double pf[3];
    m3_vec(vp.Rcw, pos, pf);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) pf[k] = pf[k] + vp.Pcw[k];
    if (!(pf[2] > 0.0)) return;
    double pc[2];
    world2cam(cam, pf, pc);
    if (!(fabs(pc[0]) < 1e6) || !(fabs(pc[1]) < 1e6)) return;
    {
        const double x = pf[0], y = pf[1], z_inv = 1. / pf[2], z_inv_2 = z_inv * z_inv;
        g.Ja = cam.jfx * z_inv; g.Jb = -cam.jfx * x * z_inv_2;
        g.Jc = cam.jfy * z_inv; g.Jd = -cam.jfy * y * z_inv_2;
    }
    g.pf[0] = pf[0]; g.pf[1] = pf[1]; g.pf[2] = pf[2];
    const float u_ref = (float)pc[0];
    const float v_ref = (float)pc[1];
    const int u_i = (int)(floorf((float)(pc[0] / scale)) * (float)scale);   // :809
    const int v_i = (int)(floorf((float)(pc[1] / scale)) * (float)scale);
    if (u_i - 5 * scale < 0 || u_i + 5 * scale > cam.width - 1 || v_i - 5 * scale < 0 ||
        v_i + 5 * scale > cam.height - 1)
        return;
    const float su = (u_ref - (float)u_i) / (float)scale;
    const float sv = (v_ref - (float)v_i) / (float)scale;
    g.w_tl = (float)((1.0 - (double)su) * (1.0 - (double)sv));    // :813-816 (double expressions -> float)
    g.w_tr = (float)((double)su * (1.0 - (double)sv));
    g.w_bl = (float)((1.0 - (double)su) * (double)sv);
    g.w_br = su * sv;
    g.u_i = u_i;
    g.v_i = v_i;
    g.valid = true;
}

// One pixel of the 8x8 loop, src/lidar_selection.cpp:819-847.
// L is the patch's 11x11 tap lattice (stride `scale` pixels, centred on the anchor):
//   L[r][c] = img[(v_i + (r-5)*scale) * W + u_i + (c-5)*scale]  as float.
// Pixel (x = row, y = col) reads img_ptr[a*scale + b*scale*W] = L[x+1+b][y+1+a].
template <typename Lat>
FLB_HD void vio_pixel(const Lat& L, const PatchGeom& g, const VioPose& vp, int x, int y, float ref, double* row,
                      double* res_out) {
    const int r = x + 1, c = y + 1;
    const float wtl = g.w_tl, wtr = g.w_tr, wbl = g.w_bl, wbr = g.w_br;
    const float du = 0.5f * ((wtl * L(r, c + 1) + wtr * L(r, c + 2) + wbl * L(r + 1, c + 1) + wbr * L(r + 1, c + 2)) -
                             (wtl * L(r, c - 1) + wtr * L(r, c) + wbl * L(r + 1, c - 1) + wbr * L(r + 1, c)));
    const float dv = 0.5f * ((wtl * L(r + 1, c) + wtr * L(r + 1, c + 1) + wbl * L(r + 2, c) + wbr * L(r + 2, c + 1)) -
                             (wtl * L(r - 1, c) + wtr * L(r - 1, c + 1) + wbl * L(r, c) + wbr * L(r, c + 1)));
    const double inv_scale = (1.0 / g.scale);
    const double J0 = (double)du * inv_scale, J1 = (double)dv * inv_scale;
    // Jimg * Jdpi, Jimg * Jdpi * p_hat and -Jimg * Jdpi (:829-833) with the structural zeros of Jdpi and of
    // p_hat = [0 -z y; z 0 -x; -y x 0] dropped: x*0 + v == v, so only the sign of an exact zero can differ.
    double JJ[3], Jdphi[3], Jdp[3];
    JJ[0] = J0 * g.Ja;
    JJ[1] = J1 * g.Jc;
    JJ[2] = J0 * g.Jb + J1 * g.Jd;
    Jdphi[0] = JJ[1] * g.pf[2] + JJ[2] * (-g.pf[1]);
    Jdphi[1] = JJ[0] * (-g.pf[2]) + JJ[2] * g.pf[0];
    Jdphi[2] = JJ[0] * g.pf[1] + JJ[1] * (-g.pf[0]);
    Jdp[0] = (-J0) * g.Ja;
    Jdp[1] = (-J1) * g.Jc;
    Jdp[2] = (-J0) * g.Jb + (-J1) * g.Jd;
    FLB_UNROLL
    for (int k = 0; k < 3; ++k)
        row[k] = (Jdphi[0] * vp.Jdphi_dR[k] + Jdphi[1] * vp.Jdphi_dR[3 + k] + Jdphi[2] * vp.Jdphi_dR[6 + k]) +
                 (Jdp[0] * vp.Jdp_dR[k] + Jdp[1] * vp.Jdp_dR[3 + k] + Jdp[2] * vp.Jdp_dR[6 + k]);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k)
        row[3 + k] = Jdp[0] * vp.Jdp_dt[k] + Jdp[1] * vp.Jdp_dt[3 + k] + Jdp[2] * vp.Jdp_dt[6 + k];
    const float resf = wtl * L(r, c) + wtr * L(r, c + 1) + wbl * L(r + 1, c) + wbr * L(r + 1, c + 1) - ref;  // :837
    *res_out = (double)resf;
}

// ------------------------------------------------------------------ 18-DoF state algebra
struct State18 {
    double rot[9], pos[3], vel[3], bg[3], ba[3], grav[3];
    double cov[kDim * kDim];
};

// StatesGroup::operator+=, include/common_lib.h:343-352
FLB_HD void state_boxplus(State18& x, const double* d) {
    double E[9], Rn[9];
    so3_exp(d, E);
    m3_mul(x.rot, E, Rn);
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) x.rot[i] = Rn[i];
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        x.pos[i] += d[3 + i];
        x.vel[i] += d[6 + i];
        x.bg[i] += d[9 + i];
        x.ba[i] += d[12 + i];
        x.grav[i] += d[15 + i];
    }
}

// StatesGroup::operator- (a - b), include/common_lib.h:354-365
FLB_HD void state_boxminus(const State18& a, const State18& b, double* out) {
    double bT[9], rotd[9];
    m3_T(b.rot, bT);
    m3_mul(bT, a.rot, rotd);
    so3_log(rotd, out);
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        out[3 + i] = a.pos[i] - b.pos[i];
        out[6 + i] = a.vel[i] - b.vel[i];
        out[9 + i] = a.bg[i] - b.bg[i];
        out[12 + i] = a.ba[i] - b.ba[i];
        out[15 + i] = a.grav[i] - b.grav[i];
    }
}



// ------------------------------------------------------------------ IMU propagation / undistortion (row f3)
// Exp(ang_vel, dt), include/so3_math.h:30-51
FLB_HD void so3_exp_dt(const double* w, double dt, double* R) {
    const double nrm = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (nrm > 0.0000001) {
        const double r[3] = {w[0] / nrm, w[1] / nrm, w[2] / nrm};
        double K[9], KK[9];
        skew3(r, K);
        m3_mul(K, K, KK);
        const double ang = nrm * dt, s = sin(ang), c1 = 1.0 - cos(ang);
        FLB_UNROLL
        for (int i = 0; i < 9; ++i) R[i] = R[i] + s * K[i] + c1 * KK[i];
    }
}

// Pose6D (include/common_lib.h set_pose6d): one entry of IMUpose, src/IMU_Processing.cpp:658, :737
struct ImuPose {
    double t;            // offset_time relative to pcl_beg_time
    double acc[3], gyr[3], vel[3], pos[3], rot[9];
};

struct ImuParamsDev {
    double cov_gyr[3], cov_acc[3], cov_bias_gyr[3], cov_bias_acc[3];
    double G_m_s2, mean_acc_norm;
    double R_LI[9], t_LI[3];
};

// One point of the backward pass, src/IMU_Processing.cpp:792-805: compensate p (lidar frame, float) taken at
// time t (seconds after pcl_beg_time) to the frame end, given the IMU pose `head` that precedes it.
FLB_HD void imu_compensate_point(const ImuPose& head, const double* R_LI, const double* t_LI, const double* extR_Ri,
                                 const double* exrR_extT, const double* pos_end, double t, float* p) {
    const double dt = t - head.t;
    double E[9], R_i[9], T_ei[3], a[3], b[3], c[3];
    so3_exp_dt(head.gyr, dt, E);
    m3_mul(head.rot, E, R_i);                                                    // :796
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) T_ei[k] = head.pos[k] + head.vel[k] * dt + 0.5 * head.acc[k] * dt * dt - pos_end[k];   // :797
    const double P_i[3] = {(double)p[0], (double)p[1], (double)p[2]};
    m3_vec(R_LI, P_i, a);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) a[k] += t_LI[k];
    m3_vec(R_i, a, b);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) b[k] += T_ei[k];
    m3_vec(extR_Ri, b, c);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) p[k] = (float)(c[k] - exrR_extT[k]);              // :800-805
}

// ------------------------------------------------------------------ visual-map growth: candidate scoring (row f4)
// vk::shiTomasiScore (rpg_vikit vikit_common/src/vision.cpp): 8x8 box of central differences around (u, v), smaller
// eigenvalue of the normalised structure tensor.  Every partial sum is an integer < 2^24, exact in float.
FLB_HD float shi_tomasi_score(const unsigned char* img, int width, int height, int stride, int u, int v) {
    const int x_min = u - 4, x_max = u + 4, y_min = v - 4, y_max = v + 4;
    if (x_min < 1 || x_max >= width - 1 || y_min < 1 || y_max >= height - 1) return 0.0f;
    float dXX = 0.0f, dYY = 0.0f, dXY = 0.0f;
    for (int y = y_min; y < y_max; ++y) {
        const unsigned char* row = img + (size_t)stride * y + x_min;
        FLB_UNROLL
        for (int x = 0; x < 8; ++x) {
            const float dx = (float)((int)row[x + 1] - (int)row[x - 1]);
            const float dy = (float)((int)row[x + stride] - (int)row[x - stride]);
            dXX += dx * dx;
            dYY += dy * dy;
            dXY += dx * dy;
        }
    }
    dXX = (float)((double)dXX / (2.0 * 64));
    dYY = (float)((double)dYY / (2.0 * 64));
    dXY = (float)((double)dXY / (2.0 * 64));
    const float tr = dXX + dYY;
    return (float)(0.5 * (double)(tr - sqrtf(tr * tr - 4 * (dXX * dYY - dXY * dXY))));
}

// One scan point of LidarSelector::addSparseMap's first loop (src/lidar_selection.cpp:152-158): grid cell it
// falls into (-1: not in the frame with the `border` margin) and its corner score.
FLB_HD int visual_candidate(const CamModel& cam, const double* Rcw, const double* Pcw, const unsigned char* img, int stride,
                            const float* p, int grid_size, int grid_n_height, int border, float* score) {
    const double pt[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double pf[3], pc[2];
    m3_vec(Rcw, pt, pf);
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) pf[k] += Pcw[k];
    world2cam(cam, pf, pc);                                                         // Frame::w2c, include/frame.h:89
    if (!(fabs(pc[0]) < 1e9) || !(fabs(pc[1]) < 1e9)) return -1;
    const int ox = (int)pc[0], oy = (int)pc[1];                                     // pc.cast<int>()
    if (!(ox >= border && ox < cam.width - border && oy >= border && oy < cam.height - border)) return -1;   // isInFrame
    *score = shi_tomasi_score(img, cam.width, cam.height, stride, ox, oy);          // :158
    return (int)(pc[0] / grid_size) * grid_n_height + (int)(pc[1] / grid_size);     // :156
}

// ------------------------------------------------------------------ visual map: selection + warp (row f2), growth (row f4)
// Per-element math of LidarSelector::addFromSparseMap (src/lidar_selection.cpp:346-587) and its helpers.  vikit /
// Sophus / OpenCV pieces are restated from their published sources exactly as in oracle/flo_vmap.cpp.
FLB_HD void se3_apply(const double* R, const double* t, const double* p, double* o) {      // T * p
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) o[k] = R[3 * k] * p[0] + R[3 * k + 1] * p[1] + R[3 * k + 2] * p[2] + t[k];
}
FLB_HD void se3_pos(const double* R, const double* t, double* o) {                          // T.inverse().translation()
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) o[k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);
}

// vikit PinholeCamera::cam2world(px): unit bearing.  Distorted: cv::undistortPoints on one CV_32FC2 point
// (float in, five fixed-point iterations in double, float out).
FLB_HD void cam2world(const CamModel& cam, double u, double v, double* f) {
    double x, y;
    if (!(fabs(cam.d[0]) > 0.0000001)) {
        x = (u - cam.cx) / cam.fx;
        y = (v - cam.cy) / cam.fy;
    } else {
        const float uf = (float)u, vf = (float)v;
        const double x0 = ((double)uf - cam.cx) / cam.fx, y0 = ((double)vf - cam.cy) / cam.fy;
        double xx = x0, yy = y0;
        for (int j = 0; j < 5; ++j) {
            const double r2 = xx * xx + yy * yy;
            const double icdist = 1. / (1 + ((cam.d[4] * r2 + cam.d[1]) * r2 + cam.d[0]) * r2);
            const double deltaX = 2 * cam.d[2] * xx * yy + cam.d[3] * (r2 + 2 * xx * xx);
            const double deltaY = cam.d[2] * (r2 + 2 * yy * yy) + 2 * cam.d[3] * xx * yy;
            xx = (x0 - deltaX) * icdist;
            yy = (y0 - deltaY) * icdist;
        }
        x = (double)(float)xx;
        y = (double)(float)yy;
    }
    const double n = sqrt(x * x + y * y + 1.0);
    f[0] = x / n; f[1] = y / n; f[2] = 1.0 / n;
}

// vk::interpolateMat_8u
FLB_HD float interpolate_8u(const unsigned char* img, int stride, float u, float v) {
    const int x = (int)floorf(u), y = (int)floorf(v);
    const float subpix_x = u - x, subpix_y = v - y;
    const float w00 = (1.0f - subpix_x) * (1.0f - subpix_y);
    const float w01 = (1.0f - subpix_x) * subpix_y;
    const float w10 = subpix_x * (1.0f - subpix_y);
    const float w11 = 1.0f - w00 - w01 - w10;
    const unsigned char* ptr = img + (size_t)y * stride + x;
    return w00 * ptr[0] + w01 * ptr[stride] + w10 * ptr[1] + w11 * ptr[stride + 1];
}

// AbstractCamera::isInFrame(px.cast<int>(), boundary)
FLB_HD bool vm_in_frame(const CamModel& cam, double px0, double px1, int boundary) {
    if (!(fabs(px0) < 1e9) || !(fabs(px1) < 1e9)) return false;
    const int ox = (int)px0, oy = (int)px1;
    return ox >= boundary && ox < cam.width - boundary && oy >= boundary && oy < cam.height - boundary;
}

// Voxel keys.  sub_feat_map (:384-388): floor(pt / 0.5f) per axis; feat_map (AddPoint, :204-216): float quotient,
// "-= 1.0" for negatives, truncation.  Packed into 21 bits per axis (+-2^20 voxels of 0.5 m).
FLB_HD unsigned long long vm_pack_key(long long x, long long y, long long z) {
    const unsigned long long b = 1ull << 20;
    return (((unsigned long long)(z + (long long)b) & 0x1fffffull) << 42) | (((unsigned long long)(y + (long long)b) & 0x1fffffull) << 21) |
           ((unsigned long long)(x + (long long)b) & 0x1fffffull);
}
FLB_HD unsigned long long vm_scan_key(const float* p) {
    const float voxel_size = 0.5;
    long long k[3];
    FLB_UNROLL
    for (int j = 0; j < 3; ++j) k[j] = (long long)(int)floor((double)p[j] / voxel_size);
    return vm_pack_key(k[0], k[1], k[2]);
}
FLB_HD void vm_feat_key(const double* pt_w, long long* key) {
    const double voxel_size = 0.5;
    FLB_UNROLL
    for (int j = 0; j < 3; ++j) {
        float loc = (float)(pt_w[j] / voxel_size);
        if (loc < 0) loc -= 1.0;
        key[j] = (long long)loc;
    }
}

// getWarpMatrixAffine (:232-256) with level_ref = 0, pyramid_level = 0 (the only call site, :528-530).
// Rcr, tcr = T_cur_ref = T_cur * T_ref^-1.  A row-major 2x2.
FLB_HD void vm_warp_matrix(const CamModel& cam, const double* px_ref, const double* f_ref, double depth_ref, const double* Rcr,
                           const double* tcr, int halfpatch_size, double* A) {
    const double xyz_ref[3] = {f_ref[0] * depth_ref, f_ref[1] * depth_ref, f_ref[2] * depth_ref};
    const double step = (double)(halfpatch_size * (1 << 0) * (1 << 0));
    double xyz_du[3], xyz_dv[3];
    cam2world(cam, px_ref[0] + step, px_ref[1], xyz_du);
    cam2world(cam, px_ref[0], px_ref[1] + step, xyz_dv);
    const double su = xyz_ref[2] / xyz_du[2], sv = xyz_ref[2] / xyz_dv[2];
    FLB_UNROLL
    for (int k = 0; k < 3; ++k) { xyz_du[k] *= su; xyz_dv[k] *= sv; }
    double pc[3], pdu[3], pdv[3], px_cur[2], px_du[2], px_dv[2];
    se3_apply(Rcr, tcr, xyz_ref, pc);
    se3_apply(Rcr, tcr, xyz_du, pdu);
    se3_apply(Rcr, tcr, xyz_dv, pdv);
    world2cam(cam, pc, px_cur);
    world2cam(cam, pdu, px_du);
    world2cam(cam, pdv, px_dv);
    A[0] = (px_du[0] - px_cur[0]) / halfpatch_size;
    A[2] = (px_du[1] - px_cur[1]) / halfpatch_size;
    A[1] = (px_dv[0] - px_cur[0]) / halfpatch_size;
    A[3] = (px_dv[1] - px_cur[1]) / halfpatch_size;
}

FLB_HD int vm_best_search_level(const double* A, int max_level) {      // :317-331
    int search_level = 0;
    double D = A[0] * A[3] - A[1] * A[2];
    while (D > 3.0 && search_level < max_level) {
        search_level += 1;
        D *= 0.25;
    }
    return search_level;
}

// A_ref_cur = A_cur_ref.inverse().cast<float>() (:268): adjugate / determinant.  Returns false when NaN (:269).
FLB_HD bool vm_warp_inverse(const double* A_cur_ref, float* a) {
    const double det = A_cur_ref[0] * A_cur_ref[3] - A_cur_ref[1] * A_cur_ref[2];
    const double inv = 1.0 / det;
    a[0] = (float)(A_cur_ref[3] * inv); a[1] = (float)(-A_cur_ref[1] * inv);
    a[2] = (float)(-A_cur_ref[2] * inv); a[3] = (float)(A_cur_ref[0] * inv);
    return !(a[0] != a[0]);
}

// One element of warpAffine (:279-295): patch[64 * pyramid_level + 8 * y + x]
FLB_HD float vm_warp_pixel(const float* a, const unsigned char* img_ref, int width, int height, const double* px_ref,
                           int search_level, int pyramid_level, int halfpatch_size, int x, int y) {
    float px_patch0 = (float)(x - halfpatch_size), px_patch1 = (float)(y - halfpatch_size);
    px_patch0 *= (float)(1 << search_level); px_patch1 *= (float)(1 << search_level);
    px_patch0 *= (float)(1 << pyramid_level); px_patch1 *= (float)(1 << pyramid_level);
    const float pxr0 = (float)px_ref[0], pxr1 = (float)px_ref[1];
    const float px0 = a[0] * px_patch0 + a[1] * px_patch1 + pxr0, px1 = a[2] * px_patch0 + a[3] * px_patch1 + pxr1;
    if (px0 < 0 || px1 < 0 || px0 >= width - 1 || px1 >= height - 1) return 0.0f;
    return interpolate_8u(img_ref, width, px0, px1);
}

// One element of getpatch at level 0 (:121-141): patch_tmp[x * 8 + y], x = row, y = column.
struct VmPatchGeom { int u_i, v_i; float w_tl, w_tr, w_bl, w_br; };
FLB_HD void vm_getpatch_geom(const double* pc, VmPatchGeom& g) {
    const float u_ref = pc[0];
    const float v_ref = pc[1];
    const int scale = 1;
    g.u_i = floorf(pc[0] / scale) * scale;
    g.v_i = floorf(pc[1] / scale) * scale;
    const float subpix_u_ref = (u_ref - g.u_i) / scale;
    const float subpix_v_ref = (v_ref - g.v_i) / scale;
    g.w_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
    g.w_tr = subpix_u_ref * (1.0 - subpix_v_ref);
    g.w_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
    g.w_br = subpix_u_ref * subpix_v_ref;
}
FLB_HD float vm_getpatch_pixel(const unsigned char* img, int width, const VmPatchGeom& g, int halfpatch_size, int x, int y) {
    const unsigned char* p = img + (size_t)(g.v_i - halfpatch_size + x) * width + (g.u_i - halfpatch_size) + y;
    return g.w_tl * p[0] + g.w_tr * p[1] + g.w_bl * p[width] + g.w_br * p[width + 1];
}

// One point of publish_frame_world_rgb (src/laserMapping.cpp:726-741): project into the current frame, bilinear BGR
// sample (LidarSelector::getpixel, src/lidar_selection.cpp:1007-1025), stored as r, g, b bytes.  false: not coloured.
FLB_HD bool vm_colorize_point(const CamModel& cam, const double* Rcw, const double* Pcw, const unsigned char* bgr, const float* p,
                              unsigned char* rgb) {
    const double p_w[3] = {(double)p[0], (double)p[1], (double)p[2]};
    double pf[3], pc[2];
    se3_apply(Rcw, Pcw, p_w, pf);
    if (pf[2] < 0) return false;
    world2cam(cam, pf, pc);
    if (!vm_in_frame(cam, pc[0], pc[1], 0)) return false;
    const int width = cam.width;
    const float u_ref = pc[0];
    const float v_ref = pc[1];
    const int u_ref_i = floorf(pc[0]);
    const int v_ref_i = floorf(pc[1]);
    const float subpix_u_ref = (u_ref - u_ref_i);
    const float subpix_v_ref = (v_ref - v_ref_i);
    const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
    const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
    const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
    const float w_ref_br = subpix_u_ref * subpix_v_ref;
    // isInFrame(pc.cast<int>(), 0) lets pc in (-1, 0) through (its integer cast is 0) and the last row / column has no
    // bilinear neighbour: the reference then reads outside the image.  Defined here: both taps are clamped into it.
    const int u0 = min(max(u_ref_i, 0), cam.width - 1), u1 = min(max(u_ref_i + 1, 0), cam.width - 1);
    const int v0 = min(max(v_ref_i, 0), cam.height - 1), v1 = min(max(v_ref_i + 1, 0), cam.height - 1);
    const int du = (u1 - u0) * 3, dv = (v1 - v0) * width * 3;
    const unsigned char* img_ptr = bgr + ((size_t)v0 * width + u0) * 3;
    const float B = w_ref_tl * img_ptr[0] + w_ref_tr * img_ptr[0 + du] + w_ref_bl * img_ptr[dv] + w_ref_br * img_ptr[dv + 0 + du];
    const float G = w_ref_tl * img_ptr[1] + w_ref_tr * img_ptr[1 + du] + w_ref_bl * img_ptr[1 + dv] + w_ref_br * img_ptr[dv + 1 + du];
    const float R = w_ref_tl * img_ptr[2] + w_ref_tr * img_ptr[2 + du] + w_ref_bl * img_ptr[2 + dv] + w_ref_br * img_ptr[dv + 2 + du];
    rgb[0] = (unsigned char)(int)R; rgb[1] = (unsigned char)(int)G; rgb[2] = (unsigned char)(int)B;
    return true;
}

// ---- flb_rgb_cloud: laserCloudWorldRGB (src/laserMapping.cpp:726-747) as records, and its run-long save (pcl_wait_save,
// :777).  Words, not floats, so that no colour word is ever moved through a float register (r >= 128 makes it a NaN).
#if defined(__CUDACC__)
typedef uint4 rgb_word4;
#else
struct rgb_word4 { unsigned x, y, z, w; };
#endif
// The colour word of a kept point: pcl::PointXYZRGB's b, g, r, a bytes (offsets 16..19), a = 255 as PCL 1.8+ constructs it.
FLB_HD unsigned rgb_bgra_word(const unsigned char* rgb) {
    return (unsigned)rgb[2] | ((unsigned)rgb[1] << 8) | ((unsigned)rgb[0] << 16) | 0xFF000000u;
}
// k_rgb_flags, one world point: vm_colorize_point's verdict as the 0/1 keep flag, its colour word (0 when not kept).
FLB_HD int rgb_flag_point(const CamModel& cam, const double* Rcw, const double* Pcw, const unsigned char* bgr, const float* p,
                          unsigned* bgra) {
    unsigned char c[3] = {0, 0, 0};
    const bool ok = vm_colorize_point(cam, Rcw, Pcw, bgr, p, c);
    *bgra = ok ? rgb_bgra_word(c) : 0u;
    return ok ? 1 : 0;
}
// The save lives in chunks of 2^kRgbChunkLog2 16-byte records {x, y, z, bgra}; record i is entry i & mask of chunk i >> log2.
constexpr int kRgbChunkLog2 = 20;
FLB_HD rgb_word4* rgb_save_slot(rgb_word4* const* chunks, long long i, int chunk_log2) {
    return chunks[i >> chunk_log2] + (i & ((1LL << chunk_log2) - 1));
}
// The ABI's 32-byte record (pcl::PointXYZRGB): x, y, z, data[3] = 1.0f | bgra, three zero words; two 16-byte halves.
FLB_HD void rgb_record32(unsigned x, unsigned y, unsigned z, unsigned bgra, rgb_word4* rec) {
    rgb_word4 a, b;
    a.x = x; a.y = y; a.z = z; a.w = 0x3F800000u;
    b.x = bgra; b.y = 0u; b.z = 0u; b.w = 0u;
    rec[0] = a;
    rec[1] = b;
}
// k_rgb_scatter, one kept point p at its rank `slot`: its record in the frame's cloud and, chunks != NULL, its save record
// at save_base + slot.
FLB_HD void rgb_scatter_point(const float* p, unsigned bgra, int slot, rgb_word4* out, rgb_word4* const* chunks, long long save_base,
                              int chunk_log2) {
    const unsigned x = float_as_u32(p[0]), y = float_as_u32(p[1]), z = float_as_u32(p[2]);
    rgb_record32(x, y, z, bgra, out + 2 * (size_t)slot);
    if (chunks) {
        rgb_word4 s;
        s.x = x; s.y = y; s.z = z; s.w = bgra;
        *rgb_save_slot(chunks, save_base + slot, chunk_log2) = s;
    }
}
// k_rgb_save_pack, one save record expanded to the 32-byte record.
FLB_HD void rgb_save_expand(const rgb_word4& s, rgb_word4* rec) { rgb_record32(s.x, s.y, s.z, s.w, rec); }

// The device-resident visual map: Point (include/point.h) and Feature (include/feature.h) flattened.
constexpr int kVmMaxObs = 20;            // addObservation keeps obs_.size() < 20 before adding one (:946-952)
struct VmFeature {
    double px[2], f[3];                  // pixel on level 0, unit bearing
    double R[9], t[3];                   // T_f_w
    float score;
    int level, id, img;                  // img: slot of the keyframe image in the pool
};
struct VmPoint {
    double pos[3];
    float value;
    int n_obs;
    long long key[3];                    // feat_map voxel (AddPoint)
    int obs[kVmMaxObs + 1];              // obs[0] = newest (addFrameRef: push_front)
    int pad;
};
// Reclaim (flb_vmap_reclaim).  The reference's Feature is owned by Point::obs_ alone and its keyframe image by the
// Features that point to it (src/lidar_selection.cpp:183, :946-957), so both die with their last reference.  The device
// map restates that lifetime in one pass: a feature is live iff some point's obs[0..n_obs) names it; live features
// move to their rank among live features (creation order kept); an image slot is live iff a live feature names it.
// The point array is read as 32-bit words, one word per thread, so the passes over it are coalesced.
constexpr int kVmPointWords = (int)(sizeof(VmPoint) / 4);
constexpr int kVmNObsWord = (int)(offsetof(VmPoint, n_obs) / 4);
constexpr int kVmObsWord = (int)(offsetof(VmPoint, obs) / 4);
static_assert(sizeof(VmPoint) % 4 == 0, "VmPoint is read as 32-bit words");

// The live test: the feature id that word k of a point names (obs[q] with q < n_obs), or -1.
FLB_HD int vm_point_word_feature(const int* point_words, int k) {
    const int q = k - kVmObsWord;
    return (q >= 0 && q < point_words[kVmNObsWord]) ? point_words[k] : -1;
}
// rank = exclusive scan of the live flags over [0, n_features]: feature f is live iff its rank steps, and its new id is its
// rank (rank[n_features] = live features).
FLB_HD bool vm_feature_live(const int* rank, int f) { return rank[f + 1] != rank[f]; }
FLB_HD int vm_feature_remap(const int* rank, int f) { return rank[f]; }
// A slot goes onto the free-slot stack when no live feature names it and it is not the current frame's slot (pinned: a
// reclaim between select and grow / add_observations of one frame must leave that frame's committed image alone).
FLB_HD bool vm_slot_free(const int* slot_live, int pinned, int s) { return !slot_live[s] && s != pinned; }
// The slot the next keyframe image goes to: the top of the free-slot stack when it holds any, else the pool's tail.
FLB_HD int vm_image_slot(int n_free, const int* free_stack, int tail) { return n_free > 0 ? free_stack[n_free - 1] : tail; }

struct VmParams {
    int grid_size, grid_n_width, grid_n_height, length;
    int halfpatch;                       // patch_size_half = 4
    int ncc_en;
    double outlier_threshold, ncc_thre;
};

// Point::getCloseViewObs (src/point.cpp:141-178): the observation whose viewing direction is closest to the current
// one; -1 when there is none within 60 degrees.
FLB_HD int vm_close_view_obs(const VmPoint& pt, const VmFeature* feats, const double* frame_pos) {
    if (pt.n_obs <= 0) return -1;
    double obs_dir[3] = {frame_pos[0] - pt.pos[0], frame_pos[1] - pt.pos[1], frame_pos[2] - pt.pos[2]};
    {
        const double nn = norm3(obs_dir);
        FLB_UNROLL
        for (int k = 0; k < 3; ++k) obs_dir[k] /= nn;
    }
    int min_it = pt.obs[0];
    double min_cos_angle = 0;
    for (int q = 0; q < pt.n_obs; ++q) {
        const VmFeature& ft = feats[pt.obs[q]];
        double fpos[3], dir[3];
        se3_pos(ft.R, ft.t, fpos);
        FLB_UNROLL
        for (int k = 0; k < 3; ++k) dir[k] = fpos[k] - pt.pos[k];
        const double nn = norm3(dir);
        FLB_UNROLL
        for (int k = 0; k < 3; ++k) dir[k] /= nn;
        const double cos_angle = obs_dir[0] * dir[0] + obs_dir[1] * dir[1] + obs_dir[2] * dir[2];
        if (cos_angle > min_cos_angle) { min_cos_angle = cos_angle; min_it = pt.obs[q]; }
    }
    if (min_cos_angle < 0.5) return -1;
    return min_it;
}

// One grid cell of the third loop of addFromSparseMap (:479-580), executed by a team of cx.n lanes (a warp on the
// device, a single "lane" in the host emulation): depth-continuity test, closest-view observation, affine warp of the
// reference patch at three pyramid levels, current patch, NCC / SSD gates.  depth_img holds {scan index + 1 : depth
// bits} per pixel (the last scan point projecting into a pixel wins, :408-414).  Writes patch_wrap[192] and returns
// true (to every lane) when the cell is selected.
template <class Ctx>
FLB_HD bool vm_build_cell(const Ctx& cx, const CamModel& cam, const VmParams& prm, const double* Rcw, const double* Pcw,
                          const double* frame_pos, const VmPoint& pt, const VmFeature* feats, const unsigned char* img_pool,
                          const unsigned char* img_cur, const unsigned long long* depth_img, float* patch_wrap, float* patch_cur,
                          double* shared8, int* search_level_out, float* error_out) {
    const int width = cam.width, height = cam.height, hp = prm.halfpatch;
    double pt_cam[3], pc[2];
    se3_apply(Rcw, Pcw, pt.pos, pt_cam);
    world2cam(cam, pt_cam, pc);
    // depth continuity (:492-514): any scan depth in the (2hp+1)^2 window (centre excluded) more than 1.5 m off
    bool bad = false;
    const int side = 2 * hp + 1;
    for (int e = cx.lane; e < side * side; e += cx.n) {
        const int u = e / side - hp, v = e % side - hp;
        if (u == 0 && v == 0) continue;
        const unsigned long long cell = depth_img[(size_t)width * (v + (int)pc[1]) + u + (int)pc[0]];
        const float depth = u32_as_float((unsigned)cell);
        if (depth == 0.) continue;
        const double delta_dist = fabs(pt_cam[2] - depth);
        if (delta_dist > 1.5) bad = true;
    }
    if (cx.any(bad)) return false;
    // closest-view observation + warp matrix: lane 0, then shared with the team
    if (cx.lane == 0) {
        const int fi = vm_close_view_obs(pt, feats, frame_pos);
        shared8[7] = (double)fi;
        if (fi >= 0) {
            const VmFeature& ref = feats[fi];
            double Rcr[9], tcr[3], rpos[3];
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    Rcr[3 * a + b] = Rcw[3 * a] * ref.R[3 * b] + Rcw[3 * a + 1] * ref.R[3 * b + 1] + Rcw[3 * a + 2] * ref.R[3 * b + 2];
            se3_pos(ref.R, ref.t, rpos);
            se3_apply(Rcw, Pcw, rpos, tcr);
            const double dvec[3] = {rpos[0] - pt.pos[0], rpos[1] - pt.pos[1], rpos[2] - pt.pos[2]};
            vm_warp_matrix(cam, ref.px, ref.f, norm3(dvec), Rcr, tcr, hp, shared8);             // :528-530
            shared8[4] = (double)vm_best_search_level(shared8, 2);                               // :532
        }
    }
    cx.sync();
    const int fi = (int)shared8[7];
    const int search_level = (int)shared8[4];
    float a[4];
    const bool inv_ok = vm_warp_inverse(shared8, a);
    cx.sync();                                    // every lane has read lane 0's results: shared8 may be reused
    if (fi < 0) return false;
    const VmFeature& ref = feats[fi];
    const unsigned char* img_ref = img_pool + (size_t)ref.img * (size_t)width * (size_t)height;
    const int ps = 2 * hp, total = ps * ps;
    for (int e = cx.lane; e < 3 * total; e += cx.n) {                                           // :542-545
        const int lvl = e / total, r = e % total, y = r / ps, x = r % ps;
        patch_wrap[e] = inv_ok ? vm_warp_pixel(a, img_ref, width, height, ref.px, search_level, lvl, hp, x, y) : 0.0f;
    }
    VmPatchGeom g;
    vm_getpatch_geom(pc, g);
    for (int e = cx.lane; e < total; e += cx.n) patch_cur[e] = vm_getpatch_pixel(img_cur, width, g, hp, e / ps, e % ps);   // :547
    cx.sync();
    if (cx.lane == 0) {
        bool keep = true;
        if (prm.ncc_en) {                                                                        // NCC, :298-315
            double sum_ref = 0.0, sum_cur = 0.0;
            for (int i = 0; i < total; ++i) sum_ref += patch_wrap[i];
            const double mean_ref = sum_ref / total;
            for (int i = 0; i < total; ++i) sum_cur += patch_cur[i];
            const double mean_curr = sum_cur / total;
            double numerator = 0, demoniator1 = 0, demoniator2 = 0;
            for (int i = 0; i < total; i++) {
                const double n = (patch_wrap[i] - mean_ref) * (patch_cur[i] - mean_curr);
                numerator += n;
                demoniator1 += (patch_wrap[i] - mean_ref) * (patch_wrap[i] - mean_ref);
                demoniator2 += (patch_cur[i] - mean_curr) * (patch_cur[i] - mean_curr);
            }
            const double ncc = numerator / sqrt(demoniator1 * demoniator2 + 1e-10);
            if (ncc < prm.ncc_thre) keep = false;
        }
        float error = 0.0;
        for (int ind = 0; ind < total; ind++) error += (patch_wrap[ind] - patch_cur[ind]) * (patch_wrap[ind] - patch_cur[ind]);
        if (error > prm.outlier_threshold * total) keep = false;                                 // :560
        shared8[5] = keep ? 1.0 : 0.0;
        shared8[6] = (double)error;
    }
    cx.sync();
    const bool keep = shared8[5] != 0.0;
    *search_level_out = search_level;
    *error_out = (float)shared8[6];
    cx.sync();
    return keep;
}

// One selected patch of addObservation (:913-965): should a new observation be added (pose / pixel-distance tests),
// which observation goes when the list is full (Point::getFurthestViewObs, src/point.cpp:219-247).
FLB_HD bool vm_observation_test(const CamModel& cam, const double* Rcw, const double* Pcw, const double* cur_pos, const VmPoint& pt,
                                const VmFeature* feats, double* pc, int* erase_slot) {
    double pf[3];
    se3_apply(Rcw, Pcw, pt.pos, pf);
    world2cam(cam, pf, pc);
    bool add_flag = false;
    const VmFeature& last = feats[pt.obs[pt.n_obs - 1]];                                         // obs_.back()
    double Rd[9], td[3];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) Rd[3 * a + b] = last.R[3 * a] * Rcw[3 * b] + last.R[3 * a + 1] * Rcw[3 * b + 1] + last.R[3 * a + 2] * Rcw[3 * b + 2];
    se3_apply(last.R, last.t, cur_pos, td);
    const double delta_p = norm3(td);
    const double tr = Rd[0] + Rd[4] + Rd[8];
    const double delta_theta = (tr > 3.0 - 1e-6) ? 0.0 : acos(0.5 * (tr - 1));
    if (delta_p > 0.5 || delta_theta > 10) add_flag = true;
    const double dpx[2] = {pc[0] - last.px[0], pc[1] - last.px[1]};
    const double pixel_dist = sqrt(dpx[0] * dpx[0] + dpx[1] * dpx[1]);
    if (pixel_dist > 40) add_flag = true;
    *erase_slot = -1;
    if (pt.n_obs >= kVmMaxObs) {
        int max_it = 0;
        double maxdist = 0.0;
        for (int q = 0; q < pt.n_obs; ++q) {
            double fpos[3];
            se3_pos(feats[pt.obs[q]].R, feats[pt.obs[q]].t, fpos);
            const double d[3] = {fpos[0] - cur_pos[0], fpos[1] - cur_pos[1], fpos[2] - cur_pos[2]};
            const double dist = norm3(d);
            if (dist > maxdist) { maxdist = dist; max_it = q; }
        }
        *erase_slot = max_it;
    }
    return add_flag;
}

// ------------------------------------------------------------------ IKFoM manifold algebra (row a8)
// state_ikfom = pos, rot(SO3), offset_R_L_I(SO3), offset_T_L_I, vel, bg, ba, grav(S2, |g| = 9.8090)
// (include/use-ikfom.hpp:12-21; DOF 23).  Quaternions are (x, y, z, w) like Eigen's coeffs().
// MTK primitives restated from include/IKFoM_toolkit/mtk/{src/mtkmath.hpp, types/SOn.hpp, types/S2.hpp}.
constexpr int kIk = 23;
constexpr double kMtkTol = 1e-11;                 // MTK::tolerance<double>()
constexpr double kGravLen = 98090.0 / 10000.0;    // S2<double, 98090, 10000, 1>::length

struct StateIkfom {
    double pos[3], rot[4], offset_R_L_I[4], offset_T_L_I[3], vel[3], bg[3], ba[3], grav[3];
    double P[kIk * kIk];
};
constexpr int kIkHead = 26;   // doubles before P

FLB_HD void mm_small(const double* A, int ra, int ca, const double* B, int cb, double* C) {
    for (int i = 0; i < ra; ++i)
        for (int j = 0; j < cb; ++j) {
            double s = 0;
            for (int k = 0; k < ca; ++k) s += A[i * ca + k] * B[k * cb + j];
            C[i * cb + j] = s;
        }
}
FLB_HD void transpose_small(const double* A, int r, int c, double* T) {
    for (int i = 0; i < r; ++i)
        for (int j = 0; j < c; ++j) T[j * r + i] = A[i * c + j];
}

// mtkmath.hpp:141-171
FLB_HD void mtk_cos_sinc_sqrt(double x2, double* c, double* sc) {
    const double taylor_0 = 2.220446049250313e-16;
    const double taylor_2 = sqrt(taylor_0);
    const double taylor_n = sqrt(taylor_2);
    if (x2 >= taylor_n) {
        const double x = sqrt(x2);
        *c = cos(x);
        *sc = sin(x) / x;
        return;
    }
    const double inv[7] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
    double cosi = 1., sinc = 1;
    double term = -1 / 2. * x2;
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        cosi += term;
        term *= inv[2 * i];
        sinc += term;
        term *= -inv[2 * i + 1] * x2;
    }
    *c = cosi;
    *sc = sinc;
}
// SO3::exp(vec, scale) (SOn.hpp:282-286, mtkmath.hpp:249-256)
FLB_HD void quat_exp(const double* v, double scale, double* q) {
    const double n2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    double c, sc;
    mtk_cos_sinc_sqrt(scale * scale * n2, &c, &sc);
    const double mult = sc * scale;
    q[0] = mult * v[0]; q[1] = mult * v[1]; q[2] = mult * v[2];
    q[3] = c;
}
FLB_HD void quat_mul(const double* a, const double* b, double* o) {
    const double ax = a[0], ay = a[1], az = a[2], aw = a[3], bx = b[0], by = b[1], bz = b[2], bw = b[3];
    o[3] = aw * bw - ax * bx - ay * by - az * bz;
    o[0] = aw * bx + ax * bw + ay * bz - az * by;
    o[1] = aw * by + ay * bw + az * bx - ax * bz;
    o[2] = aw * bz + az * bw + ax * by - ay * bx;
}
FLB_HD void quat_to_R(const double* q, double* R) {   // Eigen::Quaternion::toRotationMatrix
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y,
                 tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
// SO3::log (SOn.hpp:291-295, mtkmath.hpp:269-289 with plus_minus_periodicity = true)
FLB_HD void quat_log(const double* q, double* out) {
    double nv = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    if (nv < kMtkTol) nv = kMtkTol;
    const double s = 2.0 / nv * atan(nv / q[3]);
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) out[i] = s * q[i];
}
// MTK::A_matrix, mtkmath.hpp:235-247
FLB_HD void mtk_A_matrix(const double* v, double* A) {
    const double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    const double nrm = sqrt(sq);
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) A[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (nrm < kMtkTol) return;
    double K[9], KK[9];
    skew3(v, K);
    mm_small(K, 3, 3, K, 3, KK);
    const double a = (1 - cos(nrm)) / sq, b = (1 - sin(nrm) / nrm) / sq;
    FLB_UNROLL
    for (int i = 0; i < 9; ++i) A[i] = A[i] + a * K[i] + b * KK[i];
}
// S2 (S2_typ = 1), S2.hpp:206-231
FLB_HD void s2_Bx(const double* vec, double* Bx /*3x2*/) {
    if (vec[0] + kGravLen > kMtkTol) {
        const double d = kGravLen + vec[0];
        Bx[0] = -vec[1];                        Bx[1] = -vec[2];
        Bx[2] = kGravLen - vec[1] * vec[1] / d; Bx[3] = -vec[2] * vec[1] / d;
        Bx[4] = -vec[2] * vec[1] / d;           Bx[5] = kGravLen - vec[2] * vec[2] / d;
        FLB_UNROLL
        for (int i = 0; i < 6; ++i) Bx[i] /= kGravLen;
    } else {
        FLB_UNROLL
        for (int i = 0; i < 6; ++i) Bx[i] = 0;
        Bx[3] = -1;
        Bx[4] = 1;
    }
}
FLB_HD void s2_boxplus(double* vec, const double* delta) {   // S2.hpp:112-118
    double Bx[6], Bu[3], q[4], R[9], o[3];
    s2_Bx(vec, Bx);
    mm_small(Bx, 3, 2, delta, 1, Bu);
    quat_exp(Bu, 0.5, q);
    quat_to_R(q, R);
    mm_small(R, 3, 3, vec, 1, o);
    vec[0] = o[0]; vec[1] = o[1]; vec[2] = o[2];
}
FLB_HD void s2_boxminus(const double* vec, const double* other, double* res) {   // S2.hpp:120-144
    double K[9], t[3];
    skew3(vec, K);
    mm_small(K, 3, 3, other, 1, t);
    const double v_sin = sqrt(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
    const double v_cos = vec[0] * other[0] + vec[1] * other[1] + vec[2] * other[2];
    const double theta = atan2(v_sin, v_cos);
    if (v_sin < kMtkTol) {
        if (fabs(theta) > kMtkTol) { res[0] = 3.1415926; res[1] = 0; }
        else { res[0] = 0; res[1] = 0; }
    } else {
        double Bx[6], BxT[6], Ko[9], u[3], r2[2];
        s2_Bx(other, Bx);
        transpose_small(Bx, 3, 2, BxT);
        skew3(other, Ko);
        mm_small(Ko, 3, 3, vec, 1, u);
        mm_small(BxT, 2, 3, u, 1, r2);
        res[0] = theta / v_sin * r2[0];
        res[1] = theta / v_sin * r2[1];
    }
}
FLB_HD void s2_Nx_yy(const double* vec, double* Nx /*2x3*/) {   // S2.hpp:262-267
    double Bx[6], BxT[6], K[9];
    s2_Bx(vec, Bx);
    transpose_small(Bx, 3, 2, BxT);
    skew3(vec, K);
    mm_small(BxT, 2, 3, K, 3, Nx);
    FLB_UNROLL
    for (int i = 0; i < 6; ++i) Nx[i] = 1 / kGravLen / kGravLen * Nx[i];
}
FLB_HD void s2_Mx(const double* vec, const double* delta, double* Mx /*3x2*/) {   // S2.hpp:269-283
    double Bx[6], K[9];
    s2_Bx(vec, Bx);
    skew3(vec, K);
    if (sqrt(delta[0] * delta[0] + delta[1] * delta[1]) < kMtkTol) {
        mm_small(K, 3, 3, Bx, 2, Mx);
        FLB_UNROLL
        for (int i = 0; i < 6; ++i) Mx[i] = -Mx[i];
    } else {
        // the reference passes scalar(1/2) == 0 (integer division) to MTK::exp here (S2.hpp:280):
        // exp_delta is the identity rotation.  Mirrored.
        double Bu[3], q[4], R[9], A[9], AT[9], t1[9], t2[9];
        mm_small(Bx, 3, 2, delta, 1, Bu);
        quat_exp(Bu, 0.0, q);
        quat_to_R(q, R);
        mtk_A_matrix(Bu, A);
        transpose_small(A, 3, 3, AT);
        mm_small(R, 3, 3, K, 3, t1);
        mm_small(t1, 3, 3, AT, 3, t2);
        mm_small(t2, 3, 3, Bx, 2, Mx);
        FLB_UNROLL
        for (int i = 0; i < 6; ++i) Mx[i] = -Mx[i];
    }
}
// state_ikfom::boxplus / boxminus (build_manifold.hpp:192-202)
FLB_HD void ikfom_boxplus(StateIkfom& x, const double* d) {
    double q[4], o[4];
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) x.pos[i] += d[i];
    quat_exp(d + 3, 0.5, q);
    quat_mul(x.rot, q, o);
    FLB_UNROLL
    for (int i = 0; i < 4; ++i) x.rot[i] = o[i];
    quat_exp(d + 6, 0.5, q);
    quat_mul(x.offset_R_L_I, q, o);
    FLB_UNROLL
    for (int i = 0; i < 4; ++i) x.offset_R_L_I[i] = o[i];
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        x.offset_T_L_I[i] += d[9 + i];
        x.vel[i] += d[12 + i];
        x.bg[i] += d[15 + i];
        x.ba[i] += d[18 + i];
    }
    s2_boxplus(x.grav, d + 21);
}
FLB_HD void ikfom_boxminus(const StateIkfom& a, const StateIkfom& b, double* res) {   // a [-] b
    double c[4], q[4];
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) res[i] = a.pos[i] - b.pos[i];
    c[0] = -b.rot[0]; c[1] = -b.rot[1]; c[2] = -b.rot[2]; c[3] = b.rot[3];
    quat_mul(c, a.rot, q);
    quat_log(q, res + 3);
    c[0] = -b.offset_R_L_I[0]; c[1] = -b.offset_R_L_I[1]; c[2] = -b.offset_R_L_I[2]; c[3] = b.offset_R_L_I[3];
    quat_mul(c, a.offset_R_L_I, q);
    quat_log(q, res + 6);
    FLB_UNROLL
    for (int i = 0; i < 3; ++i) {
        res[9 + i] = a.offset_T_L_I[i] - b.offset_T_L_I[i];
        res[12 + i] = a.vel[i] - b.vel[i];
        res[15 + i] = a.bg[i] - b.bg[i];
        res[18 + i] = a.ba[i] - b.ba[i];
    }
    s2_boxminus(a.grav, b.grav, res + 21);
}

// ------------------------------------------------------------------ camera frame preparation (LidarSelector::detect)
// cv::cvtColor(img, img, CV_BGR2GRAY) on 8-bit BGR (src/lidar_selection.cpp:1037): OpenCV's fixed-point weights, with
// the rounding shift of the OpenCV generation the caller links (FLB_GRAY_CV4 / FLB_GRAY_CV3 in the C ABI).
enum { kGrayCv4 = 0, kGrayCv3 = 1 };
FLB_HD unsigned bgr_to_gray(unsigned b, unsigned g, unsigned r, int rule) {
    return rule == kGrayCv3 ? (1868u * b + 9617u * g + 4899u * r + (1u << 13)) >> 14
                            : (3735u * b + 19235u * g + 9798u * r + (1u << 14)) >> 15;
}
// cv::resize(img, img, Size(), 0.5, 0.5, INTER_LINEAR) of an even-sized 8-bit frame (:1031-1034): OpenCV takes its
// 2x2 area path there, one rounded mean per channel of each 2x2 source block.
FLB_HD unsigned mean2x2(unsigned a, unsigned b, unsigned c, unsigned d) { return (a + b + c + d + 2u) >> 2; }

// The camera message's encodings (FLB_ENC_* in the C ABI), each as cv_bridge::toCvCopy(msg, "bgr8") converts it.
enum { kEncBgr8 = 0, kEncRgb8 = 1, kEncMono8 = 2, kEncBgra8 = 3, kEncRgba8 = 4,
       kEncBayerRggb8 = 5, kEncBayerBggr8 = 6, kEncBayerGbrg8 = 7, kEncBayerGrbg8 = 8 };
FLB_HD constexpr int enc_bpp(int enc) { return (enc == kEncMono8 || enc >= kEncBayerRggb8) ? 1 : (enc == kEncBgra8 || enc == kEncRgba8) ? 4 : 3; }
// The byte of a packed pixel (BGR8, RGB8, MONO8, BGRA8, RGBA8) that holds BGR channel ch (0 b, 1 g, 2 r): the
// cvtColor of each to BGR is this byte permutation (GRAY2BGR repeats the one byte, the alpha byte is dropped).
FLB_HD constexpr int enc_byte(int enc, int ch) { return enc == kEncMono8 ? 0 : (enc == kEncRgb8 || enc == kEncRgba8) ? 2 - ch : ch; }

// The colour (0 b, 1 g, 2 r) of site (x, y) of a Bayer mosaic; the ROS encoding names the 2x2 tile from its top-left.
FLB_HD int bayer_site(int enc, int x, int y) {
    const unsigned tile = enc == kEncBayerRggb8 ? 0x0112u : enc == kEncBayerBggr8 ? 0x2110u : enc == kEncBayerGbrg8 ? 0x1201u : 0x1021u;
    return (int)((tile >> (4 * (2 * (y & 1) + (x & 1)))) & 0xfu);
}
// cv_bridge's Bayer -> bgr8 (cvtColor COLOR_Bayer{BG,RG,GR,GB}2BGR for rggb8, bggr8, gbrg8, grbg8): OpenCV's bilinear
// demosaic of pixel (x, y) of a dense w x h mosaic m, w >= 3 and h >= 3.  Interior: the site's own colour as it is; G
// at an R / B site the rounded mean of its 4 edge neighbours, the other of R / B the rounded mean of its 4 diagonals;
// R and B at a G site the rounded mean of the horizontal or the vertical pair of that colour.  The outer rows and
// columns copy the nearest interior pixel.
FLB_HD void bayer_bgr(const unsigned char* m, int w, int h, int enc, int x, int y, unsigned& b, unsigned& g, unsigned& r) {
    x = x < 1 ? 1 : (x > w - 2 ? w - 2 : x);
    y = y < 1 ? 1 : (y > h - 2 ? h - 2 : y);
    const unsigned char* p = m + (size_t)y * w + x;
    const unsigned v = p[0];
    const int site = bayer_site(enc, x, y);
    if (site == 1) {
        const unsigned hp = (p[-1] + p[1] + 1u) >> 1, vp = (p[-w] + p[w] + 1u) >> 1;
        const bool b_horizontal = bayer_site(enc, x - 1, y) == 0;
        g = v;
        b = b_horizontal ? hp : vp;
        r = b_horizontal ? vp : hp;
    } else {
        const unsigned diag = (p[-w - 1] + p[-w + 1] + p[w - 1] + p[w + 1] + 2u) >> 2;
        g = (p[-w] + p[w] + p[-1] + p[1] + 2u) >> 2;
        b = site == 0 ? v : diag;
        r = site == 2 ? v : diag;
    }
}

// cv::resize(img, Size(w * 0.5, h * 0.5), INTER_LINEAR) of an 8-bit frame that is not exactly twice the output size
// (an odd side): OpenCV's fixed-point linear rule, 11-bit weights (INTER_RESIZE_COEF_BITS).  Output index d of n from
// a source axis of s: the first tap o (the second is min(o + 1, s - 1)) and the weights a0, a1, each rounded on its own
// from the float position as OpenCV rounds them; positions outside the source take the edge pixel with weights
// (2048, 0).  Needs double division, products and sums that round once each (no FMA contraction).
struct LinearTap {
    int o, a0, a1;
};
FLB_HD LinearTap linear_tap(int d, int n, int s) {
    const double scale = 1.0 / ((double)n / s);
    float f = (float)((d + 0.5) * scale - 0.5);
    int o = (int)floorf(f);
    f -= (float)o;
    if (o < 0) { f = 0.f; o = 0; }
    if (o >= s - 1) { f = 0.f; o = s - 1; }
    return LinearTap{o, (int)rintf((1.f - f) * 2048.f), (int)rintf(f * 2048.f)};
}
// The vertical step of that rule on two horizontal sums (src * 2048 scale): OpenCV's 8-bit rounding, which drops 4
// bits of each sum and 16 of each product before the final rounded shift.
FLB_HD unsigned linear_v(int s0, int s1, int b0, int b1) { return (unsigned)((((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2); }

// ------------------------------------------------------------------ LiDAR message decode (Preprocess::process)
// The non-feature (`else`) branches of the four handlers of src/preprocess.cpp, one driver record at a time
// (flb_lidar_upload).  A record is `step` bytes; its fields sit at the byte offsets of LidarFmt.
enum { kLidarLivox = 1, kLidarVelodyne = 2, kLidarOuster = 3, kLidarXt32 = 4 };
struct LidarFmt {
    int kind, step, off_x, off_y, off_z, off_time, off_tag, off_line, n_scans, filter_num;
    double blind;
    double time_head;      // XT32: points[0].timestamp (:441)
};
struct LidarPoint { float x, y, z, t; };      // t: PointType::curvature, the offset from the scan start in ms

// 32 bits of a little-endian record field.  PointCloud2 steps are arbitrary and a Livox record is 20 bytes, so a field is
// 4-byte aligned in memory only when the record's address is.
FLB_HD unsigned lidar_ld32(const unsigned char* p) {
    if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) return *reinterpret_cast<const unsigned*>(p);
    return (unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24);
}
FLB_HD double lidar_ld64f(const unsigned char* p) {
    const unsigned long long u = (unsigned long long)lidar_ld32(p) | ((unsigned long long)lidar_ld32(p + 4) << 32);
    double d;
    memcpy(&d, &u, sizeof(d));
    return d;
}

// x, y, z and the per-point time of record r, with each handler's own arithmetic.
FLB_HD LidarPoint lidar_decode(const unsigned char* r, const LidarFmt& f) {
    LidarPoint q;
    q.x = u32_as_float(lidar_ld32(r + f.off_x));
    q.y = u32_as_float(lidar_ld32(r + f.off_y));
    q.z = u32_as_float(lidar_ld32(r + f.off_z));
    if (f.kind == kLidarLivox) q.t = (float)lidar_ld32(r + f.off_time) / float(1000000);          // :149
    else if (f.kind == kLidarOuster) q.t = (float)lidar_ld32(r + f.off_time) * 1.e-6f;            // :250
    else if (f.kind == kLidarVelodyne) q.t = u32_as_float(lidar_ld32(r + f.off_time)) * 1.e-3f;   // :387
    else q.t = (float)((lidar_ld64f(r + f.off_time) - f.time_head) * (double)1000.f);             // :454
    return q;
}
// Livox: the record counts in valid_num (:140).  The loop starts at record 1 (:138), so record 0 never does.
FLB_HD bool lidar_livox_valid(const unsigned char* r, int i, const LidarFmt& f) {
    const unsigned tag = r[f.off_tag] & 0x30u;
    return i >= 1 && (int)r[f.off_line] < f.n_scans && (tag == 0x10u || tag == 0x00u);
}
// Livox: record i reaches :145 when it is valid and valid_num (the count of valid records up to and including it)
// is a multiple of point_filter_num (:143, unsigned arithmetic).
FLB_HD bool lidar_livox_candidate(bool valid, unsigned valid_num, const LidarFmt& f) {
    return valid && valid_num % (unsigned)f.filter_num == 0u;
}
// Livox, :151-154.  prev is pl_full[i-1]: record i-1's coordinates when that record was itself a candidate, otherwise
// the zeros pl_full.resize left there (:83).  abs is the float overload; 1e-7 and blind * blind are doubles.
FLB_HD bool lidar_livox_keep(const LidarPoint& q, float px, float py, float pz, double blind) {
    const bool moved = (double)fabsf(q.x - px) > 1e-7 || (double)fabsf(q.y - py) > 1e-7 || (double)fabsf(q.z - pz) > 1e-7;
    return moved && (double)(q.x * q.x + q.y * q.y + q.z * q.z) > blind * blind;
}
// Ouster :235-239, Velodyne :421-423, XT32 :456-458 (which compares with blind itself, not its square).
FLB_HD bool lidar_pc2_keep(const LidarPoint& q, int i, const LidarFmt& f) {
    if (i % f.filter_num != 0) return false;
    const float range = q.x * q.x + q.y * q.y + q.z * q.z;
    if (f.kind == kLidarOuster) return !((double)range < f.blind * f.blind);
    if (f.kind == kLidarVelodyne) return (double)range > f.blind * f.blind;
    return (double)range > f.blind;
}
// Order-preserving 32-bit key of a finite time for the radix sort: -0.0 and +0.0 share a key, as they compare equal in
// time_list (include/common_lib.h), so that ties keep record order.
FLB_HD unsigned lidar_time_key(float t) {
    const unsigned u = float_as_u32(t == 0.f ? 0.f : t);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
FLB_HD bool lidar_finite(float v) { return (float_as_u32(v) & 0x7f800000u) != 0x7f800000u; }

// ------------------------------------------------------------------ Velodyne times from the yaw angle
// velodyne_handler's non-feature branch without per-point times (src/preprocess.cpp:376-428, flb_lidar_upload_velodyne).
// Per ring, the first record sets yaw_fp and time_last = 0 and is never kept; every later record j gets
//   base_j = float((yaw_fp - yaw_j [+ 360]) / omega_l),  t_j = base_j < time_last ? float(base_j + 360 / omega_l) : base_j,
// and time_last = t_j.  Each step is the map x -> x > c ? a : b on time_last; such maps compose into one of the same form,
// so the walk over a ring is an inclusive scan of VeloMap under velo_compose.

// 16 bits of a little-endian record field at any offset (the ring)
FLB_HD unsigned lidar_ld16(const unsigned char* p) { return (unsigned)p[0] | ((unsigned)p[1] << 8); }

// omega_l (:272) and 360.0 / omega_l (:415), in the reference's double arithmetic
FLB_HD double velo_omega() { return 0.361 * 10; }
FLB_HD double velo_wrap() { return 360.0 / velo_omega(); }

// The yaw of :392 in degrees.  The reference calls atan2 on two floats, which resolves to the float overload and so to
// the libm it links; the project defines the angle as the double atan2 rounded to float (DESIGN §2).  The widening to
// double before the multiply is the reference's.
FLB_HD double velo_yaw(float x, float y) { return (double)(float)atan2((double)y, (double)x) * 57.2957; }

struct VeloMap { float c, a, b; };    // x -> (x > c) ? a : b

FLB_HD float velo_apply(const VeloMap& m, float x) { return x > m.c ? m.a : m.b; }
// `first` then `then`: x > first.c selects first.a or first.b, which `then` maps on.  Exact for every input, NaN
// included (a NaN compares false), so the operator is associative.
FLB_HD VeloMap velo_compose(const VeloMap& first, const VeloMap& then) {
    VeloMap m;
    m.c = first.c;
    m.a = velo_apply(then, first.a);
    m.b = velo_apply(then, first.b);
    return m;
}
// The first record of a ring: time_last = 0 whatever came before (:394-403).  A constant map, so a scan in ring order
// needs no segment boundaries: the head absorbs the prefix of the rings before it.
FLB_HD VeloMap velo_head() { VeloMap m; m.c = 0.f; m.a = 0.f; m.b = 0.f; return m; }
// Every later record of the ring (:406-417).  A NaN yaw gives a NaN base, so the next record cannot wrap.
FLB_HD VeloMap velo_step(double yaw, double yaw_fp) {
    const float base = yaw <= yaw_fp ? (float)((yaw_fp - yaw) / velo_omega()) : (float)((yaw_fp - yaw + 360.0) / velo_omega());
    VeloMap m;
    m.c = base;
    m.a = (float)((double)base + velo_wrap());
    m.b = base;
    return m;
}

// ------------------------------------------------------------------ LiDAR surface features (give_feature)
// The feature branches of avia_handler (:94-135), oust64_handler (:174-227) and velodyne_handler (:299-373), with
// give_feature (:466-775), plane_judge (:786-898) and edge_jump_judge (:900-936), one point at a time
// (flb_lidar_upload_features).  The points sit line-major in one array; a line is the segment [b, b + m) of it and the
// functions below take `pl`, `rng` and `dista` already offset to the line's first point, with local indices.
enum { kFtNor = 0, kFtPossPlane = 1, kFtRealPlane = 2, kFtEdgeJump = 3, kFtEdgePlane = 4, kFtWire = 5 };   // Feature
enum { kNrNor = 0, kNrZero = 1, kNr180 = 2, kNrInf = 3, kNrBlind = 4 };                                  // E_jump
enum { kStepNone = -1, kStepNonPlane = 0, kStepPlane = 1, kStepBlind = 2, kStepSkip = 3 };   // plane_judge's result; kStepSkip: a blind i (:495)
constexpr int kFeatGroup = 8;          // group_size (:11)

// Preprocess's constants (:9-30).  The four cosines are the constructor's std::cos values, computed on the host.
struct FeatConst {
    double blind, dis_b;
    double jump_up, jump_down, cos160, smallp_intersect;
    int avia;                          // lidar_type == AVIA: plane_judge's median test and range without sqrt
};

FLB_HD unsigned long long feat_d2u(double d) {
#if defined(__CUDA_ARCH__)
    return (unsigned long long)__double_as_longlong(d);
#else
    unsigned long long u;
    memcpy(&u, &d, sizeof(u));
    return u;
#endif
}
FLB_HD double feat_u2d(unsigned long long u) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double d;
    memcpy(&d, &u, sizeof(d));
    return d;
#endif
}
FLB_HD bool feat_isnan(double d) { return d != d; }

// Livox, :94-111: the line of record i, or n_scans when the record is not kept.  abs is the float overload on the raw
// previous record; x*x + y*y is compared with blind itself.  line == N_SCANS passes the filter but lands in a buffer
// that is never processed (:114), so it is dropped too.
FLB_HD int feat_livox_line(const unsigned char* r, int i, const LidarFmt& f) {
    if (i < 1) return f.n_scans;
    const LidarPoint q = lidar_decode(r, f), p = lidar_decode(r - f.step, f);
    const int line = r[f.off_line];
    if ((double)fabsf(q.x - p.x) < 1e-8 || (double)fabsf(q.y - p.y) < 1e-8 || (double)fabsf(q.z - p.z) < 1e-8 ||
        (double)(q.x * q.x + q.y * q.y) < f.blind || line > f.n_scans || (r[f.off_tag] & 0x30u) != 0x10u)
        return f.n_scans;
    return line;
}
// Ouster, :182-205: the 3-D float sum widened to double against blind * blind; the u8 ring (off_line) below N_SCANS.
FLB_HD int feat_ouster_line(const unsigned char* r, const LidarFmt& f) {
    const LidarPoint q = lidar_decode(r, f);
    if ((double)(q.x * q.x + q.y * q.y + q.z * q.z) < f.blind * f.blind) return f.n_scans;
    const int ring = r[f.off_line];
    return ring < f.n_scans ? ring : f.n_scans;
}

// types[i].range (:126, :218, :364): Livox the unsquared 2-D sum, the others its float sqrt.
FLB_HD double feat_range(const LidarPoint& p, int avia) {
    const float s = p.x * p.x + p.y * p.y;
    return avia ? (double)s : (double)sqrtf(s);
}
// types[i].dista (:127-130): float differences into the double members vx, vy, vz.  The line's last point has none
// (types.resize leaves it unwritten); the project defines it as 0.0.
FLB_HD double feat_dista(const LidarPoint& a, const LidarPoint& b) {
    const double vx = a.x - b.x, vy = a.y - b.y, vz = a.z - b.z;
    return vx * vx + vy * vy + vz * vz;
}

// The value at position `pos` of disarr[0, n) after plane_judge's exchange sort (:855-867).  A NaN never moves there
// (both comparisons with it are false), and the other values end up sorted descending in the remaining positions, as
// the same exchange sort of them alone would leave them.  So a NaN position reads NaN, and any other reads the r-th
// largest non-NaN value, r = the non-NaN positions before it.  Dista values are >= +0.0 or NaN, so their bit patterns
// order as the values; the r-th largest is found bit by bit.
// The largest, the smallest and the second smallest (the positions plane_judge reads in a group without NaN) take one
// pass; any other rank is found bit by bit.
FLB_HD double feat_sorted_at(const double* d, int n, int pos) {
    if (feat_isnan(d[pos])) return d[pos];
    int r = 0, cnt = 0;
    for (int j = 0; j < n; ++j) {
        const int ok = !feat_isnan(d[j]);
        r += j < pos ? ok : 0;
        cnt += ok;
    }
    if (r == 0 || r >= cnt - 2) {
        unsigned long long hi = 0ull, lo1 = ~0ull, lo2 = ~0ull;     // the max; the two smallest, with multiplicity
        for (int j = 0; j < n; ++j) {
            if (feat_isnan(d[j])) continue;
            const unsigned long long u = feat_d2u(d[j]);
            hi = u > hi ? u : hi;
            if (u < lo1) lo2 = lo1, lo1 = u;
            else if (u < lo2) lo2 = u;
        }
        return feat_u2d(r == 0 ? hi : r == cnt - 1 ? lo1 : lo2);
    }
    unsigned long long pre = 0ull;
    for (int bit = 62; bit >= 0; --bit) {
        const unsigned long long cand = pre | (1ull << bit);
        int cnt = 0;
        for (int j = 0; j < n; ++j) cnt += (!feat_isnan(d[j]) && feat_d2u(d[j]) >= cand) ? 1 : 0;
        if (cnt > r) pre = cand;
    }
    return feat_u2d(pre);
}

struct FeatStep {
    int type;            // kStepNonPlane, kStepPlane, kStepBlind
    int nex;             // i_nex on return; == m when a plane group reaches the line's last point
    float vx, vy, vz;    // the last (vx, vy, vz) of :815-817: exact float differences
};

// plane_judge (:786-898) for a point i with i + group_size < m (the caller's loop bound, :483).  The first loop pushes
// group_size values; the second runs at least once, so vx, vy, vz and two_dis are always this call's own.
FLB_HD FeatStep feat_plane_judge(const LidarPoint* pl, const double* rng, const double* dista, int m, int i, const FeatConst& c) {
    FeatStep s;
    s.type = kStepNonPlane, s.vx = s.vy = s.vz = 0.f;
    double group_dis = 0.1 * rng[i] + c.dis_b;                                    // disA = 0.1 (:13)
    group_dis = group_dis * group_dis;
    int nex;
    for (nex = i; nex < i + kFeatGroup; nex++)
        if (rng[nex] < c.blind) { s.type = kStepBlind, s.nex = nex; return s; }
    double vx = 0.0, vy = 0.0, vz = 0.0, two_dis = 0.0;
    for (;;) {
        if (i >= m || nex >= m) break;
        if (rng[nex] < c.blind) { s.type = kStepBlind, s.nex = nex; return s; }
        vx = pl[nex].x - pl[i].x;
        vy = pl[nex].y - pl[i].y;
        vz = pl[nex].z - pl[i].z;
        two_dis = vx * vx + vy * vy + vz * vz;
        if (two_dis >= group_dis) break;
        nex++;
    }
    s.nex = nex;
    double leng_wid = 0.0;
    for (int j = i + 1; j < nex; j++) {
        const double v1x = pl[j].x - pl[i].x, v1y = pl[j].y - pl[i].y, v1z = pl[j].z - pl[i].z;
        const double v2x = v1y * vz - vy * v1z, v2y = v1z * vx - v1x * vz, v2z = v1x * vy - vx * v1y;
        const double lw = v2x * v2x + v2y * v2y + v2z * v2z;
        if (lw > leng_wid) leng_wid = lw;
    }
    const int n = nex - i;                                                        // disarr = dista[i, nex)
    if ((two_dis * two_dis / leng_wid) < 225.0) return s;                         // p2l_ratio (:14)
    const double dlow = feat_sorted_at(dista + i, n, n - 2);
    if (dlow < 1e-16) return s;
    const double d0 = feat_sorted_at(dista + i, n, 0);
    if (c.avia) {
        const double dmid = feat_sorted_at(dista + i, n, n / 2);
        const double dismax_mid = d0 / dmid, dismid_min = dmid / dlow;
        if (dismax_mid >= 6.25 || dismid_min >= 6.25) return s;                    // limit_maxmid, limit_midmin
    } else {
        if (d0 / dlow >= 3.24) return s;                                           // limit_maxmin
    }
    s.type = kStepPlane;
    s.vx = (float)vx, s.vy = (float)vy, s.vz = (float)vz;
    return s;
}

// Eigen's Vector3d dot, norm and normalize as DESIGN §2 defines them: left to right, no FMA.
FLB_HD double feat_dot(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
FLB_HD void feat_normalize(float vx, float vy, float vz, double* v) {
    v[0] = vx, v[1] = vy, v[2] = vz;
    const double z = feat_dot(v, v);
    if (z > 0.0) {
        const double s = sqrt(z);
        v[0] /= s, v[1] /= s, v[2] /= s;
    }
}

// The ftype of point j after the plane loop (:493-590), given the visited steps: j's own step when j is visited, and
// p, the last visited point before j (-1: none).  A visited plane step writes [i, i_nex] (:506-516); consecutive plane
// steps share one endpoint, and the later step's write wins there.  last_state == 1 exactly when p is a plane step: a
// plane's i_nex is never within blind, so a blind step never follows one.
FLB_HD int feat_plane_ftype(int j, bool vis_j, const FeatStep& sj, int p, const FeatStep& sp) {
    const bool p_plane = p >= 0 && sp.type == kStepPlane;
    if (vis_j && sj.type == kStepPlane) {
        if (p_plane) {
            double last_direct[3], curr_direct[3];
            feat_normalize(sp.vx, sp.vy, sp.vz, last_direct);
            feat_normalize(sj.vx, sj.vy, sj.vz, curr_direct);
            if (sqrt(feat_dot(last_direct, last_direct)) > 0.1) {                 // :519
                const double mod = feat_dot(last_direct, curr_direct);
                return (mod > -0.707 && mod < 0.707) ? kFtEdgePlane : kFtRealPlane;
            }
        }
        return kFtPossPlane;
    }
    if (p_plane && sp.nex >= j) return j == sp.nex ? kFtPossPlane : kFtRealPlane;
    return kFtNor;
}

// edge_jump_judge (:900-936)
FLB_HD bool feat_edge_jump_judge(const double* rng, const double* dista, int i, int nor_dir, const FeatConst& c) {
    if (nor_dir == 0) {
        if (rng[i - 1] < c.blind || rng[i - 2] < c.blind) return false;
    } else {
        if (rng[i + 1] < c.blind || rng[i + 2] < c.blind) return false;
    }
    double d1 = dista[i + nor_dir - 1];
    double d2 = dista[i + 3 * nor_dir - 2];
    if (d1 < d2) {
        const double d = d1;
        d1 = d2, d2 = d;
    }
    d1 = sqrt(d1), d2 = sqrt(d2);
    if (d1 > 2.0 * d2 || (d1 - d2) > 0.1) return false;                        // edgea, edgeb
    return true;
}

struct FeatEdge {
    int ftype;
    double intersect;    // types[i].intersect: 2 (the constructor's) unless both neighbours were measured
};

// The edge pass for point i (:592-686); ftype is i's type after the plane loop.  Each point reads only its own type.
// When a neighbour is within blind its vecs[] entry is not computed and the reference's intersect reads stale stack
// memory; intersect is then used by neither this pass nor the small-plane pass (which skips a blind neighbour), so it
// is recorded as 2.
FLB_HD FeatEdge feat_edge(const LidarPoint* pl, const double* rng, const double* dista, int m, int head, int i, int ftype,
                          const FeatConst& c) {
    FeatEdge e;
    e.ftype = ftype, e.intersect = 2.0;
    const int plsize2 = m > 3 ? m - 3 : 0;
    if (i < head + 3 || i >= plsize2) return e;
    if (rng[i] < c.blind || ftype >= kFtRealPlane) return e;
    if (dista[i - 1] < 1e-16 || dista[i] < 1e-16) return e;
    const double vec_a[3] = {(double)pl[i].x, (double)pl[i].y, (double)pl[i].z};
    double vecs[2][3];
    int edj[2] = {kNrNor, kNrNor};
    bool both = true;
    for (int j = 0; j < 2; j++) {
        const int k = j == 1 ? i + 1 : i - 1;
        if (rng[k] < c.blind) {
            edj[j] = rng[i] > 10.0 ? kNrInf : kNrBlind;                             // inf_bound (:9)
            both = false;
            continue;
        }
        vecs[j][0] = (double)pl[k].x - vec_a[0];
        vecs[j][1] = (double)pl[k].y - vec_a[1];
        vecs[j][2] = (double)pl[k].z - vec_a[2];
        const double angle = feat_dot(vec_a, vecs[j]) / sqrt(feat_dot(vec_a, vec_a)) / sqrt(feat_dot(vecs[j], vecs[j]));
        if (angle < c.jump_up) edj[j] = kNr180;
        else if (angle > c.jump_down) edj[j] = kNrZero;
    }
    if (both) e.intersect = feat_dot(vecs[0], vecs[1]) / sqrt(feat_dot(vecs[0], vecs[0])) / sqrt(feat_dot(vecs[1], vecs[1]));
    const double di = dista[i], dp = dista[i - 1];
    if (edj[0] == kNrNor && edj[1] == kNrZero && di > 0.0225 && di > 4 * dp) {
        if (e.intersect > c.cos160 && feat_edge_jump_judge(rng, dista, i, 0, c)) e.ftype = kFtEdgeJump;
    } else if (edj[0] == kNrZero && edj[1] == kNrNor && dp > 0.0225 && dp > 4 * di) {
        if (e.intersect > c.cos160 && feat_edge_jump_judge(rng, dista, i, 1, c)) e.ftype = kFtEdgeJump;
    } else if (edj[0] == kNrNor && edj[1] == kNrInf) {
        if (feat_edge_jump_judge(rng, dista, i, 0, c)) e.ftype = kFtEdgeJump;
    } else if (edj[0] == kNrInf && edj[1] == kNrNor) {
        if (feat_edge_jump_judge(rng, dista, i, 1, c)) e.ftype = kFtEdgeJump;
    } else if (edj[0] > kNrNor && edj[1] > kNrNor) {
        if (e.ftype == kFtNor) e.ftype = kFtWire;
    }
    return e;
}

// The small-plane pass (:688-726): iteration i would fire on the types the edge pass left (ftype, intersect).
// Iteration i-1 changes ftype[i] only when it fires, so fire(i) = small_cond(i) && !fire(i-1): along a run of
// consecutive conditions the firing alternates from the run's first point.
FLB_HD bool feat_small_cond(const double* rng, const double* dista, int m, int head, int i, int ftype, double intersect,
                            const FeatConst& c) {
    if (i < head + 1 || i >= m - 1) return false;
    if (rng[i] < c.blind || rng[i - 1] < c.blind || rng[i + 1] < c.blind) return false;
    if (dista[i - 1] < 1e-8 || dista[i] < 1e-8) return false;
    if (ftype != kFtNor) return false;
    const double ratio = dista[i - 1] > dista[i] ? dista[i - 1] / dista[i] : dista[i] / dista[i - 1];
    return intersect < c.smallp_intersect && ratio < 1.2;                          // smallp_ratio (:24)
}
FLB_HD bool feat_is_surf(int ftype) { return ftype == kFtPossPlane || ftype == kFtRealPlane; }

// ---- the parallel formulation: one function per kernel, over the global line-major index q ----------------------
// lbeg / lend: each line's segment (0 / 0 when empty); lhead: the first point not within blind (INT_MAX: none).
struct FeatLine { int b, m, head; };   // head == m: the line yields nothing (skipped by its size, or all within blind)
FLB_HD FeatLine feat_line(const int* lbeg, const int* lend, const int* lhead, int k, int min_size) {
    FeatLine L;
    L.b = lbeg[k], L.m = lend[k] - lbeg[k];
    L.head = (L.m < min_size || lhead[k] >= lend[k]) ? L.m : lhead[k] - L.b;
    return L;
}
FLB_HD int feat_plsize2(const FeatLine& L) { return L.m > kFeatGroup ? L.m - kFeatGroup : 0; }

// The step of the plane loop (:493-590) that would start at q.  A step depends on its own i alone, never on the walk
// that reaches it.
FLB_HD FeatStep feat_step_at(const LidarPoint* P, const double* rng, const double* dista, const FeatLine& L, int q,
                             const FeatConst& c) {
    const int j = q - L.b;
    FeatStep s;
    s.type = kStepNone, s.nex = j, s.vx = s.vy = s.vz = 0.f;
    if (j < L.head || j >= feat_plsize2(L)) return s;
    if (rng[q] < c.blind) {
        s.type = kStepSkip;
        return s;
    }
    return feat_plane_judge(P + L.b, rng + L.b, dista + L.b, L.m, j, c);
}
// The next point the loop visits after the step s at q: i_nex for a plane, i_nex + 1 otherwise, i + 1 for a blind i;
// -1 for no step, or once that leaves the loop's range.
FLB_HD int feat_succ(const FeatStep& s, const FeatLine& L, int q) {
    if (s.type == kStepNone) return -1;
    const int nx = s.type == kStepSkip ? q - L.b + 1 : s.type == kStepPlane ? s.nex : s.nex + 1;
    return nx < feat_plsize2(L) ? L.b + nx : -1;
}

// ftype after the plane loop and the edge pass for point q.  vis: q is visited; p: the last visited point before q
// (global, -1 or outside the line: none).
FLB_HD FeatEdge feat_types_at(const LidarPoint* P, const double* rng, const double* dista, const FeatLine& L, int q, bool vis,
                              const FeatStep& sq, int p, const FeatStep& sp, const FeatConst& c) {
    const int j = q - L.b;
    const int pj = p >= L.b ? p - L.b : -1;
    const int ft = feat_plane_ftype(j, vis, sq, pj, sp);
    return feat_edge(P + L.b, rng + L.b, dista + L.b, L.m, L.head, j, ft, c);
}

// The type after the small-plane pass: fire(x) = small(x) && x is an even distance from its run's start (rs[x]).
FLB_HD bool feat_fire(const unsigned char* small, const int* rs, int M, int x) {
    return x >= 0 && x < M && small[x] && ((x - rs[x]) & 1) == 0;
}
FLB_HD int feat_final_at(const int* ft_edge, const unsigned char* small, const int* rs, int M, int q) {
    const int ft = ft_edge[q];
    if (ft == kFtNor && (feat_fire(small, rs, M, q - 1) || feat_fire(small, rs, M, q) || feat_fire(small, rs, M, q + 1)))
        return kFtRealPlane;
    return ft;
}

// The surface output (:728-774) at q: runs of Poss_Plane / Real_Plane from head on, cut into chunks of filter_num from
// the run's start (rs2 = that start).  A full chunk emits its last point; a partial one the float mean of its points,
// in index order, at the non-surface point that closes it; a partial one at the line's end is dropped.
FLB_HD bool feat_emit_at(const LidarPoint* P, const int* ft_final, const int* rs2, const FeatLine& L, int q, int filter_num,
                         LidarPoint* out) {
    const int j = q - L.b;
    if (j < L.head || j >= L.m) return false;
    if (feat_is_surf(ft_final[q])) {
        if ((q - rs2[q]) % filter_num != filter_num - 1) return false;
        *out = P[q];
        return true;
    }
    if (j == L.head || !feat_is_surf(ft_final[q - 1])) return false;
    const int len = q - rs2[q - 1], r = len % filter_num;
    if (r == 0) return false;
    LidarPoint ap;
    ap.x = ap.y = ap.z = ap.t = 0.f;
    for (int k = q - r; k < q; k++) ap.x += P[k].x, ap.y += P[k].y, ap.z += P[k].z, ap.t += P[k].t;
    const float d = (float)(unsigned)r;
    ap.x /= d, ap.y /= d, ap.z /= d, ap.t /= d;
    *out = ap;
    return true;
}

// ------------------------------------------------------------------ display_keypatch (src/lidar_selection.cpp:985-1005)
// One pixel coordinate of a circle's centre: cv::Point2f rounds the double to float, cv::circle's cv::Point takes
// cvRound of that float (half to even, as x86-64's cvtss2si does).  false, and nothing is drawn, for a non-finite
// coordinate or one that rounds beyond +-2^30: cvRound gives INT_MIN there and OpenCV's clipping overflows, so this
// is a definition, not the reference's behaviour.  Floats are integers from 2^23 on, so the bound holds for the float.
FLB_HD bool keypatch_round(double v, int* out) {
    const float f = (float)v;
    if (!(fabsf(f) <= 1073741824.f)) return false;
    *out = (int)rintf(f);
    return true;
}
// The centre of patch position pos: new_frame_->w2c(pos) = world2cam(Rcw * pos + Pcw), then keypatch_round.
FLB_HD bool keypatch_center(const CamModel& cam, const double* Rcw, const double* Pcw, const double* pos, int* cx, int* cy) {
    double pf[3], pc[2];
    se3_apply(Rcw, Pcw, pos, pf);
    world2cam(cam, pf, pc);
    return keypatch_round(pc[0], cx) && keypatch_round(pc[1], cy);
}
// cv::circle(img, c, 6, colour, FILLED, LINE_8) with no shift: 113 pixels, rows 1 7 9 11 11 11 13 11 11 11 9 7 1 wide
// (half-widths 6 5 5 5 4 3 0 by |dy|), clipped to the image and nothing else.
constexpr int kKeypatchRadius = 6;
FLB_HD bool keypatch_in_disk(int dx, int dy) {
    const int ax = dx < 0 ? -dx : dx, ay = dy < 0 ? -dy : dy;
    const int hw = ay == 0 ? 6 : ay <= 3 ? 5 : ay == 4 ? 4 : ay == 5 ? 3 : ay == 6 ? 0 : -1;
    return ax <= hw;
}
// errors[i] < 8000 (float compare): green; otherwise, NaN included, cv::Scalar(255, 0, 0), i.e. blue.  BGR bytes.
FLB_HD void keypatch_colour(float err, unsigned char* bgr) {
    const bool green = err < 8000.f;
    bgr[0] = green ? 0 : 255;
    bgr[1] = green ? 255 : 0;
    bgr[2] = 0;
}

}  // namespace flb
