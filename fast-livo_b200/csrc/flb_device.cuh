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
struct GridDesc {
    float ox, oy, oz;     // origin (min corner)
    float cell, inv_cell;
    int nx, ny, nz;       // cells per axis; cell id = (z*ny + y)*nx + x  (x fastest)
    float max_d2;         // 5.0
    int max_ring;         // ceil(sqrt(max_d2)/cell) + 1
};

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
FLB_HD void knn5_grid(const GridDesc& g, const int* __restrict__ cell_start, const map_pt* __restrict__ pts,
                      float qx, float qy, float qz, Top5& t, int* rows, int rstride) {
    // rows: per-thread scratch for 18 ints, element k at rows[k * rstride] (shared memory on the device,
    // one column per thread, so a warp's accesses are conflict-free)
    top5_init(t);
    const float fx = (qx - g.ox) * g.inv_cell, fy = (qy - g.oy) * g.inv_cell, fz = (qz - g.oz) * g.inv_cell;
    // far outside the grid: nothing within sqrt(max_d2)
    const float lim = (float)(g.max_ring + 2);
    if (!(fx > -lim && fy > -lim && fz > -lim && fx < (float)g.nx + lim && fy < (float)g.ny + lim &&
          fz < (float)g.nz + lim))
        return;
    const int cx = (int)floorf(fx), cy = (int)floorf(fy), cz = (int)floorf(fz);
    float mx = fminf(fx - (float)cx, (float)(cx + 1) - fx);
    float my = fminf(fy - (float)cy, (float)(cy + 1) - fy);
    float mz = fminf(fz - (float)cz, (float)(cz + 1) - fz);
    const float margin = fmaxf(fminf(mx, fminf(my, mz)) * g.cell - 1e-3f * g.cell, 0.f);
    {
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
        knn_walk_runs(pts, rows, rstride, 9, qx, qy, qz, t);
        const float bound = g.cell + margin;
        const float b2 = bound * bound;
        if (t.d[4] <= b2) return;                 // 5th best is certainly final
        if (b2 > g.max_d2 * 1.0001f) return;      // everything unscanned is beyond max_d2
    }
    for (int r = 2; r <= g.max_ring; ++r) {
        const int z0 = cz - r, z1 = cz + r, y0 = cy - r, y1 = cy + r, x0 = cx - r, x1 = cx + r;
        const int xa = x0 < 0 ? 0 : x0, xb = x1 >= g.nx ? g.nx - 1 : x1;
        int cnt = 0;
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

}  // namespace flb
