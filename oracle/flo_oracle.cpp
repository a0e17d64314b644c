// TEST INFRASTRUCTURE -- NOT PRODUCT CODE.  See flo_oracle.h for the rules on who
// may load this library.  "parity unpinned": the reference has no tests and its
// node cannot be built in this image; every function below follows the cited
// reference lines (paths relative to the reference tree, hku-mars/FAST-LIVO @ dcebf84) op for op.
//
// Build: oracle/Makefile (g++ -std=c++17 -O3 -fopenmp -ffp-contract=off, no
// -march=native: mirrors reference CMakeLists.txt:8,39-41; x86-64 baseline has
// no FMA so float/double expressions round exactly as written).
#include "flo_oracle.h"

#include <omp.h>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

namespace {

constexpr int kMatch = 5;  // NUM_MATCH_POINTS, include/common_lib.h:39
constexpr int kDim = 18;   // DIM_STATE, include/common_lib.h:34

// ---------- tiny dense helpers (row-major 3x3, double) ------------------------
inline void mat3_mul(const double* A, const double* B, double* C) {  // C = A*B
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            C[3 * i + j] = A[3 * i + 0] * B[0 + j] + A[3 * i + 1] * B[3 + j] + A[3 * i + 2] * B[6 + j];
}
inline void mat3_T(const double* A, double* T) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[3 * i + j] = A[3 * j + i];
}
inline void mat3_vec(const double* A, const double* v, double* o) {
    for (int i = 0; i < 3; ++i) o[i] = A[3 * i + 0] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2];
}
// SKEW_SYM_MATRX, include/so3_math.h:9
inline void skew(const double* v, double* K) {
    K[0] = 0.0;   K[1] = -v[2]; K[2] = v[1];
    K[3] = v[2];  K[4] = 0.0;   K[5] = -v[0];
    K[6] = -v[1]; K[7] = v[0];  K[8] = 0.0;
}

// PartialPivLU-based inverse (Eigen's inverse() for sizes > 4, SURVEY App. C).
int inverse_lu(const double* Ain, int n, double* Ainv) {
    std::vector<double> A(Ain, Ain + (size_t)n * n);
    std::vector<int> perm(n);
    for (int i = 0; i < n; ++i) perm[i] = i;
    for (int k = 0; k < n; ++k) {
        int piv = k;
        double best = std::fabs(A[(size_t)k * n + k]);
        for (int i = k + 1; i < n; ++i) {
            double v = std::fabs(A[(size_t)i * n + k]);
            if (v > best) { best = v; piv = i; }
        }
        if (best == 0.0) return -1;
        if (piv != k) {
            for (int j = 0; j < n; ++j) std::swap(A[(size_t)k * n + j], A[(size_t)piv * n + j]);
            std::swap(perm[k], perm[piv]);
        }
        const double d = A[(size_t)k * n + k];
        for (int i = k + 1; i < n; ++i) {
            const double l = A[(size_t)i * n + k] / d;
            A[(size_t)i * n + k] = l;
            for (int j = k + 1; j < n; ++j) A[(size_t)i * n + j] -= l * A[(size_t)k * n + j];
        }
    }
    // Solve L U X = P I column by column.
    std::vector<double> y(n);
    for (int c = 0; c < n; ++c) {
        for (int i = 0; i < n; ++i) {
            double s = (perm[i] == c) ? 1.0 : 0.0;
            for (int j = 0; j < i; ++j) s -= A[(size_t)i * n + j] * y[j];
            y[i] = s;
        }
        for (int i = n - 1; i >= 0; --i) {
            double s = y[i];
            for (int j = i + 1; j < n; ++j) s -= A[(size_t)i * n + j] * Ainv[(size_t)j * n + c];
            Ainv[(size_t)i * n + c] = s / A[(size_t)i * n + i];
        }
    }
    return 0;
}

// The shared 18-DoF iterated-EKF step, src/laserMapping.cpp:1664-1683 (LIO) and
// src/lidar_selection.cpp:871-880 (VIO; sign = -1 on the K*HTz term).
//   K1 = (H_T_H + (cov/sigma)^-1)^-1 ; G[:, :6] = K1[:, :6]*HTH6
//   solution = sign*K1[:, :6]*HTz + vec - G[:, :6]*vec[:6] ; x += solution
void ekf18_step(flo_state18* x, const flo_state18* x_prop, const double* HTH6, const double* HTz6,
                double sigma, double sign, double* G /*18x18*/, double* solution /*18*/) {
    double HTH18[kDim * kDim] = {0};
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) HTH18[i * kDim + j] = HTH6[i * 6 + j];
    double Ps[kDim * kDim], Pinv[kDim * kDim], S[kDim * kDim], K1[kDim * kDim];
    for (int i = 0; i < kDim * kDim; ++i) Ps[i] = x->cov[i] / sigma;
    inverse_lu(Ps, kDim, Pinv);
    for (int i = 0; i < kDim * kDim; ++i) S[i] = HTH18[i] + Pinv[i];
    inverse_lu(S, kDim, K1);
    std::memset(G, 0, sizeof(double) * kDim * kDim);
    for (int i = 0; i < kDim; ++i)
        for (int j = 0; j < 6; ++j) {
            double s = 0.0;
            for (int k = 0; k < 6; ++k) s += K1[i * kDim + k] * HTH6[k * 6 + j];
            G[i * kDim + j] = s;
        }
    double vec[kDim];
    flo_state_boxminus(x_prop, x, vec);
    for (int i = 0; i < kDim; ++i) {
        double kz = 0.0, gv = 0.0;
        for (int k = 0; k < 6; ++k) {
            kz += K1[i * kDim + k] * HTz6[k];
            gv += G[i * kDim + k] * vec[k];
        }
        solution[i] = sign * kz + vec[i] - gv;
    }
    flo_state_boxplus(x, solution);
}

inline double norm3(const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

}  // namespace

extern "C" {

// ---------------------------------------------------------------------------------
// so3_math.h:54-72  Exp(v1,v2,v3)
void flo_exp3(const double v[3], double R[9]) {
    const double norm = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (norm > 0.00001) {
        const double r[3] = {v[0] / norm, v[1] / norm, v[2] / norm};
        double K[9], KK[9];
        skew(r, K);
        mat3_mul(K, K, KK);
        const double s = std::sin(norm), c1 = 1.0 - std::cos(norm);
        for (int i = 0; i < 9; ++i) R[i] = R[i] + s * K[i] + c1 * KK[i];
    }
}

// so3_math.h:75-81  Log(R)
void flo_log3(const double R[9], double out[3]) {
    const double tr = R[0] + R[4] + R[8];
    const double theta = (tr > 3.0 - 1e-6) ? 0.0 : std::acos(0.5 * (tr - 1));
    const double K[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    if (std::fabs(theta) < 0.001) {
        for (int i = 0; i < 3; ++i) out[i] = 0.5 * K[i];
    } else {
        const double f = 0.5 * theta / std::sin(theta);
        for (int i = 0; i < 3; ++i) out[i] = f * K[i];
    }
}

// common_lib.h:343-352  StatesGroup::operator+=
void flo_state_boxplus(flo_state18* x, const double d[18]) {
    double E[9], Rn[9];
    flo_exp3(d, E);
    mat3_mul(x->rot, E, Rn);
    std::memcpy(x->rot, Rn, sizeof(Rn));
    for (int i = 0; i < 3; ++i) {
        x->pos[i] += d[3 + i];
        x->vel[i] += d[6 + i];
        x->bg[i] += d[9 + i];
        x->ba[i] += d[12 + i];
        x->grav[i] += d[15 + i];
    }
}

// common_lib.h:354-365  StatesGroup::operator-  (a - b)
void flo_state_boxminus(const flo_state18* a, const flo_state18* b, double out[18]) {
    double bT[9], rotd[9];
    mat3_T(b->rot, bT);
    mat3_mul(bT, a->rot, rotd);
    flo_log3(rotd, out);
    for (int i = 0; i < 3; ++i) {
        out[3 + i] = a->pos[i] - b->pos[i];
        out[6 + i] = a->vel[i] - b->vel[i];
        out[9 + i] = a->bg[i] - b->bg[i];
        out[12 + i] = a->ba[i] - b->ba[i];
        out[15 + i] = a->grav[i] - b->grav[i];
    }
}

int flo_inverse(const double* A, int n, double* Ainv) { return inverse_lu(A, n, Ainv); }

// ---------------------------------------------------------------------------------
// Brute-force exact kNN with the reference's float32 distance
// (ikd_Tree.cpp:1291-1295: (dx*dx + dy*dy) + dz*dz, left to right), strict `<`
// acceptance (ikd_Tree.cpp:860) and ascending output order (ikd_Tree.cpp:374-378).
struct BruteCtx {
    std::vector<float> xyz;
    int M;
};

void* flo_knn_brute_ctx(const float* map_xyz, int M) {
    BruteCtx* c = new BruteCtx;
    c->xyz.assign(map_xyz, map_xyz + (size_t)3 * M);
    c->M = M;
    return c;
}
void flo_free(void* p) { delete static_cast<BruteCtx*>(p); }

int flo_knn_brute(void* map_ctx, const float* q, int nq, int k, int* idx, float* d2, int nthreads) {
    const BruteCtx* c = static_cast<const BruteCtx*>(map_ctx);
    if (k > 16) return -1;
    omp_set_num_threads(nthreads < 1 ? 1 : nthreads);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < nq; ++i) {
        float bd[16];
        int bi[16];
        for (int j = 0; j < k; ++j) { bd[j] = std::numeric_limits<float>::infinity(); bi[j] = -1; }
        const float qx = q[3 * (size_t)i], qy = q[3 * (size_t)i + 1], qz = q[3 * (size_t)i + 2];
        for (int m = 0; m < c->M; ++m) {
            const float dx = qx - c->xyz[3 * (size_t)m], dy = qy - c->xyz[3 * (size_t)m + 1],
                        dz = qz - c->xyz[3 * (size_t)m + 2];
            const float d = dx * dx + dy * dy + dz * dz;
            if (d < bd[k - 1]) {
                int j = k - 1;
                while (j > 0 && d < bd[j - 1]) { bd[j] = bd[j - 1]; bi[j] = bi[j - 1]; --j; }
                bd[j] = d;
                bi[j] = m;
            }
        }
        for (int j = 0; j < k; ++j) { idx[(size_t)i * k + j] = bi[j]; d2[(size_t)i * k + j] = bd[j]; }
    }
    return 0;
}

// ---------------------------------------------------------------------------------
// esti_plane<float>, include/common_lib.h:448-493.
//
// The reference solves A(5x3) x = -1 with Eigen's colPivHouseholderQr().solve().
// Eigen is not in this image and its fixed-size float reductions are
// SSE-packet-ordered, so THIS FUNCTION DEFINES the float32 operation order
// (SURVEY.md Appendix C: the one place where "reference parity" means "oracle
// parity"): plain left-to-right sums, no FMA; Eigen 3.3/3.4's algorithm --
// column norms, pivot on the largest updated norm, Householder
// (beta = -sign(c0)*sqrt(c0^2+|tail|^2), essential = tail/(c0-beta),
// tau = (beta-c0)/beta), LAPACK-WN176 norm down-dating, rank cut-off, c = Q^T b,
// column-oriented back-substitution, un-permute.
int flo_esti_plane(const float nb[15], float threshold, float pabcd[4]) {
    const int rows = kMatch, cols = 3;
    float qr[kMatch][3];
    for (int j = 0; j < rows; ++j)
        for (int c = 0; c < cols; ++c) qr[j][c] = nb[3 * j + c];
    float hcoef[3];
    int colidx[3] = {0, 1, 2};
    float normsUpdated[3], normsDirect[3];
    for (int c = 0; c < cols; ++c) {
        float s = 0.f;
        for (int j = 0; j < rows; ++j) s = s + qr[j][c] * qr[j][c];
        normsDirect[c] = normsUpdated[c] = std::sqrt(s);
    }
    const float eps = std::numeric_limits<float>::epsilon();
    float maxnorm = normsUpdated[0];
    for (int c = 1; c < cols; ++c) if (normsUpdated[c] > maxnorm) maxnorm = normsUpdated[c];
    const float th0 = maxnorm * eps;
    const float threshold_helper = (th0 * th0) / float(rows);
    const float norm_downdate_threshold = std::sqrt(eps);
    int nonzero_pivots = cols;
    for (int k = 0; k < cols; ++k) {
        int big = k;
        float bigv = normsUpdated[k];
        for (int c = k + 1; c < cols; ++c) if (normsUpdated[c] > bigv) { bigv = normsUpdated[c]; big = c; }
        const float big_sq = bigv * bigv;
        if (nonzero_pivots == cols && big_sq < threshold_helper * float(rows - k)) nonzero_pivots = k;
        if (big != k) {
            for (int j = 0; j < rows; ++j) std::swap(qr[j][k], qr[j][big]);
            std::swap(normsUpdated[k], normsUpdated[big]);
            std::swap(normsDirect[k], normsDirect[big]);
            std::swap(colidx[k], colidx[big]);
        }
        // makeHouseholderInPlace on qr[k..rows-1][k]
        float tailSq = 0.f;
        for (int j = k + 1; j < rows; ++j) tailSq = tailSq + qr[j][k] * qr[j][k];
        const float c0 = qr[k][k];
        float beta, tau;
        if (tailSq <= std::numeric_limits<float>::min()) {
            tau = 0.f;
            beta = c0;
            for (int j = k + 1; j < rows; ++j) qr[j][k] = 0.f;
        } else {
            beta = std::sqrt(c0 * c0 + tailSq);
            if (c0 >= 0.f) beta = -beta;
            const float den = c0 - beta;
            for (int j = k + 1; j < rows; ++j) qr[j][k] = qr[j][k] / den;
            tau = (beta - c0) / beta;
        }
        qr[k][k] = beta;
        hcoef[k] = tau;
        // applyHouseholderOnTheLeft to the trailing columns
        if (tau != 0.f) {
            for (int c = k + 1; c < cols; ++c) {
                float tmp = 0.f;
                for (int j = k + 1; j < rows; ++j) tmp = tmp + qr[j][k] * qr[j][c];
                tmp = tmp + qr[k][c];
                qr[k][c] = qr[k][c] - tau * tmp;
                for (int j = k + 1; j < rows; ++j) qr[j][c] = qr[j][c] - (tau * qr[j][k]) * tmp;
            }
        }
        // column-norm down-date
        for (int c = k + 1; c < cols; ++c) {
            if (normsUpdated[c] != 0.f) {
                float temp = std::fabs(qr[k][c]) / normsUpdated[c];
                temp = (1.f + temp) * (1.f - temp);
                temp = temp < 0.f ? 0.f : temp;
                const float ratio = normsUpdated[c] / normsDirect[c];
                const float temp2 = temp * (ratio * ratio);
                if (temp2 <= norm_downdate_threshold) {
                    float s = 0.f;
                    for (int j = k + 1; j < rows; ++j) s = s + qr[j][c] * qr[j][c];
                    normsDirect[c] = std::sqrt(s);
                    normsUpdated[c] = normsDirect[c];
                } else {
                    normsUpdated[c] = normsUpdated[c] * std::sqrt(temp);
                }
            }
        }
    }
    // solve: c = Q^T b, b = -1
    float cvec[kMatch];
    for (int j = 0; j < rows; ++j) cvec[j] = -1.0f;
    float x[3] = {0.f, 0.f, 0.f};
    if (nonzero_pivots > 0) {
        for (int k = 0; k < nonzero_pivots; ++k) {
            const float tau = hcoef[k];
            if (tau != 0.f) {
                float tmp = 0.f;
                for (int j = k + 1; j < rows; ++j) tmp = tmp + qr[j][k] * cvec[j];
                tmp = tmp + cvec[k];
                cvec[k] = cvec[k] - tau * tmp;
                for (int j = k + 1; j < rows; ++j) cvec[j] = cvec[j] - (tau * qr[j][k]) * tmp;
            }
        }
        for (int i = nonzero_pivots - 1; i >= 0; --i) {
            cvec[i] = cvec[i] / qr[i][i];
            for (int r = 0; r < i; ++r) cvec[r] = cvec[r] - cvec[i] * qr[r][i];
        }
        for (int i = 0; i < nonzero_pivots; ++i) x[colidx[i]] = cvec[i];
    }
    // common_lib.h:465-469
    const float n = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    pabcd[0] = x[0] / n;
    pabcd[1] = x[1] / n;
    pabcd[2] = x[2] / n;
    pabcd[3] = (float)(1.0 / (double)n);  // `1.0 / n` is a double expression in the reference
    // common_lib.h:471-477
    for (int j = 0; j < rows; ++j) {
        const float v = pabcd[0] * nb[3 * j] + pabcd[1] * nb[3 * j + 1] + pabcd[2] * nb[3 * j + 2] + pabcd[3];
        if (!(std::fabs(v) <= threshold)) return 0;  // `fabs(..) > threshold` -> false; NaN also rejects
    }
    return 1;
}

}  // extern "C"

// =================================================================================
// LIO
// =================================================================================
struct flo_lio {
    std::vector<float> map;   // M x 3
    int M = 0;
    std::vector<float> body;  // N x 3 (feats_down_body)
    int N = 0;
    flo_knn_fn knn = nullptr;
    void* knn_ctx = nullptr;
    void* own_ctx = nullptr;
    // per-point persistent arrays (laserMapping.cpp:140-151)
    std::vector<int> nn_idx;        // Nearest_Points as indices, N x 5
    std::vector<float> nn_d2;
    std::vector<uint8_t> selected;  // point_selected_surf
    std::vector<double> res_last;
    std::vector<float> normvec;     // N x 4 (x,y,z,intensity=pd2)
    std::vector<float> world;       // feats_down_world
};

extern "C" {

flo_lio* flo_lio_create(const float* map_xyz, int M, const float* scan_body_xyz, int N, flo_knn_fn knn,
                        void* knn_ctx) {
    flo_lio* L = new flo_lio;
    L->map.assign(map_xyz, map_xyz + (size_t)3 * M);
    L->M = M;
    L->body.assign(scan_body_xyz, scan_body_xyz + (size_t)3 * N);
    L->N = N;
    if (knn) {
        L->knn = knn;
        L->knn_ctx = knn_ctx;
    } else {
        L->own_ctx = flo_knn_brute_ctx(map_xyz, M);
        L->knn = flo_knn_brute;
        L->knn_ctx = L->own_ctx;
    }
    L->nn_idx.assign((size_t)N * kMatch, -1);
    L->nn_d2.assign((size_t)N * kMatch, std::numeric_limits<float>::infinity());
    L->selected.assign(N, 1);        // point_selected_surf.resize(N, true), :1469
    L->res_last.assign(N, 1000.0);   // res_last.resize(N, 1000.0), :1441
    L->normvec.assign((size_t)N * 4, 0.f);
    L->world.assign((size_t)N * 3, 0.f);
    return L;
}

void flo_lio_reset(flo_lio* L) {
    std::fill(L->selected.begin(), L->selected.end(), 1);
    std::fill(L->res_last.begin(), L->res_last.end(), 1000.0);
}

void flo_lio_destroy(flo_lio* L) {
    if (!L) return;
    if (L->own_ctx) flo_free(L->own_ctx);
    delete L;
}

int flo_lio_pass(flo_lio* L, const flo_lio_params* prm, const double R[9], const double p[3], int rematch,
                 float* world_xyz, int* nn_idx_out, float* nn_d2_out, float* pabcd_out, float* pd2_out,
                 uint8_t* selected_out, double* Hsub, double* h_x, double* meas, int* sel_idx,
                 double* HTH6, double* HTz6, double* HTH12, double* HTh12, double* total_residual_out) {
    const int N = L->N;
    const int nthreads = prm->nthreads < 1 ? 1 : prm->nthreads;
    omp_set_num_threads(nthreads);

    // pointBodyToWorld, laserMapping.cpp:272-286 / :1527: double math, float store.
#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        const double pb[3] = {L->body[3 * (size_t)i], L->body[3 * (size_t)i + 1], L->body[3 * (size_t)i + 2]};
        double pI[3], pw[3];
        mat3_vec(prm->R_LI, pb, pI);
        for (int k = 0; k < 3; ++k) pI[k] = pI[k] + prm->t_LI[k];
        mat3_vec(R, pI, pw);
        for (int k = 0; k < 3; ++k) L->world[3 * (size_t)i + k] = (float)(pw[k] + p[k]);
    }

    if (rematch) {
        // ikdtree.Nearest_Search(point_world, 5, ...), :1543
        L->knn(L->knn_ctx, L->world.data(), N, kMatch, L->nn_idx.data(), L->nn_d2.data(), nthreads);
    }

#pragma omp parallel for schedule(static)
    for (int i = 0; i < N; ++i) {
        const size_t i5 = (size_t)i * kMatch;
        if (rematch) {
            // :1549 (and :1567's size check: fewer than 5 neighbours -> never selected)
            const bool five = L->nn_idx[i5 + kMatch - 1] >= 0;
            L->selected[i] = (five && !(L->nn_d2[i5 + kMatch - 1] > 5)) ? 1 : 0;
        }
        if (!L->selected[i] || L->nn_idx[i5 + kMatch - 1] < 0) continue;  // :1567
        L->selected[i] = 0;                                                // :1570
        float nb[15];
        for (int j = 0; j < kMatch; ++j)
            for (int c = 0; c < 3; ++c) nb[3 * j + c] = L->map[3 * (size_t)L->nn_idx[i5 + j] + c];
        float pabcd[4];
        const int ok = flo_esti_plane(nb, 0.1f, pabcd);                    // :1571
        if (pabcd_out) std::memcpy(pabcd_out + 4 * (size_t)i, pabcd, sizeof(pabcd));
        if (ok) {
            const float* w = &L->world[3 * (size_t)i];
            const float pd2 = pabcd[0] * w[0] + pabcd[1] * w[1] + pabcd[2] * w[2] + pabcd[3];  // :1573
            const double pb[3] = {L->body[3 * (size_t)i], L->body[3 * (size_t)i + 1], L->body[3 * (size_t)i + 2]};
            const float s = (float)(1 - 0.9 * std::fabs(pd2) / std::sqrt(norm3(pb)));  // :1574
            if (s > 0.9) {                                                              // :1576
                L->selected[i] = 1;
                L->normvec[4 * (size_t)i + 0] = pabcd[0];
                L->normvec[4 * (size_t)i + 1] = pabcd[1];
                L->normvec[4 * (size_t)i + 2] = pabcd[2];
                L->normvec[4 * (size_t)i + 3] = pd2;
                L->res_last[i] = std::fabs(pd2);                                        // :1583
            }
        }
    }

    // serial compaction, :1588-1602 (heap-allocated per pass like the reference)
    std::vector<int> ori;
    ori.reserve(N);
    double total_residual = 0.0;
    for (int i = 0; i < N; ++i) {
        if (L->selected[i] && (L->res_last[i] <= 2.0)) {
            ori.push_back(i);
            total_residual += L->res_last[i];
        }
    }
    const int n = (int)ori.size();
    if (total_residual_out) *total_residual_out = total_residual;

    // rows, :1608-1629 (live) and :1059-1089 (IKFoM layout)
    std::vector<double> Hloc((size_t)n * 6), zloc(n), H12;
    const bool want12 = h_x || HTH12 || HTh12;
    if (want12) H12.resize((size_t)n * 12);
    double Rt[9], RLIt[9];
    mat3_T(R, Rt);
    mat3_T(prm->R_LI, RLIt);
    for (int k = 0; k < n; ++k) {
        const int i = ori[k];
        const double pb[3] = {L->body[3 * (size_t)i], L->body[3 * (size_t)i + 1], L->body[3 * (size_t)i + 2]};
        double pI[3];
        mat3_vec(prm->R_LI, pb, pI);
        for (int c = 0; c < 3; ++c) pI[c] = pI[c] + prm->t_LI[c];
        double cross[9], M1[9], A[3];
        skew(pI, cross);
        const double nv[3] = {L->normvec[4 * (size_t)i], L->normvec[4 * (size_t)i + 1], L->normvec[4 * (size_t)i + 2]};
        mat3_mul(cross, Rt, M1);   // point_crossmat * rot_end^T   (:1624, evaluated left to right)
        mat3_vec(M1, nv, A);
        double* h = &Hloc[(size_t)k * 6];
        h[0] = A[0]; h[1] = A[1]; h[2] = A[2];
        h[3] = nv[0]; h[4] = nv[1]; h[5] = nv[2];
        zloc[k] = -(double)L->normvec[4 * (size_t)i + 3];  // :1628
        if (want12) {
            // C = R^T n ; A = [p_I]x C ; B = [p_b]x R_LI^T C   (:1078-1082)
            double C[3], A2[3], B[3], crossb[9], M2[9];
            mat3_vec(Rt, nv, C);
            mat3_vec(cross, C, A2);
            skew(pb, crossb);
            mat3_mul(crossb, RLIt, M2);
            mat3_vec(M2, C, B);
            double* r = &H12[(size_t)k * 12];
            r[0] = nv[0]; r[1] = nv[1]; r[2] = nv[2];
            r[3] = A2[0]; r[4] = A2[1]; r[5] = A2[2];
            r[6] = B[0];  r[7] = B[1];  r[8] = B[2];
            r[9] = C[0];  r[10] = C[1]; r[11] = C[2];
        }
    }
    if (Hsub) std::memcpy(Hsub, Hloc.data(), sizeof(double) * Hloc.size());
    if (meas) std::memcpy(meas, zloc.data(), sizeof(double) * n);
    if (h_x) std::memcpy(h_x, H12.data(), sizeof(double) * H12.size());
    if (sel_idx) std::memcpy(sel_idx, ori.data(), sizeof(int) * n);
    if (HTH6 || HTz6) {
        double hth[36] = {0}, htz[6] = {0};
        for (int k = 0; k < n; ++k) {
            const double* h = &Hloc[(size_t)k * 6];
            for (int a = 0; a < 6; ++a) {
                for (int b = 0; b < 6; ++b) hth[a * 6 + b] += h[a] * h[b];
                htz[a] += h[a] * zloc[k];
            }
        }
        if (HTH6) std::memcpy(HTH6, hth, sizeof(hth));
        if (HTz6) std::memcpy(HTz6, htz, sizeof(htz));
    }
    if (HTH12 || HTh12) {
        double hth[144] = {0}, hth_v[12] = {0};
        for (int k = 0; k < n; ++k) {
            const double* h = &H12[(size_t)k * 12];
            for (int a = 0; a < 12; ++a) {
                for (int b = 0; b < 12; ++b) hth[a * 12 + b] += h[a] * h[b];
                hth_v[a] += h[a] * zloc[k];
            }
        }
        if (HTH12) std::memcpy(HTH12, hth, sizeof(hth));
        if (HTh12) std::memcpy(HTh12, hth_v, sizeof(hth_v));
    }
    if (world_xyz) std::memcpy(world_xyz, L->world.data(), sizeof(float) * 3 * (size_t)N);
    if (nn_idx_out) std::memcpy(nn_idx_out, L->nn_idx.data(), sizeof(int) * kMatch * (size_t)N);
    if (nn_d2_out) std::memcpy(nn_d2_out, L->nn_d2.data(), sizeof(float) * kMatch * (size_t)N);
    if (pd2_out)
        for (int i = 0; i < N; ++i) pd2_out[i] = L->normvec[4 * (size_t)i + 3];
    if (selected_out) std::memcpy(selected_out, L->selected.data(), N);
    return n;
}

// laserMapping.cpp:1469-1733 -- see SURVEY.md Appendix A for the restated control flow.
int flo_lio_update(flo_lio* L, const flo_lio_params* prm, flo_state18* x, const flo_state18* x_prop,
                   flo_lio_report* rep) {
    const int T = prm->max_iteration;
    int rematch_num = 0;
    bool nearest_search_en = true;                           // :1472-1473
    std::fill(L->selected.begin(), L->selected.end(), 1);    // fresh frame
    std::fill(L->res_last.begin(), L->res_last.end(), 1000.0);
    double G[kDim * kDim] = {0};
    flo_lio_report r = {};
    for (int iterCount = -1; iterCount < T; ++iterCount) {   // :1506
        double HTH6[36], HTz6[6], total = 0.0;
        const int n = flo_lio_pass(L, prm, x->rot, x->pos, nearest_search_en ? 1 : 0, nullptr, nullptr, nullptr,
                                   nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, HTH6, HTz6,
                                   nullptr, nullptr, &total);
        r.passes++;
        r.knn_passes += nearest_search_en ? 1 : 0;
        r.n_eff_last = n;
        r.res_mean_last = total / n;                          // :1602
        r.rows_total += n;
        bool EKF_stop = false, converged = false;             // :1634-1635
        double solution[kDim];
        ekf18_step(x, x_prop, HTH6, HTz6, prm->laser_point_cov, +1.0, G, solution);  // :1664-1683
        if ((norm3(solution) * 57.3 < prm->conv_rot_deg) && (norm3(solution + 3) * 100 < prm->conv_pos_cm))
            converged = true;                                 // :1688-1691
        nearest_search_en = false;                            // :1700
        if (converged || ((rematch_num == 0) && (iterCount == (T - 2)))) {  // :1701
            nearest_search_en = true;
            rematch_num++;
        }
        if (!EKF_stop && (rematch_num >= 2 || (iterCount == T - 1))) {      // :1708
            // state.cov = (I_STATE - G) * state.cov, :1715
            double IG[kDim * kDim], Pn[kDim * kDim];
            for (int i = 0; i < kDim; ++i)
                for (int j = 0; j < kDim; ++j) IG[i * kDim + j] = (i == j ? 1.0 : 0.0) - G[i * kDim + j];
            for (int i = 0; i < kDim; ++i)
                for (int j = 0; j < kDim; ++j) {
                    double s = 0.0;
                    for (int k = 0; k < kDim; ++k) s += IG[i * kDim + k] * x->cov[k * kDim + j];
                    Pn[i * kDim + j] = s;
                }
            std::memcpy(x->cov, Pn, sizeof(Pn));
            EKF_stop = true;
        }
        r.converged_last = converged ? 1 : 0;
        if (EKF_stop) break;                                  // :1731
    }
    if (rep) *rep = r;
    return 0;
}

}  // extern "C"

// =================================================================================
// VIO
// =================================================================================
struct flo_vio {
    std::vector<uint8_t> img;  // continuous, stride == width (lidar_selection.cpp:821 assumes it)
    int width = 0, height = 0;
    int Pn = 0;
    std::vector<double> pos;                  // Point::pos_, include/point.h:44
    std::vector<std::vector<float>> patch;    // SubSparseMap::patch, common_lib.h:269 (3*64 floats each)
    std::vector<int> search_level;
    std::vector<float> errors;
    flo_cam cam;
};

namespace {

// LidarSelector::init(), lidar_selection.cpp:41-59 + set_extrinsic :35-39
struct VioConst {
    double Rci[9], Pci[3], Jdphi_dR[9], Jdp_dR[9];
    double fx, fy;  // used by dpi (:92-103)
};

void vio_constants(const flo_vio_params* prm, const flo_cam* cam, VioConst* c) {
    double Rli[9], Pli[3], t[3];
    mat3_T(prm->R_LI, Rli);                         // Rli = rot^T
    mat3_vec(Rli, prm->t_LI, t);                    // Pli = -rot^T * transl
    for (int i = 0; i < 3; ++i) Pli[i] = -t[i];
    mat3_mul(prm->Rcl, Rli, c->Rci);                // Rci = Rcl * Rli
    mat3_vec(prm->Rcl, Pli, t);
    for (int i = 0; i < 3; ++i) c->Pci[i] = t[i] + prm->Pcl[i];  // Pci = Rcl*Pli + Pcl
    std::memcpy(c->Jdphi_dR, c->Rci, sizeof(c->Rci));            // Jdphi_dR = Rci
    double RciT[9], Pic[3], sk[9], m[9];
    mat3_T(c->Rci, RciT);
    mat3_vec(RciT, c->Pci, Pic);
    for (int i = 0; i < 3; ++i) Pic[i] = -Pic[i];               // Pic = -Rci^T * Pci
    skew(Pic, sk);
    mat3_mul(c->Rci, sk, m);
    for (int i = 0; i < 9; ++i) c->Jdp_dR[i] = -m[i];           // Jdp_dR = -Rci * [Pic]x
    // vikit PinholeCamera: errorMultiplier2() = |fx|, errorMultiplier() = |4 fx fy| (App. C)
    c->fx = std::fabs(cam->fx);
    c->fy = std::fabs(4.0 * cam->fx * cam->fy) / (4. * c->fx);  // :58-59
}

// One pass of the measurement loop of UpdateState, lidar_selection.cpp:772-857.
float vio_pass_core(flo_vio* V, const VioConst& K, const double R[9], const double p[3], int level,
                    double* z, double* H_sub, double* HTH6, double* HTz6, int64_t* n_meas_out,
                    int* skipped_out) {
    const int width = V->width, height = V->height;
    const int patch_size = 8, patch_size_total = 64, patch_size_half = 4;
    float error = 0.0f;
    size_t n_meas = 0;
    int skipped = 0;
    double Rwi_T[9], Rcw[9], Pcw[3], Jdp_dt[9], t[3];
    mat3_T(R, Rwi_T);
    mat3_mul(K.Rci, Rwi_T, Rcw);                          // :780
    double RciRt[9];
    mat3_mul(K.Rci, Rwi_T, RciRt);
    mat3_vec(RciRt, p, t);
    for (int i = 0; i < 3; ++i) Pcw[i] = -t[i] + K.Pci[i];  // :781  (-Rci*Rwi^T*Pwi + Pci)
    std::memcpy(Jdp_dt, RciRt, sizeof(RciRt));            // :782
    double hth[36] = {0}, htz[6] = {0};
    const uint8_t* data = V->img.data();

    for (int i = 0; i < V->Pn; ++i) {
        float patch_error = 0.0f;
        const int search_level = V->search_level[i];
        const int pyramid_level = level + search_level;
        const int scale = (1 << pyramid_level);
        double pf[3];
        mat3_vec(Rcw, &V->pos[3 * (size_t)i], pf);
        for (int k = 0; k < 3; ++k) pf[k] = pf[k] + Pcw[k];                    // :800
        double* zi = z ? z + (size_t)i * patch_size_total : nullptr;
        double* Hi = H_sub ? H_sub + (size_t)i * patch_size_total * 6 : nullptr;
        if (zi) std::memset(zi, 0, sizeof(double) * patch_size_total);
        if (Hi) std::memset(Hi, 0, sizeof(double) * patch_size_total * 6);
        V->errors[i] = 0.f;
        // Guard (OUR definition, SURVEY.md §7 H5): the reference reads pixels
        // unchecked (:821-837) and relies on selection-time borders; a patch whose
        // tap footprint (+-5*scale around the integer anchor) leaves the image, or
        // that is not in front of the camera, is skipped and counted -- on both
        // the oracle and the CUDA path.
        if (!(pf[2] > 0.0)) { skipped++; continue; }
        double pc[2];
        flo_world2cam(&V->cam, pf, pc);                                         // :801
        if (!(std::fabs(pc[0]) < 1e6) || !(std::fabs(pc[1]) < 1e6)) { skipped++; continue; }
        double Jdpi[6], p_hat[9];
        {   // dpi, :92-103
            const double x = pf[0], y = pf[1], z_inv = 1. / pf[2], z_inv_2 = z_inv * z_inv;
            Jdpi[0] = K.fx * z_inv; Jdpi[1] = 0.0; Jdpi[2] = -K.fx * x * z_inv_2;
            Jdpi[3] = 0.0; Jdpi[4] = K.fy * z_inv; Jdpi[5] = -K.fy * y * z_inv_2;
        }
        skew(pf, p_hat);                                                         // :805
        const float u_ref = pc[0];
        const float v_ref = pc[1];
        const int u_ref_i = floorf(pc[0] / scale) * scale;                      // :809
        const int v_ref_i = floorf(pc[1] / scale) * scale;
        if (u_ref_i - 5 * scale < 0 || u_ref_i + 5 * scale > width - 1 || v_ref_i - 5 * scale < 0 ||
            v_ref_i + 5 * scale > height - 1) { skipped++; continue; }
        const float subpix_u_ref = (u_ref - u_ref_i) / scale;
        const float subpix_v_ref = (v_ref - v_ref_i) / scale;
        const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);     // :813-816
        const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
        const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
        const float w_ref_br = subpix_u_ref * subpix_v_ref;

        std::vector<float> P = V->patch[i];                                      // :818 (copied per pass)
        for (int x = 0; x < patch_size; x++) {
            const uint8_t* img_ptr =
                data + (v_ref_i + x * scale - patch_size_half * scale) * width + u_ref_i - patch_size_half * scale;
            for (int y = 0; y < patch_size; ++y, img_ptr += scale) {
                float du = 0.5f * ((w_ref_tl * img_ptr[scale] + w_ref_tr * img_ptr[scale * 2] +
                                    w_ref_bl * img_ptr[scale * width + scale] + w_ref_br * img_ptr[scale * width + scale * 2]) -
                                   (w_ref_tl * img_ptr[-scale] + w_ref_tr * img_ptr[0] +
                                    w_ref_bl * img_ptr[scale * width - scale] + w_ref_br * img_ptr[scale * width]));
                float dv = 0.5f * ((w_ref_tl * img_ptr[scale * width] + w_ref_tr * img_ptr[scale + scale * width] +
                                    w_ref_bl * img_ptr[width * scale * 2] + w_ref_br * img_ptr[width * scale * 2 + scale]) -
                                   (w_ref_tl * img_ptr[-scale * width] + w_ref_tr * img_ptr[-scale * width + scale] +
                                    w_ref_bl * img_ptr[0] + w_ref_br * img_ptr[scale]));
                double Jimg[2] = {du, dv};
                const double inv_scale = (1.0 / scale);
                Jimg[0] = Jimg[0] * inv_scale;                                   // :831
                Jimg[1] = Jimg[1] * inv_scale;
                double JJ[3], Jdphi[3], Jdp[3], JdR[3], Jdt[3];
                for (int c = 0; c < 3; ++c) JJ[c] = Jimg[0] * Jdpi[c] + Jimg[1] * Jdpi[3 + c];
                for (int c = 0; c < 3; ++c)                                       // Jdphi = Jimg*Jdpi*p_hat
                    Jdphi[c] = JJ[0] * p_hat[c] + JJ[1] * p_hat[3 + c] + JJ[2] * p_hat[6 + c];
                for (int c = 0; c < 3; ++c) Jdp[c] = (-Jimg[0]) * Jdpi[c] + (-Jimg[1]) * Jdpi[3 + c];  // :833
                for (int c = 0; c < 3; ++c)                                       // :834
                    JdR[c] = (Jdphi[0] * K.Jdphi_dR[c] + Jdphi[1] * K.Jdphi_dR[3 + c] + Jdphi[2] * K.Jdphi_dR[6 + c]) +
                             (Jdp[0] * K.Jdp_dR[c] + Jdp[1] * K.Jdp_dR[3 + c] + Jdp[2] * K.Jdp_dR[6 + c]);
                for (int c = 0; c < 3; ++c)                                       // :835
                    Jdt[c] = Jdp[0] * Jdp_dt[c] + Jdp[1] * Jdp_dt[3 + c] + Jdp[2] * Jdp_dt[6 + c];
                double res = w_ref_tl * img_ptr[0] + w_ref_tr * img_ptr[scale] + w_ref_bl * img_ptr[scale * width] +
                             w_ref_br * img_ptr[scale * width + scale] - P[patch_size_total * level + x * patch_size + y];  // :837
                const double row[6] = {JdR[0], JdR[1], JdR[2], Jdt[0], Jdt[1], Jdt[2]};
                if (zi) zi[x * patch_size + y] = res;
                if (Hi) std::memcpy(Hi + (x * patch_size + y) * 6, row, sizeof(row));
                patch_error += res * res;                                        // :843 (float += double)
                n_meas++;
                for (int a = 0; a < 6; ++a) {
                    for (int b = 0; b < 6; ++b) hth[a * 6 + b] += row[a] * row[b];
                    htz[a] += row[a] * res;
                }
            }
        }
        V->errors[i] = patch_error;                                              // :851
        error += patch_error;                                                    // :852
    }
    error = error / n_meas;                                                      // :857 (float / size_t)
    if (HTH6) std::memcpy(HTH6, hth, sizeof(hth));
    if (HTz6) std::memcpy(HTz6, htz, sizeof(htz));
    if (n_meas_out) *n_meas_out = (int64_t)n_meas;
    if (skipped_out) *skipped_out = skipped;
    return error;
}

}  // namespace

extern "C" {

// vikit PinholeCamera::world2cam(Vector3d): project2d then (optional) radtan.  SURVEY App. C.
void flo_world2cam(const flo_cam* cam, const double pf[3], double px[2]) {
    const double x = pf[0] / pf[2], y = pf[1] / pf[2];
    if (!(std::fabs(cam->d[0]) > 0.0000001)) {
        px[0] = cam->fx * x + cam->cx;
        px[1] = cam->fy * y + cam->cy;
    } else {
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double a1 = 2 * x * y, a2 = r2 + 2 * x * x, a3 = r2 + 2 * y * y;
        const double cdist = 1 + cam->d[0] * r2 + cam->d[1] * r4 + cam->d[4] * r6;
        const double xd = x * cdist + cam->d[2] * a1 + cam->d[3] * a2;
        const double yd = y * cdist + cam->d[2] * a3 + cam->d[3] * a1;
        px[0] = xd * cam->fx + cam->cx;
        px[1] = yd * cam->fy + cam->cy;
    }
}

flo_vio* flo_vio_create(const uint8_t* gray, int width, int height, int stride, const double* pos,
                        const float* patch, const int* search_level, int Pn, const flo_cam* cam) {
    flo_vio* V = new flo_vio;
    V->width = width;
    V->height = height;
    V->img.resize((size_t)width * height);
    for (int r = 0; r < height; ++r) std::memcpy(&V->img[(size_t)r * width], gray + (size_t)r * stride, width);
    V->Pn = Pn;
    V->pos.assign(pos, pos + (size_t)3 * Pn);
    V->patch.resize(Pn);
    for (int i = 0; i < Pn; ++i) V->patch[i].assign(patch + (size_t)i * 192, patch + (size_t)(i + 1) * 192);
    V->search_level.assign(search_level, search_level + Pn);
    V->errors.assign(Pn, 0.f);
    V->cam = *cam;
    return V;
}

void flo_vio_destroy(flo_vio* V) { delete V; }

float flo_vio_pass(flo_vio* V, const flo_vio_params* prm, const double R[9], const double p[3], int level,
                   double* z, double* H_sub, float* errors, double* HTH6, double* HTz6, int64_t* n_meas_out,
                   int* skipped_out) {
    VioConst K;
    vio_constants(prm, &V->cam, &K);
    const float e = vio_pass_core(V, K, R, p, level, z, H_sub, HTH6, HTz6, n_meas_out, skipped_out);
    if (errors) std::memcpy(errors, V->errors.data(), sizeof(float) * V->Pn);
    return e;
}

void flo_vio_errors(const flo_vio* V, float* errors) { std::memcpy(errors, V->errors.data(), sizeof(float) * V->Pn); }

// LidarSelector::UpdateState(img, total_residual, level), lidar_selection.cpp:743-902.  G is the member G (:874): it
// keeps its value when no pass of this call is accepted.
static float update_state(flo_vio* V, const VioConst& K, const flo_vio_params* prm, flo_state18* x, const flo_state18* x_prop,
                          float total_residual, int level, double* G, flo_vio_report& r) {
    // H_sub / z are resized + zeroed per UpdateState call (:759-768): mirror the allocation.
    std::vector<double> z((size_t)V->Pn * 64, 0.0), H_sub((size_t)V->Pn * 64 * 6, 0.0);
    flo_state18 old_state = *x;                        // :747
    float last_error = total_residual;                 // :755
    bool EKF_end = false;
    for (int iteration = 0; iteration < prm->max_iteration; iteration++) {   // :772
        double HTH6[36], HTz6[6];
        int64_t n_meas = 0;
        int skipped = 0;
        const float error = vio_pass_core(V, K, x->rot, x->pos, level, z.data(), H_sub.data(), HTH6, HTz6,
                                          &n_meas, &skipped);
        r.passes[level]++;
        r.rows_total += n_meas;
        r.skipped_last = skipped;
        if (prm->force_all_passes || error <= last_error) {               // :861
            old_state = *x;
            last_error = error;
            double solution[kDim];
            ekf18_step(x, x_prop, HTH6, HTz6, prm->img_point_cov, -1.0, G, solution);  // :871-880
            if (!prm->force_all_passes &&
                (norm3(solution) * 57.3f < prm->conv_rot_deg) && (norm3(solution + 3) * 100.0f < prm->conv_pos_cm))
                EKF_end = true;                                              // :883-886
        } else {
            *x = old_state;                                                  // :890
            EKF_end = true;
            r.rejects++;
        }
        if (EKF_end) break;                                                  // :897
    }
    r.last_error[level] = last_error;
    return last_error;                                                       // :901
}

// UpdateState alone (one pyramid level).  G324: in/out, the 18x18 member G.
float flo_vio_update_level(flo_vio* V, const flo_vio_params* prm, int level, float total_residual, flo_state18* x,
                           const flo_state18* x_prop, double* G324, flo_vio_report* rep) {
    flo_vio_report r = {};
    if (V->Pn == 0) { if (rep) *rep = r; return 0.f; }   // :746
    VioConst K;
    vio_constants(prm, &V->cam, &K);
    const float e = update_state(V, K, prm, x, x_prop, total_residual, level, G324, r);
    if (rep) *rep = r;
    return e;
}

// ComputeJ (lidar_selection.cpp:967-983) driving UpdateState (:743-902) for level = 2,1,0.
int flo_vio_update(flo_vio* V, const flo_vio_params* prm, flo_state18* x, const flo_state18* x_prop,
                   flo_vio_report* rep) {
    flo_vio_report r = {};
    if (V->Pn == 0) { if (rep) *rep = r; return 0; }     // :969-970
    VioConst K;
    vio_constants(prm, &V->cam, &K);
    double G[kDim * kDim] = {0};
    const float error0 = 1e10f;                            // :971
    float now_error = error0;
    for (int level = 2; level >= 0; level--)               // :974
        now_error = update_state(V, K, prm, x, x_prop, error0, level, G, r);   // :976
    if (now_error < error0) {                                                    // :978
        // state->cov -= G * state->cov, :980
        double GP[kDim * kDim];
        for (int i = 0; i < kDim; ++i)
            for (int j = 0; j < kDim; ++j) {
                double s = 0.0;
                for (int k = 0; k < kDim; ++k) s += G[i * kDim + k] * x->cov[k * kDim + j];
                GP[i * kDim + j] = s;
            }
        for (int i = 0; i < kDim * kDim; ++i) x->cov[i] -= GP[i];
        r.cov_updated = 1;
    }
    if (rep) *rep = r;
    return 0;
}

}  // extern "C"
