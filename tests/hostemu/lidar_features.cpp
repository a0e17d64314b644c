// TEST INFRASTRUCTURE -- compiles the per-point math of flb_lidar_upload_features (feat_* in
// fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_lidar_features.py, composed per
// message as the kernels of flb_kernels.cuh compose it: the record filter and the stable sort by line, the per-point
// range / dista and line heads, one plane_judge per candidate, the visited chain by pointer doubling, the plane / edge
// types, the small-plane firing from a max-scan of run starts, the chunked surface output, then the compaction and the
// stable time sort.  This library is NEVER loaded by the product; it exists only under tests/.
#include <algorithm>
#include <climits>
#include <cmath>
#include <numeric>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

namespace {

// inclusive max-scan, as cub's
std::vector<int> max_scan(const std::vector<int>& v) {
    std::vector<int> o(v.size());
    int run = INT_MIN;
    for (size_t i = 0; i < v.size(); ++i) o[i] = run = std::max(run, v[i]);
    return o;
}

}  // namespace

extern "C" {

// fmt as tests/oracle_pre/feat_oracle.cpp's.  out: n x 4 floats (time-sorted pl_surf); ftypes: the final type of every
// line point, line-major.  Returns pl_surf's size; *bad = an emitted value is not finite.
int emu_feat_process(const int* fmt, double blind, double dis_b, const unsigned char* raw, int n, float* out, int* ftypes,
                     int* n_ftypes, int* bad) {
    LidarFmt f{};
    f.kind = fmt[0], f.step = fmt[1], f.off_x = fmt[2], f.off_y = fmt[3], f.off_z = fmt[4];
    f.off_time = fmt[5] >= 0 ? fmt[5] : 0, f.off_tag = fmt[6], f.off_line = fmt[7], f.n_scans = fmt[8], f.filter_num = fmt[9];
    f.blind = blind;
    const bool no_time = fmt[5] < 0;
    FeatConst c;
    c.blind = blind, c.dis_b = dis_b, c.avia = f.kind == kLidarLivox;
    c.jump_up = std::cos(170.0 / 180 * M_PI), c.jump_down = std::cos(8.0 / 180 * M_PI);
    c.cos160 = std::cos(160.0 / 180 * M_PI), c.smallp_intersect = std::cos(172.5 / 180 * M_PI);
    const int min_size = f.kind == kLidarLivox ? 6 : f.kind == kLidarVelodyne ? 2 : 1;
    *bad = 0;
    // given_offset_time (:279)
    bool yaw = false;
    if (f.kind == kLidarVelodyne && n > 0) {
        const float t_last = no_time ? 0.f : u32_as_float(lidar_ld32(raw + (size_t)(n - 1) * f.step + f.off_time));
        yaw = !(t_last > 0);
    }
    // k_feat_keys
    std::vector<int> key(n);
    for (int i = 0; i < n; ++i) {
        const unsigned char* r = raw + (size_t)i * f.step;
        if (f.kind == kLidarLivox) key[i] = feat_livox_line(r, i, f);
        else if (f.kind == kLidarOuster) key[i] = feat_ouster_line(r, f);
        else key[i] = std::min((int)lidar_ld16(r + f.off_line), f.n_scans);
    }
    std::vector<int> idx(n);
    std::iota(idx.begin(), idx.end(), 0);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return key[a] < key[b]; });
    std::vector<int> skey(n);
    for (int p = 0; p < n; ++p) skey[p] = key[idx[p]];
    std::vector<VeloMap> map(n);
    if (yaw) {                                                      // k_velo_maps and the inclusive scan
        for (int p = 0; p < n; ++p) {
            const int hp = (int)(std::lower_bound(skey.begin(), skey.begin() + p, skey[p]) - skey.begin());
            map[p] = velo_head();
            if (skey[p] < f.n_scans && hp != p) {
                const unsigned char* r = raw + (size_t)idx[p] * f.step;
                const unsigned char* h = raw + (size_t)idx[hp] * f.step;
                map[p] = velo_step(velo_yaw(u32_as_float(lidar_ld32(r + f.off_x)), u32_as_float(lidar_ld32(r + f.off_y))),
                                   velo_yaw(u32_as_float(lidar_ld32(h + f.off_x)), u32_as_float(lidar_ld32(h + f.off_y))));
            }
        }
        for (int p = 1; p < n; ++p) map[p] = velo_compose(map[p - 1], map[p]);
    }
    // k_feat_gather: the kept records in line order
    std::vector<LidarPoint> P;
    std::vector<int> lkey;
    for (int p = 0; p < n; ++p) {
        if (skey[p] >= f.n_scans) continue;
        const bool head = p == 0 || skey[p - 1] != skey[p];
        if (yaw && head) continue;                                  // a ring's first record (:324-333)
        LidarPoint q = lidar_decode(raw + (size_t)idx[p] * f.step, f);
        if (yaw) q.t = velo_apply(map[p], 0.f);           // also every Velodyne without a time field
        P.push_back(q);
        lkey.push_back(skey[p]);
    }
    const int M = (int)P.size();
    // k_feat_range
    std::vector<int> lbeg(f.n_scans, 0), lend(f.n_scans, 0), lhead(f.n_scans, INT_MAX);
    std::vector<double> rng(M), dista(M);
    for (int q = 0; q < M; ++q) {
        const int k = lkey[q];
        rng[q] = feat_range(P[q], c.avia);
        dista[q] = (q + 1 < M && lkey[q + 1] == k) ? feat_dista(P[q], P[q + 1]) : 0.0;
        if (q == 0 || lkey[q - 1] != k) lbeg[k] = q;
        if (q + 1 == M || lkey[q + 1] != k) lend[k] = q + 1;
        if (!(rng[q] < blind)) lhead[k] = std::min(lhead[k], q);
    }
    // k_feat_steps
    std::vector<FeatStep> st(M);
    int levels = 1;
    while ((1 << levels) <= M) ++levels;
    std::vector<std::vector<int>> J(levels, std::vector<int>(M));
    std::vector<unsigned char> vis(M);
    for (int q = 0; q < M; ++q) {
        const FeatLine L = feat_line(lbeg.data(), lend.data(), lhead.data(), lkey[q], min_size);
        st[q] = feat_step_at(P.data(), rng.data(), dista.data(), L, q, c);
        J[0][q] = feat_succ(st[q], L, q);
        vis[q] = (q - L.b == L.head && L.head < feat_plsize2(L)) ? 1 : 0;
    }
    // k_feat_jump, k_feat_mark
    for (int l = 0; l + 1 < levels; ++l)
        for (int q = 0; q < M; ++q) J[l + 1][q] = J[l][q] < 0 ? -1 : J[l][J[l][q]];
    for (int l = levels - 1; l >= 0; --l)
        for (int q = 0; q < M; ++q)
            if (vis[q] && J[l][q] >= 0) vis[J[l][q]] = 1;
    // exclusive max-scan of the visited indices
    std::vector<int> pv(M);
    for (int q = 0, run = -1; q < M; ++q) {
        pv[q] = run;
        if (vis[q]) run = q;
    }
    // k_feat_types
    std::vector<int> ft(M);
    std::vector<double> isect(M);
    std::vector<FeatLine> lines(M);
    for (int q = 0; q < M; ++q) {
        const FeatLine L = lines[q] = feat_line(lbeg.data(), lend.data(), lhead.data(), lkey[q], min_size);
        const int p = pv[q];
        const FeatEdge e = feat_types_at(P.data(), rng.data(), dista.data(), L, q, vis[q] != 0, st[q], p, p >= 0 ? st[p] : st[q], c);
        ft[q] = e.ftype, isect[q] = e.intersect;
    }
    // k_feat_small, seeds, max-scan
    std::vector<unsigned char> small(M);
    for (int q = 0; q < M; ++q) {
        const FeatLine& L = lines[q];
        small[q] = feat_small_cond(rng.data() + L.b, dista.data() + L.b, L.m, L.head, q - L.b, ft[q], isect[q], c) ? 1 : 0;
    }
    std::vector<int> seed(M);
    for (int q = 0; q < M; ++q) seed[q] = (small[q] && !(q > 0 && small[q - 1])) ? q : -1;
    const std::vector<int> rs = max_scan(seed);
    // k_feat_final
    std::vector<int> fin(M);
    for (int q = 0; q < M; ++q) fin[q] = feat_final_at(ft.data(), small.data(), rs.data(), M, q);
    for (int q = 0; q < M; ++q) {
        const FeatLine& L = lines[q];
        const int j = q - L.b;
        const bool s = j >= L.head && feat_is_surf(fin[q]);
        seed[q] = (s && (j == L.head || !feat_is_surf(fin[q - 1]))) ? q : -1;
    }
    const std::vector<int> rs2 = max_scan(seed);
    // k_feat_emit, then k_lidar_scatter and the stable time sort
    std::vector<LidarPoint> cloud;
    std::vector<unsigned> keys;
    for (int q = 0; q < M; ++q) {
        LidarPoint o;
        if (!feat_emit_at(P.data(), fin.data(), rs2.data(), lines[q], q, f.filter_num, &o)) continue;
        cloud.push_back(o);
        keys.push_back(lidar_time_key(o.t));
        if (!(lidar_finite(o.x) && lidar_finite(o.y) && lidar_finite(o.z) && lidar_finite(o.t))) *bad = 1;
    }
    const int m = (int)cloud.size();
    std::vector<int> order(m);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    for (int j = 0; j < m; ++j) {
        const LidarPoint& q = cloud[order[j]];
        out[4 * j] = q.x, out[4 * j + 1] = q.y, out[4 * j + 2] = q.z, out[4 * j + 3] = q.t;
    }
    for (int q = 0; q < M; ++q) ftypes[q] = fin[q];
    *n_ftypes = M;
    return m;
}

}  // extern "C"
