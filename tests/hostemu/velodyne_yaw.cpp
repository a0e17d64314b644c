// TEST INFRASTRUCTURE -- compiles the per-record math of flb_lidar_upload_velodyne's yaw route (lidar_ld16, velo_yaw,
// velo_step, velo_head, velo_compose, velo_apply, lidar_pc2_keep, lidar_time_key in fast-livo_b200/csrc/flb_device.cuh)
// with g++ for the CPU-only tests of tests/test_velodyne_yaw.py, composed per message as the kernels of flb_kernels.cuh
// compose it: k_velo_rings, the stable sort by ring, k_velo_maps (the head found by a lower bound), the inclusive scan,
// k_velo_flags, then flb_lidar_upload's compaction and stable time sort.  This library is NEVER loaded by the product; it
// exists only under tests/.
#include <algorithm>
#include <numeric>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// fmt: point_step, off_x, off_y, off_z, off_time (unused: the yaw route), off_ring, n_scans, point_filter_num.
// out: n x 4 floats.  Returns the kept count, or -1 with *bad_ring = the first record whose ring is >= n_scans.
// *bad = a kept value is not finite.
int emu_velo_process(const int* fmt, double blind, const unsigned char* raw, int n, float* out, int* bad, int* bad_ring) {
    LidarFmt f{};
    f.kind = kLidarVelodyne, f.step = fmt[0], f.off_x = fmt[1], f.off_y = fmt[2], f.off_z = fmt[3];
    f.n_scans = fmt[6], f.filter_num = fmt[7], f.blind = blind;
    const int off_ring = fmt[5], n_rings = std::min(f.n_scans, 65536);
    std::vector<unsigned> key(n);
    std::vector<int> idx(n);
    *bad_ring = -1;
    for (int i = 0; i < n; ++i) {                                  // k_velo_rings
        const unsigned ring = lidar_ld16(raw + (size_t)i * f.step + off_ring);
        key[i] = (int)ring < f.n_scans ? ring : (unsigned)n_rings;
        if (key[i] == (unsigned)n_rings && *bad_ring < 0) *bad_ring = i;
    }
    if (*bad_ring >= 0) return -1;
    std::iota(idx.begin(), idx.end(), 0);
    std::stable_sort(idx.begin(), idx.end(), [&](int a, int b) { return key[a] < key[b]; });
    std::vector<unsigned> skey(n);
    for (int p = 0; p < n; ++p) skey[p] = key[idx[p]];
    std::vector<VeloMap> map(n);
    for (int p = 0; p < n; ++p) {                                  // k_velo_maps
        const int hp = (int)(std::lower_bound(skey.begin(), skey.begin() + p, skey[p]) - skey.begin());
        map[p] = velo_head();
        if (hp != p) {
            const unsigned char* r = raw + (size_t)idx[p] * f.step;
            const unsigned char* h = raw + (size_t)idx[hp] * f.step;
            map[p] = velo_step(velo_yaw(u32_as_float(lidar_ld32(r + f.off_x)), u32_as_float(lidar_ld32(r + f.off_y))),
                               velo_yaw(u32_as_float(lidar_ld32(h + f.off_x)), u32_as_float(lidar_ld32(h + f.off_y))));
        }
    }
    for (int p = 1; p < n; ++p) map[p] = velo_compose(map[p - 1], map[p]);   // the inclusive scan
    std::vector<LidarPoint> dec(n);
    std::vector<int> kept(n);
    for (int p = 0; p < n; ++p) {                                  // k_velo_flags
        const int i = idx[p];
        const bool head = p == 0 || skey[p - 1] != skey[p];
        const unsigned char* r = raw + (size_t)i * f.step;
        LidarPoint q;
        q.x = u32_as_float(lidar_ld32(r + f.off_x));
        q.y = u32_as_float(lidar_ld32(r + f.off_y));
        q.z = u32_as_float(lidar_ld32(r + f.off_z));
        q.t = head ? 0.f : velo_apply(map[p], 0.f);
        dec[i] = q;
        kept[i] = !head && lidar_pc2_keep(q, i, f);
    }
    std::vector<LidarPoint> cloud;                                 // k_lidar_scatter
    std::vector<unsigned> keys;
    *bad = 0;
    for (int i = 0; i < n; ++i)
        if (kept[i]) {
            cloud.push_back(dec[i]);
            keys.push_back(lidar_time_key(dec[i].t));
            if (!(lidar_finite(dec[i].x) && lidar_finite(dec[i].y) && lidar_finite(dec[i].z) && lidar_finite(dec[i].t))) *bad = 1;
        }
    const int m = (int)cloud.size();
    std::vector<int> order(m);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    for (int j = 0; j < m; ++j) {
        const LidarPoint& q = cloud[order[j]];
        out[4 * j] = q.x, out[4 * j + 1] = q.y, out[4 * j + 2] = q.z, out[4 * j + 3] = q.t;
    }
    return m;
}

// the scan operator on (c, a, b) triples: out = compose(first, then); apply(m, x)
void emu_velo_compose(const float* first, const float* then, float* out) {
    const VeloMap a{first[0], first[1], first[2]}, b{then[0], then[1], then[2]};
    const VeloMap m = velo_compose(a, b);
    out[0] = m.c, out[1] = m.a, out[2] = m.b;
}
float emu_velo_apply(const float* m, float x) { return velo_apply(VeloMap{m[0], m[1], m[2]}, x); }

// velo_step(yaw, yaw_fp) as (c, a, b), and velo_yaw
void emu_velo_step(double yaw, double yaw_fp, float* out) {
    const VeloMap m = velo_step(yaw, yaw_fp);
    out[0] = m.c, out[1] = m.a, out[2] = m.b;
}
double emu_velo_yaw(float x, float y) { return velo_yaw(x, y); }

}  // extern "C"
