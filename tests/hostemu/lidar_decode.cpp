// TEST INFRASTRUCTURE -- compiles the per-record math of flb_lidar_upload (lidar_decode, lidar_livox_*, lidar_pc2_keep,
// lidar_time_key in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_lidar_decode.py,
// composed per message as the kernels of flb_kernels.cuh compose it: k_lidar_valid, the inclusive sum, k_lidar_flags,
// the exclusive sum, k_lidar_scatter, the stable sort on the 32-bit time keys, k_lidar_window's partition point.  This
// library is NEVER loaded by the product; it exists only under tests/.
#include <algorithm>
#include <numeric>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// fmt: kind, step, off_x, off_y, off_z, off_time, off_tag, off_line, n_scans, point_filter_num.  out: n x 4 floats.
// Returns the kept count; *bad = a kept value is not finite; *was_sorted = the compacted times were non-decreasing.
int emu_lidar_decode(const int* fmt, double blind, const unsigned char* raw, int n, float* out, int* bad, int* was_sorted) {
    LidarFmt f{};
    f.kind = fmt[0], f.step = fmt[1], f.off_x = fmt[2], f.off_y = fmt[3], f.off_z = fmt[4], f.off_time = fmt[5];
    f.off_tag = fmt[6], f.off_line = fmt[7], f.n_scans = fmt[8], f.filter_num = fmt[9], f.blind = blind;
    if (n > 0 && f.kind == kLidarXt32) f.time_head = lidar_ld64f(raw + f.off_time);
    std::vector<int> vnum(n, 0), kept(n, 0), pos(n, 0);
    if (f.kind == kLidarLivox) {
        for (int i = 0; i < n; ++i) vnum[i] = lidar_livox_valid(raw + (size_t)i * f.step, i, f) ? 1 : 0;
        std::partial_sum(vnum.begin(), vnum.end(), vnum.begin());
    }
    std::vector<LidarPoint> dec(n);
    for (int i = 0; i < n; ++i) {                                  // k_lidar_flags
        const unsigned char* r = raw + (size_t)i * f.step;
        const LidarPoint q = lidar_decode(r, f);
        bool keep;
        if (f.kind == kLidarLivox) {
            const int vn = vnum[i], vp = i > 0 ? vnum[i - 1] : 0;
            keep = false;
            if (lidar_livox_candidate(vn != vp, (unsigned)vn, f)) {
                float px = 0.f, py = 0.f, pz = 0.f;
                const int vpp = i > 1 ? vnum[i - 2] : 0;
                if (i > 0 && lidar_livox_candidate(vp != vpp, (unsigned)vp, f)) {
                    const LidarPoint b = lidar_decode(r - f.step, f);
                    px = b.x, py = b.y, pz = b.z;
                }
                keep = lidar_livox_keep(q, px, py, pz, f.blind);
            }
        } else {
            keep = lidar_pc2_keep(q, i, f);
        }
        dec[i] = q;
        kept[i] = keep ? 1 : 0;
    }
    std::exclusive_scan(kept.begin(), kept.end(), pos.begin(), 0);
    const int m = n > 0 ? pos[n - 1] + kept[n - 1] : 0;
    std::vector<LidarPoint> cloud(m);
    std::vector<unsigned> keys(m);
    *bad = 0;
    for (int i = 0; i < n; ++i)                                    // k_lidar_scatter
        if (kept[i]) {
            cloud[pos[i]] = dec[i];
            keys[pos[i]] = lidar_time_key(dec[i].t);
            if (!(lidar_finite(dec[i].x) && lidar_finite(dec[i].y) && lidar_finite(dec[i].z) && lidar_finite(dec[i].t))) *bad = 1;
        }
    *was_sorted = 1;
    for (int j = 1; j < m; ++j)                                    // k_lidar_order
        if (keys[j] < keys[j - 1]) *was_sorted = 0;
    std::vector<int> order(m);
    std::iota(order.begin(), order.end(), 0);
    if (!*was_sorted) std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    for (int j = 0; j < m; ++j) {
        const LidarPoint& q = cloud[order[j]];
        out[4 * j] = q.x, out[4 * j + 1] = q.y, out[4 * j + 2] = q.z, out[4 * j + 3] = q.t;
    }
    return m;
}

// k_lidar_window's partition point on a sorted x, y, z, t cloud
int emu_lidar_window(const float* cloud, int begin, int n, double pcl_offset_time) {
    int lo = begin, hi = n;
    while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if ((double)cloud[4 * mid + 3] <= pcl_offset_time) lo = mid + 1;
        else hi = mid;
    }
    return lo - begin;
}

}  // extern "C"
