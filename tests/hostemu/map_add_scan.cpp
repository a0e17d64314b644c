// TEST INFRASTRUCTURE -- compiles the per-point rule of flb_map_add_scan (map_scan_point, finite3, f32_order_key and
// f32_from_order_key in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of
// tests/test_map_add_scan.py, applied as k_map_scan_world applies it (each loop iteration is one thread; the bounds
// record is folded with the same maxima).  This library is NEVER loaded by the product; it exists only under tests/.
#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// scan4: n ordered entries {x, y, z, caller's index as int bits}.  out: n x 3 world points at the caller's index;
// rec[kScanRecWords]: the record k_map_scan_world leaves (zeroed here first).
void emu_map_scan_world(const double* R, const double* p, const double* R_LI, const double* t_LI, const float* scan4, int n, float* out,
                        unsigned* rec) {
    LioPose pose{};
    memcpy(pose.R, R, sizeof(pose.R));
    memcpy(pose.p, p, sizeof(pose.p));
    memcpy(pose.R_LI, R_LI, sizeof(pose.R_LI));
    memcpy(pose.t_LI, t_LI, sizeof(pose.t_LI));
    for (int w = 0; w < kScanRecWords; ++w) rec[w] = 0;
    const map_pt* scan = reinterpret_cast<const map_pt*>(scan4);
    for (int i = 0; i < n; ++i) {
        float pw[3];
        const int oi = map_scan_point(pose, scan[i], pw);
        for (int k = 0; k < 3; ++k) out[3 * (size_t)oi + k] = pw[k];
        if (finite3(pw)) {
            for (int k = 0; k < 3; ++k) {
                rec[kScanRecMax + k] = max(rec[kScanRecMax + k], f32_order_key(pw[k]));
                rec[kScanRecMin + k] = max(rec[kScanRecMin + k], ~f32_order_key(pw[k]));
            }
        } else {
            rec[kScanRecBad] = 1;
        }
    }
}

// The host's reading of the record (flb_map_add_scan): lo / hi per axis, and whether a point was not finite.
int emu_scan_rec_bounds(const unsigned* rec, float* lo, float* hi) {
    for (int k = 0; k < 3; ++k) {
        lo[k] = f32_from_order_key(~rec[kScanRecMin + k]);
        hi[k] = f32_from_order_key(rec[kScanRecMax + k]);
    }
    return rec[kScanRecBad] ? 1 : 0;
}

}  // extern "C"
