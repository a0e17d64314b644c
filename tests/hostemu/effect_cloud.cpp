// TEST INFRASTRUCTURE -- compiles flb_effect_cloud's per-point rules (lio_sel_byte, lio_sel_is_row,
// effect_scatter_point and map_scan_point in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of
// tests/test_effect_cloud.py: the byte a LIO pass leaves per point of the ordered scan, the capture (k_effect_scatter,
// then an order-preserving select like cub::DeviceSelect::Flagged) and the transform (k_map_scan_world<false>).  Each
// loop iteration is one thread.  This library is NEVER loaded by the product; it exists only under tests/.
#include "../../fast-livo_b200/csrc/flb_device.cuh"

#include <vector>

using namespace flb;

extern "C" {

// The byte lio_point stores for each of n points: sel = point_selected_surf after the pass, pd2 its residual.
void emu_sel_bytes(const unsigned char* sel, const float* pd2, int n, unsigned char* out) {
    for (int i = 0; i < n; ++i) out[i] = lio_sel_byte(sel[i] != 0, pd2[i]);
}

// scan4: n ordered entries {x, y, z, caller's index as int bits}; sel_bytes: the pass's byte of each.  Writes the rows'
// body points (scan-index order) to body4 and their transform at (R, p) with (R_LI, t_LI) to world; returns their count.
int emu_effect_cloud(const double* R, const double* p, const double* R_LI, const double* t_LI, const float* scan4,
                     const unsigned char* sel_bytes, int n, float* body4, float* world) {
    const map_pt* scan = reinterpret_cast<const map_pt*>(scan4);
    std::vector<unsigned char> flag(n, 0);
    std::vector<map_pt> scattered(n);
    for (int i = 0; i < n; ++i) effect_scatter_point(scan[i], sel_bytes[i], flag.data(), scattered.data());
    map_pt* body = reinterpret_cast<map_pt*>(body4);
    int m = 0;
    for (int i = 0; i < n; ++i)
        if (flag[i]) body[m++] = scattered[i];
    LioPose pose{};
    memcpy(pose.R, R, sizeof(pose.R));
    memcpy(pose.p, p, sizeof(pose.p));
    memcpy(pose.R_LI, R_LI, sizeof(pose.R_LI));
    memcpy(pose.t_LI, t_LI, sizeof(pose.t_LI));
    for (int i = 0; i < m; ++i) map_scan_point(pose, body[i], world + 3 * (size_t)i);
    return m;
}

}  // extern "C"
