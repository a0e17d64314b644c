// TEST INFRASTRUCTURE -- the checker of flb_lidar_upload_velodyne: a plain C++17 restatement, op for op, of the
// non-feature (`else`) branch of velodyne_handler (reference src/preprocess.cpp:259-297, :376-428), followed by the time
// sort of sync_packages (src/laserMapping.cpp:551, as std::stable_sort: the project defines the order of equal times as
// record order).  The reference's own file needs ROS and PCL, so this is written from its text with line citations; it
// shares no code with the product.  Loaded by tests/velo_oracle.py; never by the product.
//
// Two yaw modes.  kYawDefined: (float)atan2((double)y, (double)x), the project's definition (DESIGN §2).  kYawAtan2f:
// atan2 of the two floats, which with the reference's `using namespace std` is the float overload of the libm linked
// here: the reference as built on this host.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

using namespace std;   // as include/preprocess.h:6: atan2(float, float) is std::atan2(float, float)

namespace {

enum { kYawDefined = 0, kYawAtan2f = 1 };

struct Pt { float x, y, z, curvature; };

struct Format {
    int step, off_x, off_y, off_z, off_time, off_ring, N_SCANS, point_filter_num;
    double blind;
};

template <typename T>
T field(const unsigned char* msg, const Format& f, size_t i, int off) {
    T v;
    memcpy(&v, msg + i * (size_t)f.step + off, sizeof(T));
    return v;
}

// velodyne_ros::Point::time; a cloud without the field reads 0
float time_of(const unsigned char* msg, const Format& f, size_t i) { return f.off_time < 0 ? 0.f : field<float>(msg, f, i, f.off_time); }

double yaw_of(float x, float y, int mode) {
    if (mode == kYawAtan2f) return atan2(y, x) * 57.2957;                          // :392, float overload
    return (double)(float)atan2((double)y, (double)x) * 57.2957;
}

// :259-297 and :376-428.  Returns false at a ring >= N_SCANS (*bad = the record), which the reference does not check.
bool velodyne(const unsigned char* msg, const Format& f, int plsize, int mode, vector<Pt>& pl_surf, int* given, int* bad) {
    *given = 0;
    if (plsize == 0) return true;                                                  // :268
    const int N_SCANS = f.N_SCANS;
    double omega_l = 0.361 * 10;                                                   // :272
    vector<bool> is_first(N_SCANS, true);                                          // :273
    vector<double> yaw_fp(N_SCANS, 0.0);                                           // :274
    vector<float> yaw_last(N_SCANS, 0.0);                                          // :275
    vector<float> time_last(N_SCANS, 0.0);                                         // :276
    const bool given_offset_time = time_of(msg, f, plsize - 1) > 0;                // :279-282
    *given = given_offset_time;
    for (int i = 0; i < plsize; i++) {                                             // :376
        Pt added_pt;
        added_pt.x = field<float>(msg, f, i, f.off_x);
        added_pt.y = field<float>(msg, f, i, f.off_y);
        added_pt.z = field<float>(msg, f, i, f.off_z);
        added_pt.curvature = time_of(msg, f, i) * 1.e-3f;                          // :387
        if (!given_offset_time) {                                                  // :389
            int layer = field<uint16_t>(msg, f, i, f.off_ring);                    // :391
            if (layer >= N_SCANS) { *bad = i; return false; }
            double yaw_angle = yaw_of(added_pt.x, added_pt.y, mode);               // :392
            if (is_first[layer]) {                                                 // :394-403
                yaw_fp[layer] = yaw_angle;
                is_first[layer] = false;
                added_pt.curvature = 0.0;
                yaw_last[layer] = yaw_angle;
                time_last[layer] = added_pt.curvature;
                continue;
            }
            if (yaw_angle <= yaw_fp[layer]) {                                      // :406-413
                added_pt.curvature = (yaw_fp[layer] - yaw_angle) / omega_l;
            } else {
                added_pt.curvature = (yaw_fp[layer] - yaw_angle + 360.0) / omega_l;
            }
            if (added_pt.curvature < time_last[layer]) added_pt.curvature += 360.0 / omega_l;   // :415
            yaw_last[layer] = yaw_angle;                                           // :417
            time_last[layer] = added_pt.curvature;                                 // :418
        }
        if (i % f.point_filter_num == 0) {                                         // :421
            if (added_pt.x * added_pt.x + added_pt.y * added_pt.y + added_pt.z * added_pt.z > (f.blind * f.blind)) {   // :423
                pl_surf.push_back(added_pt);
            }
        }
    }
    return true;
}

bool time_list(const Pt& x, const Pt& y) { return (x.curvature < y.curvature); }   // include/common_lib.h

// Is the double d within `ulps` double ulps of a midpoint between two adjacent floats?  Then a double atan2 that differs
// from this libm's by a few ulps may round to the other float.
bool near_midpoint(double d, int ulps) {
    if (!std::isfinite(d)) return false;
    const float f = (float)d;
    const double lo = 0.5 * ((double)f + (double)nextafterf(f, -INFINITY));
    const double hi = 0.5 * ((double)f + (double)nextafterf(f, INFINITY));
    for (double m : {lo, hi}) {
        double a = m, b = m;
        for (int k = 0; k < ulps; ++k) a = nextafter(a, -INFINITY), b = nextafter(b, INFINITY);
        if (d >= a && d <= b) return true;
    }
    return false;
}

}  // namespace

extern "C" {

// velodyne_handler into out (n x 4 floats: x, y, z, curvature), then the stable time sort when do_sort.  fmt: the eight
// ints of Format.  *yaw_times = !given_offset_time (0 for an empty cloud).  Returns pl_surf.size(), or -1 with *bad_ring =
// the first record whose ring is >= N_SCANS on the yaw route.
int velo_process(const int* fmt, double blind, const unsigned char* msg, int n, int mode, int do_sort, float* out, int* yaw_times,
                 int* bad_ring) {
    Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], blind};
    vector<Pt> pl_surf;
    pl_surf.reserve(n);
    int given = 0;
    *bad_ring = -1;
    if (!velodyne(msg, f, n, mode, pl_surf, &given, bad_ring)) return -1;
    *yaw_times = n > 0 && !given;
    if (do_sort) stable_sort(pl_surf.begin(), pl_surf.end(), time_list);           // src/laserMapping.cpp:551
    if (!pl_surf.empty()) memcpy(out, pl_surf.data(), pl_surf.size() * sizeof(Pt));
    return (int)pl_surf.size();
}

// flags[i] = record i's double atan2 lies within `ulps` double ulps of a float rounding midpoint.  Returns the count.
int velo_midpoint_flags(const int* fmt, const unsigned char* msg, int n, int ulps, unsigned char* flags) {
    Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], 0.0};
    int count = 0;
    for (int i = 0; i < n; ++i) {
        const float x = field<float>(msg, f, i, f.off_x), y = field<float>(msg, f, i, f.off_y);
        flags[i] = near_midpoint(atan2((double)y, (double)x), ulps);
        count += flags[i];
    }
    return count;
}

// the two yaw modes of one point, for the tests of the rounding itself
double velo_yaw(float x, float y, int mode) { return yaw_of(x, y, mode); }

}  // extern "C"
