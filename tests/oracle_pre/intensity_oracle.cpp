// TEST INFRASTRUCTURE -- the checker of the intensity uploads (flb_lidar_upload_intensity,
// flb_lidar_upload_velodyne_intensity): plain C++17 restatements, op for op, of the non-feature (`else`) branches of
// Preprocess's four handlers (reference src/preprocess.cpp) with their intensity lines -- Livox `reflectivity` (:148),
// the typed cloud's `intensity` that pcl::fromROSMsg fills (:246, :386, :453), 0 for a message without a FLOAT32
// intensity field (PCL's field mapping skips it) -- and of velodyne_handler's yaw route (:259-297, :376-428), each followed
// by the time sort of sync_packages (src/laserMapping.cpp:551, as std::stable_sort: the project defines the order of equal
// times as record order).  The same statements as tests/oracle_pre/pre_oracle.cpp and velo_oracle.cpp, which check the
// uploads without intensity, plus the intensity lines.  The reference's own file needs ROS, PCL and livox_ros_driver, so
// this is written from its text with line citations; it shares no code with the product.  Loaded by
// tests/intensity_oracle.py; never by the product.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

using namespace std;   // the reference's `abs` is std::abs(float), its atan2(float, float) std::atan2(float, float)

// Preprocess::process (src/preprocess.cpp:43-70) with feature_extract_enable = 0
namespace pre {
// pcl::PointXYZINormal: 48 bytes, curvature at float index 9
struct PointType {
    float x = 0.f, y = 0.f, z = 0.f, pad0 = 1.f;
    float normal_x = 0.f, normal_y = 0.f, normal_z = 0.f, pad1 = 0.f;
    float intensity = 0.f, curvature = 0.f, pad2 = 0.f, pad3 = 0.f;
};
static_assert(sizeof(PointType) == 48, "PointXYZINormal layout");

struct Format {
    int kind, step, off_x, off_y, off_z, off_time, off_tag, off_line, n_scans, point_filter_num;
    double blind;
    int off_intensity;   // Livox reflectivity (u8) or the PointCloud2's FLOAT32 intensity; -1: none, PCL leaves 0
};

template <typename T>
T field(const unsigned char* msg, const Format& f, size_t i, int off) {
    T v;
    memcpy(&v, msg + i * (size_t)f.step + off, sizeof(T));
    return v;
}

// CustomPoint::reflectivity, or the intensity pcl::fromROSMsg copies into the typed cloud (0 when the message has no
// FLOAT32 intensity field: PCL's field mapping skips it and the point keeps its default)
float intensity_of(const unsigned char* msg, const Format& f, size_t i) {
    if (f.off_intensity < 0) return 0.f;
    if (f.kind == 1) return field<uint8_t>(msg, f, i, f.off_intensity);
    return field<float>(msg, f, i, f.off_intensity);
}

// avia_handler, :136-161
void avia(const unsigned char* msg, const Format& f, unsigned plsize, vector<PointType>& pl_surf) {
    vector<PointType> pl_full(plsize);                                             // :83
    unsigned valid_num = 0;                                                        // :90
    const int N_SCANS = f.n_scans, point_filter_num = f.point_filter_num;
    const double blind = f.blind;
    for (unsigned i = 1; i < plsize; i++) {                                        // :138
        const uint8_t line = field<uint8_t>(msg, f, i, f.off_line), tag = field<uint8_t>(msg, f, i, f.off_tag);
        if ((line < N_SCANS) && ((tag & 0x30) == 0x10 || (tag & 0x30) == 0x00)) {  // :140
            valid_num++;
            if (valid_num % point_filter_num == 0) {                               // :143
                pl_full[i].x = field<float>(msg, f, i, f.off_x);
                pl_full[i].y = field<float>(msg, f, i, f.off_y);
                pl_full[i].z = field<float>(msg, f, i, f.off_z);
                pl_full[i].intensity = intensity_of(msg, f, i);                    // :148
                pl_full[i].curvature = field<uint32_t>(msg, f, i, f.off_time) / float(1000000);   // :149
                if (((abs(pl_full[i].x - pl_full[i - 1].x) > 1e-7) || (abs(pl_full[i].y - pl_full[i - 1].y) > 1e-7) ||
                     (abs(pl_full[i].z - pl_full[i - 1].z) > 1e-7)) &&
                    (pl_full[i].x * pl_full[i].x + pl_full[i].y * pl_full[i].y + pl_full[i].z * pl_full[i].z > (blind * blind))) {   // :151-154
                    pl_surf.push_back(pl_full[i]);
                }
            }
        }
    }
}

// oust64_handler, :228-254
void oust64(const unsigned char* msg, const Format& f, int plsize, vector<PointType>& pl_surf) {
    for (int i = 0; i < plsize; i++) {
        if (i % f.point_filter_num != 0) continue;                                 // :235
        const float x = field<float>(msg, f, i, f.off_x), y = field<float>(msg, f, i, f.off_y), z = field<float>(msg, f, i, f.off_z);
        double range = x * x + y * y + z * z;                                      // :237
        if (range < (f.blind * f.blind)) continue;                                 // :239
        PointType added_pt;
        added_pt.x = x;
        added_pt.y = y;
        added_pt.z = z;
        added_pt.intensity = intensity_of(msg, f, i);                              // :246
        added_pt.curvature = field<uint32_t>(msg, f, i, f.off_time) * 1.e-6f;      // :250
        pl_surf.push_back(added_pt);
    }
}

// velodyne_handler, :374-429 with given_offset_time (:279); false: the cloud has no times
bool velodyne(const unsigned char* msg, const Format& f, int plsize, vector<PointType>& pl_surf) {
    if (plsize == 0) return true;                                                  // :268
    if (!(field<float>(msg, f, plsize - 1, f.off_time) > 0)) return false;         // :279
    for (int i = 0; i < plsize; i++) {
        PointType added_pt;
        added_pt.x = field<float>(msg, f, i, f.off_x);
        added_pt.y = field<float>(msg, f, i, f.off_y);
        added_pt.z = field<float>(msg, f, i, f.off_z);
        added_pt.intensity = intensity_of(msg, f, i);                              // :386
        added_pt.curvature = field<float>(msg, f, i, f.off_time) * 1.e-3f;         // :387
        if (i % f.point_filter_num == 0) {                                         // :421
            if (added_pt.x * added_pt.x + added_pt.y * added_pt.y + added_pt.z * added_pt.z > (f.blind * f.blind)) {   // :423
                pl_surf.push_back(added_pt);
            }
        }
    }
    return true;
}

// xt32_handler, :432-464
void xt32(const unsigned char* msg, const Format& f, int plsize, vector<PointType>& pl_surf) {
    if (plsize == 0) return;
    double time_head = field<double>(msg, f, 0, f.off_time);                       // :441
    for (int i = 0; i < plsize; i++) {
        PointType added_pt;
        added_pt.x = field<float>(msg, f, i, f.off_x);
        added_pt.y = field<float>(msg, f, i, f.off_y);
        added_pt.z = field<float>(msg, f, i, f.off_z);
        added_pt.intensity = intensity_of(msg, f, i);                              // :453
        added_pt.curvature = (field<double>(msg, f, i, f.off_time) - time_head) * 1000.f;   // :454
        if (i % f.point_filter_num == 0) {                                         // :456
            if (added_pt.x * added_pt.x + added_pt.y * added_pt.y + added_pt.z * added_pt.z > f.blind) {   // :458
                pl_surf.push_back(added_pt);
            }
        }
    }
}

bool time_list(const PointType& x, const PointType& y) { return (x.curvature < y.curvature); }   // include/common_lib.h

}  // namespace pre

// velodyne_handler (src/preprocess.cpp:259-297, :376-428), both time routes
namespace velo {

enum { kYawDefined = 0, kYawAtan2f = 1 };

struct Pt { float x, y, z, curvature, intensity; };

struct Format {
    int step, off_x, off_y, off_z, off_time, off_ring, N_SCANS, point_filter_num;
    double blind;
    int off_intensity;   // the FLOAT32 intensity; -1: none, PCL leaves 0
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
        added_pt.intensity = f.off_intensity < 0 ? 0.f : field<float>(msg, f, i, f.off_intensity);   // :386
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

}  // namespace velo

extern "C" {

// Preprocess::process into `out` (capacity n 48-byte points), then the sort of sync_packages when do_sort.  fmt: the
// ten ints of Format; off_intensity: the intensity field, or -1.  Returns pl_surf.size(), or -1 for a Velodyne cloud
// without per-point times.
int preo_process_intensity(const int* fmt, int off_intensity, double blind, const unsigned char* msg, int n, int do_sort, float* out) {
    pre::Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], fmt[8], fmt[9], blind, off_intensity};
    vector<pre::PointType> pl_surf;
    pl_surf.reserve(n);
    if (f.kind == 1) pre::avia(msg, f, (unsigned)n, pl_surf);
    else if (f.kind == 3) pre::oust64(msg, f, n, pl_surf);
    else if (f.kind == 2) { if (!pre::velodyne(msg, f, n, pl_surf)) return -1; }
    else pre::xt32(msg, f, n, pl_surf);
    if (do_sort) stable_sort(pl_surf.begin(), pl_surf.end(), pre::time_list);      // src/laserMapping.cpp:551
    if (!pl_surf.empty()) memcpy(out, pl_surf.data(), pl_surf.size() * sizeof(pre::PointType));
    return (int)pl_surf.size();
}

// velodyne_handler into out (n x 4 floats: x, y, z, curvature) and, out_intensity != NULL, each point's intensity (the
// field at off_intensity, or 0 for -1), then the stable time sort when do_sort.  fmt: the eight ints of Format.
// *yaw_times = !given_offset_time (0 for an empty cloud).  Returns pl_surf.size(), or -1 with *bad_ring = the first record
// whose ring is >= N_SCANS on the yaw route.
int velo_process_intensity(const int* fmt, int off_intensity, double blind, const unsigned char* msg, int n, int mode, int do_sort,
                           float* out, float* out_intensity, int* yaw_times, int* bad_ring) {
    velo::Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], blind, off_intensity};
    vector<velo::Pt> pl_surf;
    pl_surf.reserve(n);
    int given = 0;
    *bad_ring = -1;
    if (!velo::velodyne(msg, f, n, mode, pl_surf, &given, bad_ring)) return -1;
    *yaw_times = n > 0 && !given;
    if (do_sort) stable_sort(pl_surf.begin(), pl_surf.end(), velo::time_list);     // src/laserMapping.cpp:551
    for (size_t k = 0; k < pl_surf.size(); ++k) {
        const velo::Pt& q = pl_surf[k];
        out[4 * k] = q.x, out[4 * k + 1] = q.y, out[4 * k + 2] = q.z, out[4 * k + 3] = q.curvature;
        if (out_intensity) out_intensity[k] = q.intensity;
    }
    return (int)pl_surf.size();
}

}  // extern "C"
