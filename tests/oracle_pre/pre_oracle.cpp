// TEST INFRASTRUCTURE -- the checker of flb_lidar_upload / flb_imu_undistort_lidar's window: a plain C++17 restatement,
// op for op, of the non-feature (`else`) branches of Preprocess's four handlers (reference src/preprocess.cpp), of the
// time sort of sync_packages (src/laserMapping.cpp:551, as std::stable_sort: the project defines the order of equal
// times as record order) and of the window at the top of UndistortPcl (src/IMU_Processing.cpp:624-646).  The
// reference's own file needs ROS, PCL and livox_ros_driver, so this is written from its text with line citations; it
// shares no code with the product.  Loaded by tests/pre_oracle.py; never by the product.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

using namespace std;   // the reference's `abs` is std::abs(float) through this

namespace {

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
};

template <typename T>
T field(const unsigned char* msg, const Format& f, size_t i, int off) {
    T v;
    memcpy(&v, msg + i * (size_t)f.step + off, sizeof(T));
    return v;
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
        added_pt.curvature = (field<double>(msg, f, i, f.off_time) - time_head) * 1000.f;   // :454
        if (i % f.point_filter_num == 0) {                                         // :456
            if (added_pt.x * added_pt.x + added_pt.y * added_pt.y + added_pt.z * added_pt.z > f.blind) {   // :458
                pl_surf.push_back(added_pt);
            }
        }
    }
}

bool time_list(const PointType& x, const PointType& y) { return (x.curvature < y.curvature); }   // include/common_lib.h

}  // namespace

extern "C" {

// Preprocess::process into `out` (capacity n 48-byte points), then the sort of sync_packages when do_sort.  fmt: the
// ten ints of Format.  Returns pl_surf.size(), or -1 for a Velodyne cloud without per-point times.
int preo_process(const int* fmt, double blind, const unsigned char* msg, int n, int do_sort, float* out) {
    Format f{fmt[0], fmt[1], fmt[2], fmt[3], fmt[4], fmt[5], fmt[6], fmt[7], fmt[8], fmt[9], blind};
    vector<PointType> pl_surf;
    pl_surf.reserve(n);
    if (f.kind == 1) avia(msg, f, (unsigned)n, pl_surf);
    else if (f.kind == 3) oust64(msg, f, n, pl_surf);
    else if (f.kind == 2) { if (!velodyne(msg, f, n, pl_surf)) return -1; }
    else xt32(msg, f, n, pl_surf);
    if (do_sort) stable_sort(pl_surf.begin(), pl_surf.end(), time_list);           // src/laserMapping.cpp:551
    if (!pl_surf.empty()) memcpy(out, pl_surf.data(), pl_surf.size() * sizeof(PointType));
    return (int)pl_surf.size();
}

// UndistortPcl's window, :624-639: pcl_out (48-byte points, capacity n - index) from lidar_scan_index_now on.  Returns
// pcl_out.size(); the caller advances or resets lidar_scan_index_now (:638, :643-646).
int preo_window(const float* lidar, int n, int lidar_scan_index_now, double pcl_offset_time, float* pcl_out) {
    const PointType* points = reinterpret_cast<const PointType*>(lidar);
    const PointType* pcl_it = points + lidar_scan_index_now;
    const PointType* pcl_it_end = points + n;
    vector<PointType> out;
    while (pcl_it != pcl_it_end && pcl_it->curvature <= pcl_offset_time) {         // :634
        out.push_back(*pcl_it);
        pcl_it++;
    }
    if (pcl_out && !out.empty()) memcpy(pcl_out, out.data(), out.size() * sizeof(PointType));
    return (int)out.size();
}

}  // extern "C"
