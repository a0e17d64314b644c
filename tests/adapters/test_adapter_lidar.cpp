// Drives flb::preprocess (both overloads) and flb::undistort_pcl_from_lidar (fastlivo_b200_adapters.hpp) with mock
// stand-ins for livox_ros_driver::CustomMsg, sensor_msgs::PointCloud2, sensor_msgs::Imu, LidarMeasureGroup and
// StatesGroup.  argv[1]: input blob, argv[2]: output blob (formats: tests/test_adapter_lidar.py).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <deque>
#include <memory>
#include <string>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

template <int R, int C>
struct Mat {   // column-major, like Eigen's default
    double v[R * C] = {0};
    double& operator()(int i, int j) { return v[j * R + i]; }
    double operator()(int i, int j) const { return v[j * R + i]; }
    double& operator()(int i) { return v[i]; }
    double operator()(int i) const { return v[i]; }
};
struct StatesGroup { Mat<3, 3> rot_end; Mat<3, 1> pos_end, vel_end, bias_g, bias_a, gravity; Mat<18, 18> cov; };
struct Stamp { double s; double toSec() const { return s; } };
struct Header { Stamp stamp; };
struct V3 { double x, y, z; };
struct ImuMsg { Header header; V3 angular_velocity, linear_acceleration; };
struct CustomPoint { uint32_t offset_time; float x, y, z; uint8_t reflectivity, tag, line; };   // livox_ros_driver
static_assert(sizeof(CustomPoint) == 20, "CustomPoint layout");
struct CustomMsg { uint32_t point_num; std::vector<CustomPoint> points; };
struct PointField { std::string name; uint32_t offset; uint8_t datatype; uint32_t count; };
struct PointCloud2 { uint32_t height, width; std::vector<PointField> fields; uint32_t point_step; std::vector<uint8_t> data; };
struct MeasureGroup { double img_offset_time; };
struct LidarMeasureGroup {   // include/common_lib.h
    double lidar_beg_time, last_update_time;
    std::deque<MeasureGroup> measures;
    bool is_lidar_end;
    int lidar_scan_index_now;
};

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto hdr = rd<int>(f, 10);                        // K, kind, n, step, off x y z time, n_scans, point_filter_num
    const int K = hdr[0], kind = hdr[1], n = hdr[2], step = hdr[3];
    auto dbl = rd<double>(f, 3);                      // blind, lidar_beg_time, img_offset_time
    auto imu = rd<double>(f, (size_t)K * 7);
    auto st = rd<double>(f, 9 + 15 + 324);            // rot pos vel bg ba grav cov
    auto carryv = rd<double>(f, 7);                   // last_lidar_end_time acc_s_last angvel_last
    auto prm = rd<double>(f, 12 + 2 + 12);            // cov_gyr cov_acc cov_bias_gyr cov_bias_acc, G norm, R_LI t_LI
    auto raw = rd<uint8_t>(f, (size_t)n * step);
    fclose(f);
    flb_handle* h = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &h) != FLB_OK) { fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr)); return 3; }
    try {
        flb::LidarInfo info;
        if (kind == FLB_LIDAR_LIVOX) {
            CustomMsg msg;
            msg.point_num = (uint32_t)n;
            msg.points.resize(n);
            memcpy(msg.points.data(), raw.data(), raw.size());
            info = flb::preprocess(h, msg, hdr[8], dbl[0], hdr[9]);
        } else {
            PointCloud2 msg;
            msg.height = 1, msg.width = (uint32_t)n, msg.point_step = (uint32_t)step, msg.data = raw;
            const char* tn = kind == FLB_LIDAR_OUSTER ? "t" : (kind == FLB_LIDAR_VELODYNE ? "time" : "timestamp");
            msg.fields = {{"x", (uint32_t)hdr[4], 7, 1}, {"y", (uint32_t)hdr[5], 7, 1}, {"intensity", 16, 7, 1},
                          {"z", (uint32_t)hdr[6], 7, 1}, {tn, (uint32_t)hdr[7], 6, 1}, {"ring", 26, 2, 1}};
            info = flb::preprocess(h, msg, kind, hdr[8], dbl[0], hdr[9]);
        }
        std::vector<float> cloud((size_t)(info.n_points > 0 ? info.n_points : 1) * 4);
        int n_dl = 0;
        flb::check(h, flb_lidar_download(h, cloud.data(), info.n_points, &n_dl));

        std::deque<std::shared_ptr<const ImuMsg>> v_imu;
        for (int k = 0; k < K; ++k) {
            auto m = std::make_shared<ImuMsg>();
            m->header.stamp.s = imu[7 * k];
            m->angular_velocity = V3{imu[7 * k + 1], imu[7 * k + 2], imu[7 * k + 3]};
            m->linear_acceleration = V3{imu[7 * k + 4], imu[7 * k + 5], imu[7 * k + 6]};
            v_imu.push_back(m);
        }
        StatesGroup s;
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) s.rot_end(i, j) = st[3 * i + j];
            s.pos_end(i) = st[9 + i]; s.vel_end(i) = st[12 + i]; s.bias_g(i) = st[15 + i]; s.bias_a(i) = st[18 + i]; s.gravity(i) = st[21 + i];
        }
        for (int i = 0; i < 18; ++i) for (int j = 0; j < 18; ++j) s.cov(i, j) = st[24 + 18 * i + j];
        Mat<3, 1> cg, ca, cbg, cba, tLI;
        Mat<3, 3> RLI;
        for (int i = 0; i < 3; ++i) {
            cg(i) = prm[i]; ca(i) = prm[3 + i]; cbg(i) = prm[6 + i]; cba(i) = prm[9 + i]; tLI(i) = prm[23 + i];
            for (int j = 0; j < 3; ++j) RLI(i, j) = prm[14 + 3 * i + j];
        }
        flb_imu_params ip = flb::make_imu_params(cg, ca, cbg, cba, prm[12], prm[13], RLI, tLI);
        flb_imu_carry carry{};
        carry.last_lidar_end_time = carryv[0];
        for (int i = 0; i < 3; ++i) { carry.acc_s_last[i] = carryv[1 + i]; carry.angvel_last[i] = carryv[4 + i]; }
        // one camera update, then the scan end (sync_packages' two kinds of measures)
        LidarMeasureGroup lm{dbl[1], 0.0, {MeasureGroup{dbl[2]}}, false, 0};
        int taken[2], index_after[2];
        double update_time[2];
        for (int u = 0; u < 2; ++u) {
            lm.is_lidar_end = (u == 1);
            taken[u] = flb::undistort_pcl_from_lidar(h, ip, carry, v_imu, lm, info.last_offset_ms, s);
            index_after[u] = lm.lidar_scan_index_now;
            update_time[u] = lm.last_update_time;
        }
        int n_scan = flb::downsample_scan(h, 0.5f);
        FILE* o = fopen(argv[2], "wb");
        int head[7] = {info.n_points, n_dl, taken[0], taken[1], index_after[0], index_after[1], n_scan};
        fwrite(head, 4, 7, o);
        fwrite(&info.last_offset_ms, 4, 1, o);
        fwrite(update_time, 8, 2, o);
        double out[15];
        for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) out[3 * i + j] = s.rot_end(i, j); out[9 + i] = s.pos_end(i); out[12 + i] = s.vel_end(i); }
        fwrite(out, 8, 15, o);
        fwrite(cloud.data(), 16, (size_t)info.n_points, o);
        fclose(o);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 4;
    }
    flb_destroy(h);
    return 0;
}
