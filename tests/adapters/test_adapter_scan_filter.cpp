// Drives flb::undistort_pcl_on_device + flb::downsample_scan (fastlivo_b200_adapters.hpp) against the host chain
// flb::undistort_pcl -> flb_voxel_grid (a second handle, host in and out) -> flb::upload_scan, with mock stand-ins for
// the reference's sensor_msgs::Imu / pcl cloud / StatesGroup types.  argv[1]: input blob (test_adapter_imu.cpp's format
// followed by the leaf as one double), argv[2]: output blob, per chain: feats_down_size (int32), the scan order (int32
// each), the propagated state (rot, pos, vel: 15 doubles), the carry (7 doubles) (tests/test_adapter_scan_filter.py).
#include <cstdio>
#include <deque>
#include <memory>
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
struct PointXYZINormal { float x, y, z, pad0, nx, ny, nz, pad1, intensity, curvature, pad2, pad3; };
struct Cloud { std::vector<PointXYZINormal> points; };
struct Stamp { double s; double toSec() const { return s; } };
struct Header { Stamp stamp; };
struct V3 { double x, y, z; };
struct ImuMsg { Header header; V3 angular_velocity, linear_acceleration; };

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

static void write_chain(FILE* o, flb_handle* h, int n, const StatesGroup& s, const flb_imu_carry& carry) {
    std::vector<int> order((size_t)n + 1);
    flb::check(h, flb_debug_scan_order(h, order.data(), n + 1));
    fwrite(&n, 4, 1, o);
    fwrite(order.data(), 4, (size_t)n, o);
    double st[15];
    for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) st[3 * i + j] = s.rot_end(i, j); st[9 + i] = s.pos_end(i); st[12 + i] = s.vel_end(i); }
    fwrite(st, 8, 15, o);
    fwrite(&carry, sizeof(carry), 1, o);
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto hdr = rd<int>(f, 2);                         // K n
    const int K = hdr[0], n = hdr[1];
    auto imu = rd<double>(f, (size_t)K * 7);
    auto times = rd<double>(f, 3);                    // pcl_beg pcl_end last_lidar_end
    auto st = rd<double>(f, 9 + 15 + 324);            // rot pos vel bg ba grav cov
    auto carryv = rd<double>(f, 6);                   // acc_s_last angvel_last
    auto prm = rd<double>(f, 12 + 2 + 12);            // cov_gyr cov_acc cov_bias_gyr cov_bias_acc, G norm, R_LI t_LI
    auto pts = rd<float>(f, (size_t)n * 4);           // x y z offset_ms
    const float leaf = (float)rd<double>(f, 1)[0];
    fclose(f);
    flb_handle *hd = nullptr, *hh = nullptr, *scratch = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &hd) != FLB_OK || flb_create(&cfg, &hh) != FLB_OK || flb_create(&cfg, &scratch) != FLB_OK) {
        fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr));
        return 3;
    }
    try {
        std::deque<std::shared_ptr<const ImuMsg>> v_imu;
        for (int k = 0; k < K; ++k) {
            auto m = std::make_shared<ImuMsg>();
            m->header.stamp.s = imu[7 * k];
            m->angular_velocity = V3{imu[7 * k + 1], imu[7 * k + 2], imu[7 * k + 3]};
            m->linear_acceleration = V3{imu[7 * k + 4], imu[7 * k + 5], imu[7 * k + 6]};
            v_imu.push_back(m);
        }
        StatesGroup s0;
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) s0.rot_end(i, j) = st[3 * i + j];
            s0.pos_end(i) = st[9 + i]; s0.vel_end(i) = st[12 + i]; s0.bias_g(i) = st[15 + i]; s0.bias_a(i) = st[18 + i]; s0.gravity(i) = st[21 + i];
        }
        for (int i = 0; i < 18; ++i) for (int j = 0; j < 18; ++j) s0.cov(i, j) = st[24 + 18 * i + j];
        Mat<3, 1> cg, ca, cbg, cba, tLI;
        Mat<3, 3> RLI;
        for (int i = 0; i < 3; ++i) {
            cg(i) = prm[i]; ca(i) = prm[3 + i]; cbg(i) = prm[6 + i]; cba(i) = prm[9 + i]; tLI(i) = prm[23 + i];
            for (int j = 0; j < 3; ++j) RLI(i, j) = prm[14 + 3 * i + j];
        }
        flb_imu_params ip = flb::make_imu_params(cg, ca, cbg, cba, prm[12], prm[13], RLI, tLI);
        flb_imu_carry carry0{};
        carry0.last_lidar_end_time = times[2];
        for (int i = 0; i < 3; ++i) { carry0.acc_s_last[i] = carryv[i]; carry0.angvel_last[i] = carryv[3 + i]; }
        Cloud pc;
        pc.points.resize(n);
        for (int i = 0; i < n; ++i) {
            pc.points[i] = PointXYZINormal{};
            pc.points[i].x = pts[4 * i]; pc.points[i].y = pts[4 * i + 1]; pc.points[i].z = pts[4 * i + 2]; pc.points[i].curvature = pts[4 * i + 3];
        }
        FILE* o = fopen(argv[2], "wb");
        // device chain: feats_undistort stays on the device and becomes the scan there
        StatesGroup sd = s0;
        flb_imu_carry cd = carry0;
        flb::undistort_pcl_on_device(hd, ip, cd, v_imu, times[0], times[1], sd, static_cast<const Cloud&>(pc));
        const int nd = flb::downsample_scan(hd, leaf);
        write_chain(o, hd, nd, sd, cd);
        // host chain: undistort_pcl writes the points back, the filter and the upload go through the host
        StatesGroup sh = s0;
        flb_imu_carry ch = carry0;
        Cloud undist = pc;
        flb::undistort_pcl(hh, ip, ch, v_imu, times[0], times[1], sh, undist);
        std::vector<float> xyz((size_t)n * 3 + 3), down((size_t)n * 3 + 3);
        for (int i = 0; i < n; ++i) { xyz[3 * i] = undist.points[i].x; xyz[3 * i + 1] = undist.points[i].y; xyz[3 * i + 2] = undist.points[i].z; }
        int nh = 0;
        flb::check(scratch, flb_voxel_grid(scratch, xyz.data(), n, 3, leaf, down.data(), n, &nh));
        Cloud feats_down_body;
        feats_down_body.points.resize(nh);
        for (int i = 0; i < nh; ++i) {
            feats_down_body.points[i] = PointXYZINormal{};
            feats_down_body.points[i].x = down[3 * i]; feats_down_body.points[i].y = down[3 * i + 1]; feats_down_body.points[i].z = down[3 * i + 2];
        }
        flb::upload_scan(hh, feats_down_body);
        write_chain(o, hh, nh, sh, ch);
        fclose(o);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 4;
    }
    flb_destroy(hd);
    flb_destroy(hh);
    flb_destroy(scratch);
    return 0;
}
