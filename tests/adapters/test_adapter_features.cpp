// Drives flb::preprocess_features (fastlivo_b200_adapters.hpp) with a mock livox_ros_driver::CustomMsg or a mock
// sensor_msgs::PointCloud2 whose fields are looked up by name.  argv[1]: input blob, argv[2]: output blob (formats:
// tests/test_adapter_features.py).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct CustomPoint { uint32_t offset_time; float x, y, z; uint8_t reflectivity, tag, line; };
struct CustomMsg { uint32_t point_num; std::vector<CustomPoint> points; };
struct PointField { std::string name; uint32_t offset; uint8_t datatype; uint32_t count; };
struct PointCloud2 { uint32_t height, width; std::vector<PointField> fields; uint32_t point_step; std::vector<uint8_t> data; };

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

// 1 when fn throws flb::Error with FLB_ERR_INVALID
template <class F>
static int refused(F fn) {
    try { fn(); } catch (const flb::Error& e) { return e.code == FLB_ERR_INVALID ? 1 : 0; }
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto hdr = rd<int>(f, 10);           // kind, n, step, off x y z time (-1: no field) line/ring, n_scans, point_filter_num
    const int kind = hdr[0], n = hdr[1], step = hdr[2], n_scans = hdr[8], pfn = hdr[9];
    auto blind = rd<double>(f, 1);
    auto raw = rd<uint8_t>(f, (size_t)n * step);
    fclose(f);
    flb_handle* h = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &h) != FLB_OK) { fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr)); return 3; }
    try {
        flb::VelodyneInfo info{};
        int n_refused = 0;
        if (kind == FLB_LIDAR_LIVOX) {
            if (step != (int)sizeof(CustomPoint)) { fprintf(stderr, "record size %d\n", step); return 2; }
            CustomMsg msg;
            msg.point_num = (uint32_t)n;
            msg.points.resize(n);
            if (n) memcpy(msg.points.data(), raw.data(), raw.size());
            const flb::LidarInfo li = flb::preprocess_features(h, msg, n_scans, blind[0], pfn);
            info.n_points = li.n_points, info.last_offset_ms = li.last_offset_ms, info.yaw_times = false;
        } else {
            const bool ouster = kind == FLB_LIDAR_OUSTER;
            PointCloud2 msg;
            msg.height = 1, msg.width = (uint32_t)n, msg.point_step = (uint32_t)step, msg.data = raw;
            msg.fields = {{"x", (uint32_t)hdr[3], 7, 1}, {"y", (uint32_t)hdr[4], 7, 1}, {"z", (uint32_t)hdr[5], 7, 1},
                          {"intensity", 12, 7, 1}, {"ring", (uint32_t)hdr[7], (uint8_t)(ouster ? 2 : 4), 1}};
            if (hdr[6] >= 0) msg.fields.push_back({ouster ? "t" : "time", (uint32_t)hdr[6], (uint8_t)(ouster ? 6 : 7), 1});
            // refused before anything is uploaded: a field of the wrong datatype, a missing field, a kind without a branch
            PointCloud2 wrong = msg;
            wrong.fields[4].datatype = ouster ? 4 : 2;
            n_refused += refused([&] { flb::preprocess_features(h, wrong, kind, n_scans, blind[0], pfn); });
            PointCloud2 missing = msg;
            missing.fields.erase(missing.fields.begin() + 2);   // no z
            n_refused += refused([&] { flb::preprocess_features(h, missing, kind, n_scans, blind[0], pfn); });
            n_refused += refused([&] { flb::preprocess_features(h, msg, FLB_LIDAR_XT32, n_scans, blind[0], pfn); });
            info = flb::preprocess_features(h, msg, kind, n_scans, blind[0], pfn);
        }
        std::vector<float> cloud((size_t)(info.n_points > 0 ? info.n_points : 1) * 4);
        flb::check(h, flb_lidar_download(h, cloud.data(), info.n_points, nullptr));
        FILE* o = fopen(argv[2], "wb");
        if (!o) return 2;
        const int ints[3] = {info.n_points, info.yaw_times ? 1 : 0, n_refused};
        fwrite(ints, sizeof(int), 3, o);
        fwrite(&info.last_offset_ms, sizeof(float), 1, o);
        fwrite(cloud.data(), sizeof(float), (size_t)info.n_points * 4, o);
        fclose(o);
    } catch (const std::exception& e) {
        fprintf(stderr, "error: %s\n", e.what());
        flb_destroy(h);
        return 4;
    }
    flb_destroy(h);
    return 0;
}
