// Drives flb::preprocess_velodyne (fastlivo_b200_adapters.hpp) with a mock sensor_msgs::PointCloud2 whose fields are
// looked up by name.  argv[1]: input blob, argv[2]: output blob (formats: tests/test_adapter_velodyne.py).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct PointField { std::string name; uint32_t offset; uint8_t datatype; uint32_t count; };
struct PointCloud2 { uint32_t height, width; std::vector<PointField> fields; uint32_t point_step; std::vector<uint8_t> data; };

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
    auto hdr = rd<int>(f, 9);                         // n, step, off x y z time (-1: no field) ring, n_scans, point_filter_num
    const int n = hdr[0], step = hdr[1];
    auto blind = rd<double>(f, 1);
    auto raw = rd<uint8_t>(f, (size_t)n * step);
    fclose(f);
    flb_handle* h = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &h) != FLB_OK) { fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr)); return 3; }
    try {
        PointCloud2 msg;
        msg.height = 1, msg.width = (uint32_t)n, msg.point_step = (uint32_t)step, msg.data = raw;
        msg.fields = {{"x", (uint32_t)hdr[2], 7, 1}, {"y", (uint32_t)hdr[3], 7, 1}, {"z", (uint32_t)hdr[4], 7, 1},
                      {"intensity", 12, 7, 1}, {"ring", (uint32_t)hdr[6], 4, 1}};
        if (hdr[5] >= 0) msg.fields.push_back({"time", (uint32_t)hdr[5], 7, 1});
        // a field of the wrong datatype is refused before anything is uploaded
        PointCloud2 wrong = msg;
        wrong.fields[4].datatype = 2;                 // ring as UINT8
        int refused = 0;
        try { flb::preprocess_velodyne(h, wrong, hdr[7], blind[0], hdr[8]); } catch (const flb::Error& e) { refused = e.code == FLB_ERR_INVALID; }
        const flb::VelodyneInfo info = flb::preprocess_velodyne(h, msg, hdr[7], blind[0], hdr[8]);
        std::vector<float> cloud((size_t)(info.n_points > 0 ? info.n_points : 1) * 4);
        flb::check(h, flb_lidar_download(h, cloud.data(), info.n_points, nullptr));
        FILE* o = fopen(argv[2], "wb");
        if (!o) return 2;
        const int ints[3] = {info.n_points, info.yaw_times ? 1 : 0, refused};
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
