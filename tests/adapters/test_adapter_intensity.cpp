// TEST: the intensity adapters (fast-livo_b200/adapters/fastlivo_b200_adapters.hpp): flb::preprocess of a mock Livox
// CustomMsg and of mock PointCloud2 messages whose intensity is FLOAT32, UINT16 (PCL leaves 0) or absent (0), then
// flb::publish_frame_world and flb::save_intensity_map into a mock PointCloudXYZI (48-byte pcl::PointXYZINormal with
// PCL's defaults).  Reads what the pytest driver dumped: the Livox records, the Ouster records (48 bytes, intensity at
// 16), the IMU inputs, the state, the LIO extrinsic and a world pose.  Writes, each as (count, 48-byte records):
//   A  flb_lidar_download_points after preprocess(livox)
//   B  ... after preprocess(ouster, intensity FLOAT32),  C  ... UINT16,  D  ... without an intensity field
//   E  publish_frame_world after B's cloud is undistorted whole and transformed (a save is open)
//   F  save_intensity_map after E was published twice
// then whether save_intensity_map threw on a save capped below one frame.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct CustomPoint { uint32_t offset_time; float x, y, z; uint8_t reflectivity, tag, line; };   // livox_ros_driver
struct CustomMsg { uint32_t point_num; std::vector<CustomPoint> points; };
struct PointField { std::string name; uint32_t offset; uint8_t datatype; uint32_t count; };
struct PointCloud2 { uint32_t height, width; std::vector<PointField> fields; uint32_t point_step; std::vector<uint8_t> data; };
struct alignas(16) PointXYZINormal {   // pcl::PointXYZINormal: PCL_ADD_POINT4D, PCL_ADD_NORMAL4D, intensity, curvature
    union {
        float data[4];
        struct { float x, y, z; };
    };
    union {
        float data_n[4];
        struct { float normal_x, normal_y, normal_z; };
    };
    union {
        struct { float intensity, curvature; };
        float data_c[4];
    };
    PointXYZINormal() : x(0.f), y(0.f), z(0.f), normal_x(0.f), normal_y(0.f), normal_z(0.f) {
        data[3] = 1.0f;
        data_n[3] = 0.f;
        intensity = curvature = 0.f;
        data_c[2] = data_c[3] = 0.f;
    }
};
struct Cloud {         // pcl::PointCloud<PointXYZINormal>
    std::vector<PointXYZINormal> points;
    unsigned width = 0, height = 1;
    void resize(size_t n) { points.resize(n); width = (unsigned)n; height = 1; }
};

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}
static int rd_int(FILE* f) { return rd<int>(f, 1)[0]; }

static void dump_records(const std::vector<float>& rec, int n, FILE* o) {
    fwrite(&n, sizeof(int), 1, o);
    if (n) fwrite(rec.data(), 48, (size_t)n, o);
}
static void dump_current(flb_handle* h, FILE* o) {
    int n = 0;
    flb::check(h, flb_lidar_download_points(h, nullptr, 0, &n));
    std::vector<float> rec((size_t)n * 12);
    flb::check(h, flb_lidar_download_points(h, rec.data(), n, &n));
    dump_records(rec, n, o);
}
static void dump_cloud(const Cloud& c, FILE* o) {
    const int n = (int)c.points.size();
    if (c.width != (unsigned)n || c.height != 1) { fprintf(stderr, "cloud shape\n"); exit(3); }
    fwrite(&n, sizeof(int), 1, o);
    if (n) fwrite(c.points.data(), sizeof(PointXYZINormal), (size_t)n, o);
}

static PointCloud2 ouster_msg(const std::vector<uint8_t>& data, int n, int intensity_type) {
    PointCloud2 m;
    m.height = 1;
    m.width = (uint32_t)n;
    m.point_step = 48;
    m.fields = {{"x", 0, 7, 1}, {"y", 4, 7, 1}, {"z", 8, 7, 1}, {"t", 20, 6, 1}, {"ring", 26, 2, 1}};
    if (intensity_type) m.fields.push_back({"intensity", 16, (uint8_t)intensity_type, 1});
    m.data = data;
    return m;
}

int main(int argc, char** argv) {
    static_assert(sizeof(CustomPoint) == 20 && offsetof(CustomPoint, reflectivity) == 16, "CustomPoint layout");
    if (argc != 3) return 1;
    FILE* in = fopen(argv[1], "rb");
    FILE* out = fopen(argv[2], "wb");
    if (!in || !out) return 1;
    CustomMsg livox;
    livox.point_num = (uint32_t)rd_int(in);
    livox.points = rd<CustomPoint>(in, livox.point_num);
    const int n_ouster = rd_int(in);
    const std::vector<uint8_t> ouster = rd<uint8_t>(in, (size_t)n_ouster * 48);
    const flb_imu_params prm = rd<flb_imu_params>(in, 1)[0];
    flb_imu_carry carry = rd<flb_imu_carry>(in, 1)[0];
    const int n_imu = rd_int(in);
    const std::vector<flb_imu_sample> imu = rd<flb_imu_sample>(in, (size_t)n_imu);
    const std::vector<double> t = rd<double>(in, 2);
    const flb_state18 x = rd<flb_state18>(in, 1)[0];
    const flb_lio_params lio = rd<flb_lio_params>(in, 1)[0];
    const std::vector<double> pose = rd<double>(in, 12);
    fclose(in);
    flb_config cfg{};
    cfg.device = 0;
    cfg.cell_size = 0.6;
    cfg.knn_max_d2 = 5.0;
    cfg.plane_threshold = 0.1;
    cfg.persistent = 1;
    flb_handle* h = nullptr;
    if (flb_create(&cfg, &h) != FLB_OK) { fprintf(stderr, "flb_create\n"); return 4; }
    try {
        flb::preprocess(h, livox, 6, 0.5, 1);                                            // A
        dump_current(h, out);
        for (int type : {7, 4, 0}) {                                                     // B, C, D
            PointCloud2 m = ouster_msg(ouster, n_ouster, type);
            const flb::LidarInfo r = flb::preprocess(h, m, FLB_LIDAR_OUSTER, 64, 0.8, 1);
            if (r.n_points < 2) { fprintf(stderr, "empty cloud\n"); return 5; }
            dump_current(h, out);
        }
        PointCloud2 m = ouster_msg(ouster, n_ouster, 7);
        flb::preprocess(h, m, FLB_LIDAR_OUSTER, 64, 0.8, 1);
        flb::check(h, flb_state_upload(h, &x, &x));
        int taken = 0;
        flb::check(h, flb_imu_undistort_lidar(h, &prm, &carry, imu.data(), n_imu, t[0], t[1], 1e9, 1, &taken, nullptr, 0, nullptr, nullptr));
        int n = 0;
        flb::check(h, flb_world_cloud(h, &lio, pose.data(), pose.data() + 9, FLB_CLOUD_UNDISTORTED, &n));
        flb::check(h, flb_lidar_save_begin(h, 1 << 30));
        Cloud pub, saved;
        flb::publish_frame_world(h, pub);
        flb::publish_frame_world(h, pub);
        dump_cloud(pub, out);                                                            // E
        flb::save_intensity_map(h, saved);
        dump_cloud(saved, out);                                                          // F
        flb::check(h, flb_lidar_save_end(h));
        flb::check(h, flb_lidar_save_begin(h, 1));
        flb::publish_frame_world(h, pub);
        int threw = 0;
        try {
            flb::save_intensity_map(h, saved);
        } catch (const flb::Error&) {
            threw = 1;
        }
        fwrite(&threw, sizeof(int), 1, out);
    } catch (const std::exception& e) {
        fprintf(stderr, "adapter error: %s\n", e.what());
        return 6;
    }
    flb_destroy(h);
    fclose(out);
    return 0;
}
