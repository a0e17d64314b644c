// TEST: flb::publish_frame_world_rgb and flb::save_rgb_map (fast-livo_b200/adapters/fastlivo_b200_adapters.hpp) against
// a mock pcl::PointXYZRGB (32 bytes: x y z data[3], then the b g r a / rgb / rgba union, PCL 1.8's defaults) and a mock
// PCL cloud.  Reads the camera, a BGR frame, a body scan, the world pose, the extrinsic and the camera pose the pytest
// driver dumped; on one handle uploads the frame and the scan, builds the world cloud, opens a save and
//   A: publish_frame_world_rgb(h, Rcw, Pcw, cloud) twice (the save holds both frames)
//   B: save_rgb_map(h, cloud)
//   C: a save capped at one point: the frame is dropped, so save_rgb_map must throw
// and writes A, B (count, 32-byte records) and whether C threw.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

template <int R, int C>
struct Mat {
    double v[R * C] = {0};
    double& operator()(int i, int j) { return v[j * R + i]; }
    double operator()(int i, int j) const { return v[j * R + i]; }
    double& operator()(int i) { return v[i]; }
    double operator()(int i) const { return v[i]; }
};
struct alignas(16) PointXYZRGB {   // pcl::PointXYZRGB: PCL_ADD_POINT4D, PCL_ADD_RGB, EIGEN_ALIGN16
    union {
        float data[4];
        struct { float x, y, z; };
    };
    union {
        union {
            struct { uint8_t b, g, r, a; };
            float rgb;
        };
        uint32_t rgba;
    };
    PointXYZRGB() : x(0.f), y(0.f), z(0.f) {
        data[3] = 1.0f;
        rgba = 0;
        a = 255;
    }
};
struct Cloud {         // pcl::PointCloud<PointXYZRGB>: resize() keeps width / height in step with points
    std::vector<PointXYZRGB> points;
    unsigned width = 0, height = 1;
    void resize(size_t n) { points.resize(n); width = (unsigned)n; height = 1; }
};

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (n && fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

static void dump_cloud(const Cloud& c, FILE* o) {
    const int n = (int)c.points.size();
    if (c.width != (unsigned)n || c.height != 1) { fprintf(stderr, "cloud shape\n"); exit(3); }
    fwrite(&n, sizeof(int), 1, o);
    if (n) fwrite(c.points.data(), sizeof(PointXYZRGB), (size_t)n, o);
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto wh = rd<int>(f, 2);
    auto camv = rd<double>(f, 9);                          // fx fy cx cy d0..d4
    const int W = wh[0], H = wh[1];
    auto img = rd<uint8_t>(f, (size_t)W * H * 3);
    const int N = rd<int>(f, 1)[0];
    auto scan = rd<float>(f, (size_t)N * 3);
    auto pose = rd<double>(f, 3 * 12);                     // R p | R_LI t_LI | Rcw Pcw (row-major)
    fclose(f);
    Mat<3, 3> R_LI, Rcw;
    Mat<3, 1> t_LI, Pcw;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) { R_LI(i, j) = pose[12 + 3 * i + j]; Rcw(i, j) = pose[24 + 3 * i + j]; }
        t_LI(i) = pose[21 + i];
        Pcw(i) = pose[33 + i];
    }
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    try {
        flb_config cfg{};
        cfg.device = 0;
        cfg.cell_size = 0.6;
        cfg.knn_max_d2 = 5.0;
        cfg.plane_threshold = 0.1;
        cfg.persistent = 1;
        flb_handle* h = nullptr;
        flb::check(nullptr, flb_create(&cfg, &h));
        flb_camera cam{};
        cam.width = W;
        cam.height = H;
        cam.fx = camv[0]; cam.fy = camv[1]; cam.cx = camv[2]; cam.cy = camv[3];
        for (int k = 0; k < 5; ++k) cam.d[k] = camv[4 + k];
        flb::check(h, flb_camera_set(h, &cam));
        flb::check(h, flb_image_upload_bgr(h, img.data(), W, H, 3 * W, 0));
        flb::check(h, flb_scan_upload(h, scan.data(), N, 3));
        const flb_lio_params prm = flb::make_lio_params(R_LI, t_LI, 0.001, 3);
        flb::check(h, flb_world_cloud(h, &prm, pose.data(), pose.data() + 9, FLB_CLOUD_SCAN, nullptr));
        flb::check(h, flb_rgb_save_begin(h, (int64_t)1 << 30));
        Cloud a;
        flb::publish_frame_world_rgb(h, Rcw, Pcw, a);
        flb::publish_frame_world_rgb(h, Rcw, Pcw, a);
        dump_cloud(a, o);
        Cloud b;
        flb::save_rgb_map(h, b);
        dump_cloud(b, o);
        flb::check(h, flb_rgb_save_end(h));
        flb::check(h, flb_rgb_save_begin(h, 1));
        Cloud c;
        flb::publish_frame_world_rgb(h, Rcw, Pcw, c);
        int threw = 0;
        try {
            flb::save_rgb_map(h, c);
        } catch (const flb::Error& e) {
            threw = e.code == FLB_ERR_STATE ? 1 : 2;
        }
        fwrite(&threw, sizeof(int), 1, o);
        flb::check(h, flb_rgb_save_end(h));
        flb_destroy(h);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 1;
    }
    fclose(o);
    return 0;
}
