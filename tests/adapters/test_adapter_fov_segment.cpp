// TEST: flb::lasermap_fov_segment (fast-livo_b200/adapters/fastlivo_b200_adapters.hpp), both overloads, against mock
// Eigen-shaped types.  Reads the map, cube_side_length and a sensor trajectory the pytest driver dumped, runs it on two
// handles
//   A: the 18-DoF path  -- StatesGroup (pos_end = the frame's position) uploaded as the device state, then
//                          lasermap_fov_segment(h, cube_len, &kdtree_delete_counter); the first frame passes nullptr
//                          for the counter (the plain overload, not the position template)
//   B: the IKFoM path   -- lasermap_fov_segment(h, cube_len, pos_lid, &kdtree_delete_counter) with a Vec3 pos_lid
// and writes each frame's deleted count of A and B, then both final maps.
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
struct StatesGroup {   // include/common_lib.h:296-381
    Mat<3, 3> rot_end;
    Mat<3, 1> pos_end, vel_end, bias_g, bias_a, gravity;
    Mat<18, 18> cov;
};

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

static flb_handle* make_handle(const std::vector<float>& map, int M) {
    flb_config cfg{};
    cfg.device = 0;
    cfg.cell_size = 0.6;
    cfg.knn_max_d2 = 5.0;
    cfg.plane_threshold = 0.1;
    cfg.persistent = 1;
    flb_handle* h = nullptr;
    flb::check(nullptr, flb_create(&cfg, &h));
    flb::check(h, flb_map_upload(h, map.data(), M, 3));
    return h;
}

static void dump_map(flb_handle* h, FILE* o) {
    const int m = flb_map_size(h);
    std::vector<float> out((size_t)m * 3);
    int got = 0;
    flb::check(h, flb_map_download(h, out.data(), m, &got));
    fwrite(&m, sizeof(int), 1, o);
    fwrite(out.data(), sizeof(float), out.size(), o);
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto hdr = rd<int>(f, 2);   // M, frames
    const int M = hdr[0], K = hdr[1];
    auto map = rd<float>(f, (size_t)M * 3);
    const double cube_len = rd<double>(f, 1)[0];
    auto traj = rd<double>(f, (size_t)K * 3);
    fclose(f);
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    try {
        flb_handle* a = make_handle(map, M);
        flb_handle* b = make_handle(map, M);
        std::vector<int> cnt_a(K, 0), cnt_b(K, 0);
        for (int k = 0; k < K; ++k) {
            StatesGroup s{};
            for (int i = 0; i < 3; ++i) { s.rot_end(i, i) = 1.0; s.pos_end(i) = traj[3 * k + i]; }
            for (int i = 0; i < 18; ++i) s.cov(i, i) = 1e-3;
            flb_state18 x;
            flb::to_abi(s, x);
            flb::check(a, flb_state_upload(a, &x, &x));
            if (k == 0) flb::lasermap_fov_segment(a, cube_len, nullptr);
            else flb::lasermap_fov_segment(a, cube_len, &cnt_a[k]);
            Mat<3, 1> pos_lid;
            for (int i = 0; i < 3; ++i) pos_lid(i) = traj[3 * k + i];
            flb::lasermap_fov_segment(b, cube_len, pos_lid, &cnt_b[k]);
        }
        fwrite(cnt_a.data(), sizeof(int), K, o);
        fwrite(cnt_b.data(), sizeof(int), K, o);
        dump_map(a, o);
        dump_map(b, o);
        flb_destroy(a);
        flb_destroy(b);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 1;
    }
    fclose(o);
    return 0;
}
