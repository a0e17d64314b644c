// TEST: flb::map_incremental (fast-livo_b200/adapters/fastlivo_b200_adapters.hpp), both overloads, against mock
// Eigen-shaped types (column-major, like Eigen's default; an MTK SO3 stand-in with only toRotationMatrix()).
// Reads the map, scan, pose and extrinsic the pytest driver dumped, runs on two handles
//   A: the 18-DoF path   -- StatesGroup uploaded as the device state, map_incremental(h, lio_prm, ds)
//   B: the IKFoM path    -- map_incremental(h, prm, s.rot.toRotationMatrix(), s.pos, ds), extrinsic from offset_*_L_I
// and writes both resulting maps for comparison with flb_map_add_points on the oracle-transformed scan.
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
struct PointXYZINormal { float x, y, z, pad0, nx, ny, nz, pad1, intensity, curvature, pad2, pad3; };
struct Cloud { std::vector<PointXYZINormal> points; };
struct Quat {          // MTK SO3 stand-in
    Mat<3, 3> R;
    Mat<3, 3> toRotationMatrix() const { return R; }
};
struct StateIkfom { Mat<3, 1> pos; Quat rot, offset_R_L_I; Mat<3, 1> offset_T_L_I; };

template <class T>
static std::vector<T> rd(FILE* f, size_t n) {
    std::vector<T> v(n);
    if (fread(v.data(), sizeof(T), n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
    return v;
}

static flb_handle* make_handle(const std::vector<float>& map, int M, const Cloud& scan) {
    flb_config cfg{};
    cfg.device = 0;
    cfg.cell_size = 0.6;
    cfg.knn_max_d2 = 5.0;
    cfg.plane_threshold = 0.1;
    cfg.persistent = 1;
    flb_handle* h = nullptr;
    flb::check(nullptr, flb_create(&cfg, &h));
    flb::check(h, flb_map_upload(h, map.data(), M, 3));
    flb::upload_scan(h, scan);
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
    auto hdr = rd<int>(f, 2);   // M N
    const int M = hdr[0], N = hdr[1];
    auto map = rd<float>(f, (size_t)M * 3);
    auto scan = rd<float>(f, (size_t)N * 3);
    auto pose = rd<double>(f, 9 + 3 + 9 + 3 + 1);         // R p R_LI t_LI (row-major) downsample_size
    fclose(f);
    Cloud cloud;
    cloud.points.resize(N);
    for (int i = 0; i < N; ++i) {
        cloud.points[i] = PointXYZINormal{};
        cloud.points[i].x = scan[3 * i]; cloud.points[i].y = scan[3 * i + 1]; cloud.points[i].z = scan[3 * i + 2];
    }
    Mat<3, 3> R, R_LI;
    Mat<3, 1> p, t_LI;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) { R(i, j) = pose[3 * i + j]; R_LI(i, j) = pose[12 + 3 * i + j]; }
        p(i) = pose[9 + i];
        t_LI(i) = pose[21 + i];
    }
    const float ds = (float)pose[24];
    FILE* o = fopen(argv[2], "wb");
    if (!o) return 2;
    try {
        // A: 18-DoF -- the pose is the device state
        flb_handle* a = make_handle(map, M, cloud);
        StatesGroup s{};
        s.rot_end = R;
        s.pos_end = p;
        for (int i = 0; i < 18; ++i) s.cov(i, i) = 1e-3;
        flb_state18 x;
        flb::to_abi(s, x);
        flb::check(a, flb_state_upload(a, &x, &x));
        const flb_lio_params lio_prm = flb::make_lio_params(R_LI, t_LI, 0.001, 3);
        flb::map_incremental(a, lio_prm, ds);
        dump_map(a, o);
        flb_destroy(a);
        // B: IKFoM -- explicit pose and extrinsic from state_ikfom
        flb_handle* b = make_handle(map, M, cloud);
        StateIkfom k{};
        k.rot.R = R;
        k.pos = p;
        k.offset_R_L_I.R = R_LI;
        k.offset_T_L_I = t_LI;
        const flb_lio_params prm = flb::make_lio_params(k.offset_R_L_I.toRotationMatrix(), k.offset_T_L_I, 0.001, 3);
        flb::map_incremental(b, prm, k.rot.toRotationMatrix(), k.pos, ds);
        dump_map(b, o);
        flb_destroy(b);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 1;
    }
    fclose(o);
    return 0;
}
