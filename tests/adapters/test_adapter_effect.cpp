// TEST: flb::publish_effect_world (fast-livo_b200/adapters/fastlivo_b200_adapters.hpp), both overloads, against mock
// Eigen-shaped types (column-major, like Eigen's default; an MTK SO3 stand-in with only toRotationMatrix()) and a mock
// PCL cloud.  Reads the map, scan, prior pose and extrinsic the pytest driver dumped; on one handle runs
//   flb::lio_update at the prior, then
//   A: the 18-DoF overload  -- publish_effect_world(h, lio_prm, cloud), at the device state
//   B: the IKFoM overload   -- publish_effect_world(h, prm, s.rot.toRotationMatrix(), s.pos, cloud), extrinsic from
//                              offset_*_L_I, at the prior pose
// and writes both clouds (count, xyz) and the posterior state for comparison with the ABI's effect cloud.
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
struct Cloud {         // pcl::PointCloud<PointXYZINormal>: resize() keeps width / height in step with points
    std::vector<PointXYZINormal> points;
    unsigned width = 0, height = 1;
    void resize(size_t n) { points.resize(n); width = (unsigned)n; height = 1; }
};
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

static void dump_cloud(const Cloud& c, FILE* o) {
    const int n = (int)c.points.size();
    if (c.width != (unsigned)n || c.height != 1) { fprintf(stderr, "cloud shape\n"); exit(3); }
    fwrite(&n, sizeof(int), 1, o);
    for (const auto& q : c.points) {
        const float xyz[3] = {q.x, q.y, q.z};
        fwrite(xyz, sizeof(float), 3, o);
    }
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    auto hdr = rd<int>(f, 2);   // M N
    const int M = hdr[0], N = hdr[1];
    auto map = rd<float>(f, (size_t)M * 3);
    auto scan = rd<float>(f, (size_t)N * 3);
    auto pose = rd<double>(f, 9 + 3 + 9 + 3);             // R p R_LI t_LI (row-major)
    fclose(f);
    Cloud feats_down_body;
    feats_down_body.resize(N);
    for (int i = 0; i < N; ++i) {
        feats_down_body.points[i] = PointXYZINormal{};
        feats_down_body.points[i].x = scan[3 * i]; feats_down_body.points[i].y = scan[3 * i + 1]; feats_down_body.points[i].z = scan[3 * i + 2];
    }
    Mat<3, 3> R, R_LI;
    Mat<3, 1> p, t_LI;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) { R(i, j) = pose[3 * i + j]; R_LI(i, j) = pose[12 + 3 * i + j]; }
        p(i) = pose[9 + i];
        t_LI(i) = pose[21 + i];
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
        flb::check(h, flb_map_upload(h, map.data(), M, 3));
        flb::upload_scan(h, feats_down_body);
        StatesGroup s{};
        s.rot_end = R;
        s.pos_end = p;
        for (int i = 0; i < 18; ++i) s.cov(i, i) = 1e-3;
        const StatesGroup prior = s;
        const flb_lio_params lio_prm = flb::make_lio_params(R_LI, t_LI, 0.001, 3);
        flb::lio_update(h, lio_prm, s, prior);
        // A: 18-DoF -- the pose is the device state
        Cloud a;
        flb::publish_effect_world(h, lio_prm, a);
        dump_cloud(a, o);
        // B: IKFoM -- explicit pose and extrinsic from state_ikfom
        StateIkfom k{};
        k.rot.R = R;
        k.pos = p;
        k.offset_R_L_I.R = R_LI;
        k.offset_T_L_I = t_LI;
        const flb_lio_params prm = flb::make_lio_params(k.offset_R_L_I.toRotationMatrix(), k.offset_T_L_I, 0.001, 3);
        Cloud b;
        flb::publish_effect_world(h, prm, k.rot.toRotationMatrix(), k.pos, b);
        dump_cloud(b, o);
        flb_state18 x;
        flb::to_abi(s, x);
        fwrite(x.rot, sizeof(double), 9, o);
        fwrite(x.pos, sizeof(double), 3, o);
        flb_destroy(h);
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 1;
    }
    fclose(o);
    return 0;
}
