/* TEST INFRASTRUCTURE -- NOT PRODUCT CODE (see flo_oracle.h).
 *
 * flo_visual_candidates: CPU restatement of the scoring loop of LidarSelector::addSparseMap
 * (reference src/lidar_selection.cpp:150-168; SURVEY.md section 8 row f4): every scan point is projected into the
 * new frame, scored with vikit's Shi-Tomasi corner score and competes for its image-grid cell.
 * vikit (uzh-rpg/rpg_vikit, vikit_common/src/vision.cpp: shiTomasiScore; abstract_camera.h: isInFrame;
 * pinhole_camera.cpp: world2cam) is a third-party dependency absent from the reference tree; its published
 * algorithm is restated here (SURVEY.md Appendix C).  PARITY STATUS: "parity unpinned".
 */
#include <cmath>
#include <cstdint>

#include "flo_oracle.h"

/* vk::shiTomasiScore(const cv::Mat& img, int u, int v): 8x8 box of central differences, smaller eigenvalue of
 * the (normalised) structure tensor.  All sums are integers < 2^24, i.e. exact in float. */
extern "C" float flo_shi_tomasi(const uint8_t* img, int width, int height, int stride, int u, int v) {
    float dXX = 0.0f, dYY = 0.0f, dXY = 0.0f;
    const int halfbox_size = 4;
    const int box_size = 2 * halfbox_size;
    const int box_area = box_size * box_size;
    const int x_min = u - halfbox_size, x_max = u + halfbox_size, y_min = v - halfbox_size, y_max = v + halfbox_size;
    if (x_min < 1 || x_max >= width - 1 || y_min < 1 || y_max >= height - 1) return 0.0f;   /* too close to the border */
    for (int y = y_min; y < y_max; ++y) {
        const uint8_t* ptr_left = img + stride * y + x_min - 1;
        const uint8_t* ptr_right = img + stride * y + x_min + 1;
        const uint8_t* ptr_top = img + stride * (y - 1) + x_min;
        const uint8_t* ptr_bottom = img + stride * (y + 1) + x_min;
        for (int x = 0; x < box_size; ++x, ++ptr_left, ++ptr_right, ++ptr_top, ++ptr_bottom) {
            const float dx = (float)(*ptr_right - *ptr_left);
            const float dy = (float)(*ptr_bottom - *ptr_top);
            dXX += dx * dx;
            dYY += dy * dy;
            dXY += dx * dy;
        }
    }
    /* find and return the smaller eigenvalue */
    dXX = (float)(dXX / (2.0 * box_area));
    dYY = (float)(dYY / (2.0 * box_area));
    dXY = (float)(dXY / (2.0 * box_area));
    return (float)(0.5 * (dXX + dYY - std::sqrt((dXX + dYY) * (dXX + dYY) - 4 * (dXX * dYY - dXY * dXY))));
}

/* addSparseMap's first loop, src/lidar_selection.cpp:150-168.  map_value (length = grid_n_width * grid_n_height)
 * is in/out: addFromSparseMap has already written the scores of the visible map points into it (:447-455).
 * winner[cell] = index of the scan point that took the cell in this call, -1 otherwise. */
extern "C" void flo_visual_candidates(const flo_cam* cam, const double* Rcw, const double* Pcw, const uint8_t* img, int stride,
                                      const float* world_xyz, int n, int grid_size, int border, float* map_value,
                                      int* winner) {
    const int grid_n_width = cam->width / grid_size, grid_n_height = cam->height / grid_size;   /* :55-56 */
    for (int c = 0; c < grid_n_width * grid_n_height; ++c) winner[c] = -1;
    for (int i = 0; i < n; ++i) {
        const double pt[3] = {world_xyz[3 * i], world_xyz[3 * i + 1], world_xyz[3 * i + 2]};
        double pf[3], pc[2];
        for (int k = 0; k < 3; ++k) pf[k] = Rcw[3 * k] * pt[0] + Rcw[3 * k + 1] * pt[1] + Rcw[3 * k + 2] * pt[2] + Pcw[k];   /* T_f_w * pt */
        flo_world2cam(cam, pf, pc);                                                  /* Frame::w2c, include/frame.h:89 */
        const int ox = (int)pc[0], oy = (int)pc[1];                                 /* pc.cast<int>() */
        if (!(std::fabs(pc[0]) < 1e9) || !(std::fabs(pc[1]) < 1e9)) continue;      /* cast of a non-finite / huge value is UB in the reference */
        if (!(ox >= border && ox < cam->width - border && oy >= border && oy < cam->height - border)) continue;   /* isInFrame, :154 */
        const int index = (int)(pc[0] / grid_size) * grid_n_height + (int)(pc[1] / grid_size);   /* :156 */
        const float cur_value = flo_shi_tomasi(img, cam->width, cam->height, stride, (int)pc[0], (int)pc[1]);   /* :158 */
        if (cur_value > map_value[index]) {                                          /* :160 */
            map_value[index] = cur_value;
            winner[index] = i;
        }
    }
}

/* =====================================================================================================
 * Visual map: visible-patch selection + reference-patch warp (SURVEY.md section 8 row f2) and map growth
 * (row f4).  CPU restatement of LidarSelector::addFromSparseMap (src/lidar_selection.cpp:346-587),
 * getWarpMatrixAffine (:232-256), warpAffine (:258-296), NCC (:298-315), getBestSearchLevel (:317-331),
 * getpatch (:121-141), addSparseMap's second loop (:171-195), AddPoint (:204-230), addObservation (:913-965)
 * and Point::getCloseViewObs / getFurthestViewObs / addFrameRef / deleteFeatureRef (src/point.cpp).
 *
 * Third-party pieces absent from the reference tree, restated from their published sources (PARITY UNPINNED):
 *   vikit  PinholeCamera::cam2world (pinhole_camera.cpp), AbstractCamera::isInFrame, vk::interpolateMat_8u
 *          (vikit_common/include/vikit/vision.h)
 *   Sophus SE3 (the SVO-era, non-templated version): T * p, inverse(), composition.  Sophus keeps the rotation
 *          as a unit quaternion; here rigid transforms are 3x3 matrices + translation (the same choice the
 *          reference makes itself for the hot loop: Rcw / Pcw, :780-781), so products agree to rounding only.
 *   OpenCV cv::undistortPoints (cam2world with distortion): 5 fixed-point iterations in double on the float input.
 * Iteration order of the reference's unordered_map<VOXEL_KEY, ...> is implementation-defined; it only matters for
 * exact float ties of `cur_dist <= map_dist[index]` (:450).  Here: points are visited in insertion order.
 * ===================================================================================================== */
#include <algorithm>
#include <array>
#include <cstring>
#include <unordered_set>
#include <vector>

namespace {

struct VFeature {           /* include/feature.h:27-66 */
    double px[2], f[3];     /* pixel on level 0, unit bearing */
    double R[9], t[3];      /* T_f_w */
    float score;
    int level, id, img;     /* img: slot of the keyframe image */
};
struct VPoint {             /* include/point.h */
    double pos[3];
    float value;
    std::vector<int> obs;   /* obs_: front() = obs[0] = newest (addFrameRef push_front, point.cpp:57-61) */
    long long key[3];       /* feat_map voxel (AddPoint, :204-216) */
};
struct KeyHash {
    size_t operator()(const std::array<long long, 3>& k) const {
        return (size_t)(k[0] * 73856093ll ^ k[1] * 19349669ll ^ k[2] * 83492791ll);
    }
};

void se3_apply(const double* R, const double* t, const double* p, double* o) {
    for (int k = 0; k < 3; ++k) o[k] = R[3 * k] * p[0] + R[3 * k + 1] * p[1] + R[3 * k + 2] * p[2] + t[k];
}
/* T^-1 translation = -R^T t  (Frame::pos / Feature::pos) */
void se3_pos(const double* R, const double* t, double* o) {
    for (int k = 0; k < 3; ++k) o[k] = -(R[k] * t[0] + R[3 + k] * t[1] + R[6 + k] * t[2]);
}
double norm3d(const double* v) { return std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]); }

}  // namespace

struct flo_vmap {
    flo_cam cam;
    int grid_size, grid_n_width, grid_n_height, length;
    int patch_size = 8, patch_size_half = 4, patch_size_total = 64;
    double outlier_threshold, ncc_thre;
    int ncc_en;
    std::vector<VPoint> pts;
    std::vector<VFeature> fts;
    std::vector<std::vector<uint8_t>> imgs;
    std::vector<float> map_value;
    int img_frame_id = -1, img_slot = -1;   /* the frame whose image was stored last (one cv::Mat shared by its features) */
    /* sub_sparse_map of the last select */
    std::vector<int> sel_index, sel_point, sel_level;
    std::vector<float> sel_patch, sel_error;
};

namespace {

/* vikit PinholeCamera::cam2world(px): unit bearing. */
void cam2world(const flo_cam& cam, double u, double v, double* f) {
    double x, y;
    if (!(std::fabs(cam.d[0]) > 0.0000001)) {
        x = (u - cam.cx) / cam.fx;
        y = (v - cam.cy) / cam.fy;
    } else {
        /* cv::undistortPoints on one CV_32FC2 point: float in, double iterations, float out */
        const float uf = (float)u, vf = (float)v;
        const double x0 = ((double)uf - cam.cx) / cam.fx, y0 = ((double)vf - cam.cy) / cam.fy;
        double xx = x0, yy = y0;
        for (int j = 0; j < 5; ++j) {
            const double r2 = xx * xx + yy * yy;
            const double icdist = 1. / (1 + ((cam.d[4] * r2 + cam.d[1]) * r2 + cam.d[0]) * r2);
            const double deltaX = 2 * cam.d[2] * xx * yy + cam.d[3] * (r2 + 2 * xx * xx);
            const double deltaY = cam.d[2] * (r2 + 2 * yy * yy) + 2 * cam.d[3] * xx * yy;
            xx = (x0 - deltaX) * icdist;
            yy = (y0 - deltaY) * icdist;
        }
        x = (double)(float)xx;
        y = (double)(float)yy;
    }
    const double n = std::sqrt(x * x + y * y + 1.0);
    f[0] = x / n; f[1] = y / n; f[2] = 1.0 / n;
}

/* vk::interpolateMat_8u */
float interpolate_8u(const uint8_t* img, int stride, float u, float v) {
    const int x = (int)std::floor(u), y = (int)std::floor(v);
    const float subpix_x = u - x, subpix_y = v - y;
    const float w00 = (1.0f - subpix_x) * (1.0f - subpix_y);
    const float w01 = (1.0f - subpix_x) * subpix_y;
    const float w10 = subpix_x * (1.0f - subpix_y);
    const float w11 = 1.0f - w00 - w01 - w10;
    const uint8_t* ptr = img + y * stride + x;
    return w00 * ptr[0] + w01 * ptr[stride] + w10 * ptr[1] + w11 * ptr[stride + 1];
}

bool in_frame(const flo_cam& cam, double px0, double px1, int boundary) {   /* isInFrame(px.cast<int>(), boundary) */
    if (!(std::fabs(px0) < 1e9) || !(std::fabs(px1) < 1e9)) return false;
    const int ox = (int)px0, oy = (int)px1;
    return ox >= boundary && ox < cam.width - boundary && oy >= boundary && oy < cam.height - boundary;
}

/* getWarpMatrixAffine, :232-256 (level_ref = 0, pyramid_level = 0 at the only call site, :529) */
void warp_matrix_affine(const flo_cam& cam, const double* px_ref, const double* f_ref, double depth_ref, const double* Rcr,
                        const double* tcr, int level_ref, int pyramid_level, int halfpatch_size, double* A /*2x2 row-major*/) {
    const double xyz_ref[3] = {f_ref[0] * depth_ref, f_ref[1] * depth_ref, f_ref[2] * depth_ref};
    const double step = (double)(halfpatch_size * (1 << level_ref) * (1 << pyramid_level));
    double xyz_du[3], xyz_dv[3];
    cam2world(cam, px_ref[0] + step, px_ref[1], xyz_du);
    cam2world(cam, px_ref[0], px_ref[1] + step, xyz_dv);
    const double su = xyz_ref[2] / xyz_du[2], sv = xyz_ref[2] / xyz_dv[2];
    for (int k = 0; k < 3; ++k) { xyz_du[k] *= su; xyz_dv[k] *= sv; }
    double pc[3], pdu[3], pdv[3], px_cur[2], px_du[2], px_dv[2];
    se3_apply(Rcr, tcr, xyz_ref, pc);
    se3_apply(Rcr, tcr, xyz_du, pdu);
    se3_apply(Rcr, tcr, xyz_dv, pdv);
    flo_world2cam(&cam, pc, px_cur);
    flo_world2cam(&cam, pdu, px_du);
    flo_world2cam(&cam, pdv, px_dv);
    A[0] = (px_du[0] - px_cur[0]) / halfpatch_size;   /* col(0) */
    A[2] = (px_du[1] - px_cur[1]) / halfpatch_size;
    A[1] = (px_dv[0] - px_cur[0]) / halfpatch_size;   /* col(1) */
    A[3] = (px_dv[1] - px_cur[1]) / halfpatch_size;
}

int best_search_level(const double* A, int max_level) {   /* :317-331 */
    int search_level = 0;
    double D = A[0] * A[3] - A[1] * A[2];
    while (D > 3.0 && search_level < max_level) {
        search_level += 1;
        D *= 0.25;
    }
    return search_level;
}

/* warpAffine, :258-296.  Returns false when the inverse is NaN (the reference then leaves the level unwritten). */
bool warp_affine(const double* A_cur_ref, const uint8_t* img_ref, int width, int height, const double* px_ref, int search_level,
                 int pyramid_level, int halfpatch_size, int patch_size_total, float* patch) {
    const int patch_size = halfpatch_size * 2;
    /* Matrix2d::inverse(): adjugate / determinant */
    const double det = A_cur_ref[0] * A_cur_ref[3] - A_cur_ref[1] * A_cur_ref[2];
    const double inv = 1.0 / det;
    const float a00 = (float)(A_cur_ref[3] * inv), a01 = (float)(-A_cur_ref[1] * inv), a10 = (float)(-A_cur_ref[2] * inv),
                a11 = (float)(A_cur_ref[0] * inv);
    if (std::isnan(a00)) return false;
    const float pxr0 = (float)px_ref[0], pxr1 = (float)px_ref[1];
    for (int y = 0; y < patch_size; ++y)
        for (int x = 0; x < patch_size; ++x) {
            float px_patch0 = (float)(x - halfpatch_size), px_patch1 = (float)(y - halfpatch_size);
            px_patch0 *= (float)(1 << search_level); px_patch1 *= (float)(1 << search_level);
            px_patch0 *= (float)(1 << pyramid_level); px_patch1 *= (float)(1 << pyramid_level);
            const float px0 = a00 * px_patch0 + a01 * px_patch1 + pxr0, px1 = a10 * px_patch0 + a11 * px_patch1 + pxr1;
            float val;
            if (px0 < 0 || px1 < 0 || px0 >= width - 1 || px1 >= height - 1) val = 0;
            else val = interpolate_8u(img_ref, width, px0, px1);
            patch[patch_size_total * pyramid_level + y * patch_size + x] = val;
        }
    return true;
}

/* getpatch, :121-141 */
void getpatch(const uint8_t* img, int width, const double* pc, float* patch_tmp, int level, int patch_size, int patch_size_half,
              int patch_size_total) {
    const float u_ref = pc[0];
    const float v_ref = pc[1];
    const int scale = (1 << level);
    const int u_ref_i = floorf(pc[0] / scale) * scale;
    const int v_ref_i = floorf(pc[1] / scale) * scale;
    const float subpix_u_ref = (u_ref - u_ref_i) / scale;
    const float subpix_v_ref = (v_ref - v_ref_i) / scale;
    const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
    const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
    const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
    const float w_ref_br = subpix_u_ref * subpix_v_ref;
    for (int x = 0; x < patch_size; x++) {
        const uint8_t* img_ptr = img + (v_ref_i - patch_size_half * scale + x * scale) * width + (u_ref_i - patch_size_half * scale);
        for (int y = 0; y < patch_size; y++, img_ptr += scale)
            patch_tmp[patch_size_total * level + x * patch_size + y] =
                w_ref_tl * img_ptr[0] + w_ref_tr * img_ptr[scale] + w_ref_bl * img_ptr[scale * width] + w_ref_br * img_ptr[scale * width + scale];
    }
}

double ncc(const float* ref_patch, const float* cur_patch, int patch_size) {   /* :298-315 */
    double sum_ref = 0.0, sum_cur = 0.0;
    for (int i = 0; i < patch_size; ++i) sum_ref += ref_patch[i];
    const double mean_ref = sum_ref / patch_size;
    for (int i = 0; i < patch_size; ++i) sum_cur += cur_patch[i];
    const double mean_curr = sum_cur / patch_size;
    double numerator = 0, demoniator1 = 0, demoniator2 = 0;
    for (int i = 0; i < patch_size; i++) {
        const double n = (ref_patch[i] - mean_ref) * (cur_patch[i] - mean_curr);
        numerator += n;
        demoniator1 += (ref_patch[i] - mean_ref) * (ref_patch[i] - mean_ref);
        demoniator2 += (cur_patch[i] - mean_curr) * (cur_patch[i] - mean_curr);
    }
    return numerator / std::sqrt(demoniator1 * demoniator2 + 1e-10);
}

/* AddPoint's voxel key, :204-216 (float loc, "-= 1.0" for negatives, then truncation) */
void feat_key(const double* pt_w, long long* key) {
    const double voxel_size = 0.5;
    for (int j = 0; j < 3; ++j) {
        float loc = (float)(pt_w[j] / voxel_size);
        if (loc < 0) loc -= 1.0;
        key[j] = (long long)loc;
    }
}

int add_feature(flo_vmap* vm, int point, const double* px, const double* Rcw, const double* Pcw, float score, int level, int id, int img) {
    VFeature ft;
    ft.px[0] = px[0]; ft.px[1] = px[1];
    cam2world(vm->cam, px[0], px[1], ft.f);
    std::memcpy(ft.R, Rcw, sizeof(ft.R));
    std::memcpy(ft.t, Pcw, sizeof(ft.t));
    ft.score = score; ft.level = level; ft.id = id; ft.img = img;
    vm->fts.push_back(ft);
    const int fi = (int)vm->fts.size() - 1;
    vm->pts[point].obs.insert(vm->pts[point].obs.begin(), fi);     /* addFrameRef: push_front */
    return fi;
}

int store_image(flo_vmap* vm, const uint8_t* img, int frame_id) {
    if (vm->img_frame_id == frame_id && vm->img_slot >= 0) return vm->img_slot;
    vm->imgs.emplace_back(img, img + (size_t)vm->cam.width * vm->cam.height);
    vm->img_frame_id = frame_id;
    vm->img_slot = (int)vm->imgs.size() - 1;
    return vm->img_slot;
}

}  // namespace

extern "C" {

flo_vmap* flo_vmap_create(const flo_cam* cam, int grid_size, double outlier_threshold, int ncc_en, double ncc_thre) {
    flo_vmap* vm = new flo_vmap;
    vm->cam = *cam;
    vm->grid_size = grid_size;
    vm->grid_n_width = cam->width / grid_size;     /* :55-57 */
    vm->grid_n_height = cam->height / grid_size;
    vm->length = vm->grid_n_width * vm->grid_n_height;
    vm->outlier_threshold = outlier_threshold;
    vm->ncc_en = ncc_en;
    vm->ncc_thre = ncc_thre;
    vm->map_value.assign(vm->length, 0.0f);
    return vm;
}
void flo_vmap_destroy(flo_vmap* vm) { delete vm; }
int flo_vmap_counts(const flo_vmap* vm, int* n_points, int* n_features, int* n_images) {
    if (n_points) *n_points = (int)vm->pts.size();
    if (n_features) *n_features = (int)vm->fts.size();
    if (n_images) *n_images = (int)vm->imgs.size();
    return vm->length;
}
void flo_vmap_map_value(const flo_vmap* vm, float* out) { std::memcpy(out, vm->map_value.data(), sizeof(float) * vm->length); }

/* LidarSelector::addFromSparseMap (:346-587).  img: the current gray frame; (Rcw, Pcw) = new_frame_->T_f_w_;
 * pg_down: the scan after the caller's pcl::VoxelGrid (0.2 m, :7, :351-352), world frame.  Returns the number of
 * selected patches (sub_sparse_map->index.size()). */
int flo_vmap_select(flo_vmap* vm, const uint8_t* img, const double* Rcw, const double* Pcw, const float* pg_down, int n) {
    vm->sel_index.clear(); vm->sel_point.clear(); vm->sel_level.clear(); vm->sel_patch.clear(); vm->sel_error.clear();
    if (vm->pts.empty()) return 0;                                                  /* :348 */
    const flo_cam& cam = vm->cam;
    const int width = cam.width, height = cam.height, length = vm->length;
    const int border = (vm->patch_size_half + 1) * 8;
    /* reset_grid (:81-90) + :356 */
    std::vector<int> grid_type(length, 0), voxel_points_(length, -1);
    std::vector<float> map_dist(length, 10000.0f);
    std::fill(vm->map_value.begin(), vm->map_value.end(), 0.0f);
    std::vector<float> depth_img((size_t)width * height, 0.0f);                     /* :366 */
    std::unordered_set<std::array<long long, 3>, KeyHash> sub_feat_map;
    const float voxel_size = 0.5;
    const double fx = std::fabs(cam.fx), fy = std::fabs(4.0 * cam.fx * cam.fy) / (4. * std::fabs(cam.fx));   /* :58-59 */
    for (int i = 0; i < n; i++) {                                                   /* :378-418 */
        const double pt_w[3] = {pg_down[3 * i], pg_down[3 * i + 1], pg_down[3 * i + 2]};
        std::array<long long, 3> position;
        for (int j = 0; j < 3; j++) position[j] = (long long)(int)std::floor(pt_w[j] / voxel_size);
        sub_feat_map.insert(position);
        double pt_c[3];
        se3_apply(Rcw, Pcw, pt_w, pt_c);
        if (pt_c[2] > 0) {
            const double px0 = fx * pt_c[0] / pt_c[2] + cam.cx, px1 = fy * pt_c[1] / pt_c[2] + cam.cy;
            if (in_frame(cam, px0, px1, border)) {
                const float depth = pt_c[2];
                const int col = (int)px0, row = (int)px1;
                depth_img[(size_t)width * row + col] = depth;
            }
        }
    }
    double frame_pos[3];
    se3_pos(Rcw, Pcw, frame_pos);
    for (size_t j = 0; j < vm->pts.size(); ++j) {                                   /* :430-470 (visit order: see header) */
        const VPoint& pt = vm->pts[j];
        if (!sub_feat_map.count({pt.key[0], pt.key[1], pt.key[2]})) continue;
        double pt_cam[3], pc[2];
        se3_apply(Rcw, Pcw, pt.pos, pt_cam);
        if (pt_cam[2] < 0) continue;
        flo_world2cam(&cam, pt_cam, pc);
        if (in_frame(cam, pc[0], pc[1], border)) {
            const int index = (int)(pc[0] / vm->grid_size) * vm->grid_n_height + (int)(pc[1] / vm->grid_size);
            grid_type[index] = 1;                                                   /* TYPE_MAP */
            const double obs_vec[3] = {frame_pos[0] - pt.pos[0], frame_pos[1] - pt.pos[1], frame_pos[2] - pt.pos[2]};
            const float cur_dist = norm3d(obs_vec);
            const float cur_value = pt.value;
            if (cur_dist <= map_dist[index]) {
                map_dist[index] = cur_dist;
                voxel_points_[index] = (int)j;
            }
            if (cur_value >= vm->map_value[index]) vm->map_value[index] = cur_value;
        }
    }
    std::vector<float> patch_cache(vm->patch_size_total);
    for (int i = 0; i < length; i++) {                                              /* :479-580 */
        if (grid_type[i] != 1) continue;
        const int pj = voxel_points_[i];
        if (pj < 0) continue;
        const VPoint& pt = vm->pts[pj];
        double pt_cam[3], pc[2];
        se3_apply(Rcw, Pcw, pt.pos, pt_cam);
        flo_world2cam(&cam, pt_cam, pc);
        bool depth_continous = false;
        for (int u = -vm->patch_size_half; u <= vm->patch_size_half; u++) {
            for (int v = -vm->patch_size_half; v <= vm->patch_size_half; v++) {
                if (u == 0 && v == 0) continue;
                const float depth = depth_img[(size_t)width * (v + (int)pc[1]) + u + (int)pc[0]];
                if (depth == 0.) continue;
                const double delta_dist = std::fabs(pt_cam[2] - depth);
                if (delta_dist > 1.5) { depth_continous = true; break; }
            }
            if (depth_continous) break;
        }
        if (depth_continous) continue;
        /* Point::getCloseViewObs(new_frame_->pos(), ref_ftr, pc), point.cpp:141-178 */
        if (pt.obs.empty()) continue;
        double obs_dir[3] = {frame_pos[0] - pt.pos[0], frame_pos[1] - pt.pos[1], frame_pos[2] - pt.pos[2]};
        { const double nn = norm3d(obs_dir); for (int k = 0; k < 3; ++k) obs_dir[k] /= nn; }
        int min_it = pt.obs.front();
        double min_cos_angle = 0;
        for (int fi : pt.obs) {
            const VFeature& ft = vm->fts[fi];
            double fpos[3], dir[3];
            se3_pos(ft.R, ft.t, fpos);
            for (int k = 0; k < 3; ++k) dir[k] = fpos[k] - pt.pos[k];
            const double nn = norm3d(dir);
            for (int k = 0; k < 3; ++k) dir[k] /= nn;
            const double cos_angle = obs_dir[0] * dir[0] + obs_dir[1] * dir[1] + obs_dir[2] * dir[2];
            if (cos_angle > min_cos_angle) { min_cos_angle = cos_angle; min_it = fi; }
        }
        if (min_cos_angle < 0.5) continue;
        const VFeature& ref = vm->fts[min_it];
        std::vector<float> patch_wrap(vm->patch_size_total * 3, 0.0f);
        /* T_cur_ref = new_frame_->T_f_w_ * ref_ftr->T_f_w_.inverse() */
        double Rcr[9], tcr[3], rpos[3];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) Rcr[3 * a + b] = Rcw[3 * a] * ref.R[3 * b] + Rcw[3 * a + 1] * ref.R[3 * b + 1] + Rcw[3 * a + 2] * ref.R[3 * b + 2];
        se3_pos(ref.R, ref.t, rpos);                                               /* T_ref^-1 translation */
        se3_apply(Rcw, Pcw, rpos, tcr);
        const double dvec[3] = {rpos[0] - pt.pos[0], rpos[1] - pt.pos[1], rpos[2] - pt.pos[2]};
        double A_cur_ref_zero[4];
        warp_matrix_affine(cam, ref.px, ref.f, norm3d(dvec), Rcr, tcr, 0, 0, vm->patch_size_half, A_cur_ref_zero);   /* :528-530 */
        const int search_level = best_search_level(A_cur_ref_zero, 2);             /* :532 */
        for (int pyramid_level = 0; pyramid_level <= 2; pyramid_level++)           /* :542-545 */
            warp_affine(A_cur_ref_zero, vm->imgs[ref.img].data(), width, height, ref.px, search_level, pyramid_level,
                        vm->patch_size_half, vm->patch_size_total, patch_wrap.data());
        getpatch(img, width, pc, patch_cache.data(), 0, vm->patch_size, vm->patch_size_half, vm->patch_size_total);   /* :547 */
        if (vm->ncc_en) {
            const double v = ncc(patch_wrap.data(), patch_cache.data(), vm->patch_size_total);
            if (v < vm->ncc_thre) continue;
        }
        float error = 0.0;
        for (int ind = 0; ind < vm->patch_size_total; ind++)
            error += (patch_wrap[ind] - patch_cache[ind]) * (patch_wrap[ind] - patch_cache[ind]);
        if (error > vm->outlier_threshold * vm->patch_size_total) continue;         /* :560 */
        vm->sel_index.push_back(i);
        vm->sel_point.push_back(pj);
        vm->sel_level.push_back(search_level);
        vm->sel_error.push_back(error);
        vm->sel_patch.insert(vm->sel_patch.end(), patch_wrap.begin(), patch_wrap.end());
    }
    return (int)vm->sel_index.size();
}

/* The SubSparseMap of the last flo_vmap_select: index (grid cell), point (visual-map point id), search level,
 * propagated error, pos (Point::pos_), patch (3 x 64 floats).  Any pointer may be null. */
void flo_vmap_selected(const flo_vmap* vm, int* index, int* point, int* search_level, float* error, double* pos, float* patch) {
    const size_t n = vm->sel_index.size();
    if (index) std::memcpy(index, vm->sel_index.data(), n * sizeof(int));
    if (point) std::memcpy(point, vm->sel_point.data(), n * sizeof(int));
    if (search_level) std::memcpy(search_level, vm->sel_level.data(), n * sizeof(int));
    if (error) std::memcpy(error, vm->sel_error.data(), n * sizeof(float));
    if (patch) std::memcpy(patch, vm->sel_patch.data(), n * 192 * sizeof(float));
    if (pos) for (size_t i = 0; i < n; ++i) std::memcpy(pos + 3 * i, vm->pts[vm->sel_point[i]].pos, 3 * sizeof(double));
}

/* LidarSelector::addSparseMap (:142-202): candidate scoring (flo_visual_candidates) then one new Point + Feature
 * per won cell, in cell order.  Returns the number of points added. */
int flo_vmap_grow(flo_vmap* vm, const uint8_t* img, const double* Rcw, const double* Pcw, const float* pg, int n, int frame_id) {
    std::vector<int> winner(vm->length);
    flo_visual_candidates(&vm->cam, Rcw, Pcw, img, vm->cam.width, pg, n, vm->grid_size, (vm->patch_size_half + 1) * 8,
                          vm->map_value.data(), winner.data());
    int add = 0;
    for (int i = 0; i < vm->length; i++) {
        if (winner[i] < 0) continue;                                                /* grid_num[i] == TYPE_POINTCLOUD */
        const double pt[3] = {pg[3 * winner[i]], pg[3 * winner[i] + 1], pg[3 * winner[i] + 2]};
        double pf[3], pc[2];
        se3_apply(Rcw, Pcw, pt, pf);
        flo_world2cam(&vm->cam, pf, pc);
        VPoint p;
        std::memcpy(p.pos, pt, sizeof(pt));
        p.value = vm->map_value[i];
        feat_key(pt, p.key);
        vm->pts.push_back(p);
        const int slot = store_image(vm, img, frame_id);
        add_feature(vm, (int)vm->pts.size() - 1, pc, Rcw, Pcw, vm->map_value[i], 0, frame_id, slot);
        add += 1;
    }
    return add;
}

/* LidarSelector::addObservation (:913-965) over the SubSparseMap of the last select; (Rcw, Pcw) = new_frame_->T_f_w_
 * AFTER ComputeJ (updateFrameState, :982).  Returns the number of features added. */
int flo_vmap_add_observations(flo_vmap* vm, const uint8_t* img, const double* Rcw, const double* Pcw, int frame_id) {
    int added = 0;
    double cur_pos[3];
    se3_pos(Rcw, Pcw, cur_pos);
    for (size_t i = 0; i < vm->sel_index.size(); i++) {
        VPoint& pt = vm->pts[vm->sel_point[i]];
        double pf[3], pc[2];
        se3_apply(Rcw, Pcw, pt.pos, pf);
        flo_world2cam(&vm->cam, pf, pc);
        bool add_flag = false;
        const VFeature last = vm->fts[pt.obs.back()];                               /* obs_.back(): the OLDEST */
        /* delta_pose = pose_ref * pose_cur.inverse() */
        double Rd[9], td[3];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) Rd[3 * a + b] = last.R[3 * a] * Rcw[3 * b] + last.R[3 * a + 1] * Rcw[3 * b + 1] + last.R[3 * a + 2] * Rcw[3 * b + 2];
        se3_apply(last.R, last.t, cur_pos, td);
        const double delta_p = norm3d(td);
        const double tr = Rd[0] + Rd[4] + Rd[8];
        const double delta_theta = (tr > 3.0 - 1e-6) ? 0.0 : std::acos(0.5 * (tr - 1));
        if (delta_p > 0.5 || delta_theta > 10) add_flag = true;
        const double dpx[2] = {pc[0] - last.px[0], pc[1] - last.px[1]};
        const double pixel_dist = std::sqrt(dpx[0] * dpx[0] + dpx[1] * dpx[1]);
        if (pixel_dist > 40) add_flag = true;
        if (pt.obs.size() >= 20) {
            /* Point::getFurthestViewObs(new_frame_->pos(), ref_ftr) + deleteFeatureRef, point.cpp:100-139 */
            double obs_dir[3] = {cur_pos[0] - pt.pos[0], cur_pos[1] - pt.pos[1], cur_pos[2] - pt.pos[2]};
            { const double nn = norm3d(obs_dir); for (int k = 0; k < 3; ++k) obs_dir[k] /= nn; }
            size_t max_it = 0;
            double maxdist = 0.0;
            for (size_t q = 0; q < pt.obs.size(); ++q) {
                double fpos[3];
                se3_pos(vm->fts[pt.obs[q]].R, vm->fts[pt.obs[q]].t, fpos);
                const double d[3] = {fpos[0] - cur_pos[0], fpos[1] - cur_pos[1], fpos[2] - cur_pos[2]};
                const double dist = norm3d(d);
                if (dist > maxdist) { maxdist = dist; max_it = q; }
            }
            pt.obs.erase(pt.obs.begin() + max_it);
        }
        if (add_flag) {
            pt.value = flo_shi_tomasi(img, vm->cam.width, vm->cam.height, vm->cam.width, (int)pc[0], (int)pc[1]);
            const int slot = store_image(vm, img, frame_id);
            add_feature(vm, vm->sel_point[i], pc, Rcw, Pcw, pt.value, vm->sel_level[i], frame_id, slot);
            added++;
        }
    }
    return added;
}

/* publish_frame_world_rgb, src/laserMapping.cpp:710-745 + LidarSelector::getpixel, src/lidar_selection.cpp:1007-1025.
 * Out-of-image taps (see below) are clamped. */
void flo_colorize(const flo_cam* cam, const double* Rcw, const double* Pcw, const uint8_t* bgr, const float* xyz, int n, uint8_t* rgb,
                  uint8_t* valid) {
    const int width = cam->width;
    for (int i = 0; i < n; i++) {
        rgb[3 * i] = rgb[3 * i + 1] = rgb[3 * i + 2] = 0;
        valid[i] = 0;
        const double p_w[3] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
        double pf[3], pc[2];
        se3_apply(Rcw, Pcw, p_w, pf);
        if (pf[2] < 0) continue;
        flo_world2cam(cam, pf, pc);
        if (!in_frame(*cam, pc[0], pc[1], 0)) continue;
        const float u_ref = pc[0];
        const float v_ref = pc[1];
        const int u_ref_i = floorf(pc[0]);
        const int v_ref_i = floorf(pc[1]);
        const float subpix_u_ref = (u_ref - u_ref_i);
        const float subpix_v_ref = (v_ref - v_ref_i);
        const float w_ref_tl = (1.0 - subpix_u_ref) * (1.0 - subpix_v_ref);
        const float w_ref_tr = subpix_u_ref * (1.0 - subpix_v_ref);
        const float w_ref_bl = (1.0 - subpix_u_ref) * subpix_v_ref;
        const float w_ref_br = subpix_u_ref * subpix_v_ref;
        /* pc in (-1, 0) passes isInFrame (its integer cast is 0) and the last row / column has no neighbour: the reference
         * reads outside the image there; defined here as clamping both taps into it */
        const int u0 = std::min(std::max(u_ref_i, 0), cam->width - 1), u1 = std::min(std::max(u_ref_i + 1, 0), cam->width - 1);
        const int v0 = std::min(std::max(v_ref_i, 0), cam->height - 1), v1 = std::min(std::max(v_ref_i + 1, 0), cam->height - 1);
        const int du = (u1 - u0) * 3, dv = (v1 - v0) * width * 3;
        const uint8_t* img_ptr = bgr + ((size_t)v0 * width + u0) * 3;
        const float B = w_ref_tl * img_ptr[0] + w_ref_tr * img_ptr[0 + du] + w_ref_bl * img_ptr[dv] + w_ref_br * img_ptr[dv + 0 + du];
        const float G = w_ref_tl * img_ptr[1] + w_ref_tr * img_ptr[1 + du] + w_ref_bl * img_ptr[1 + dv] + w_ref_br * img_ptr[dv + 1 + du];
        const float R = w_ref_tl * img_ptr[2] + w_ref_tr * img_ptr[2 + du] + w_ref_bl * img_ptr[2 + dv] + w_ref_br * img_ptr[dv + 2 + du];
        rgb[3 * i] = (uint8_t)(int)R; rgb[3 * i + 1] = (uint8_t)(int)G; rgb[3 * i + 2] = (uint8_t)(int)B;
        valid[i] = 1;
    }
}

/* pcl::VoxelGrid<PointT>::applyFilter on x, y, z (PCL 1.8+, filters/include/pcl/filters/impl/voxel_grid.hpp; third-party,
 * absent from the reference tree, restated): leaf index from the cloud minimum, points of a leaf summed in float and divided by
 * the count, output in ascending leaf index.  PCL orders (leaf idx, point) pairs with std::sort on the leaf idx alone, so
 * the order INSIDE a leaf -- and with it the last bits of the float sum -- is unspecified; this restatement uses the input
 * order (a stable sort), which is one of the orders PCL can produce.  Returns the number of leaves. */
int flo_voxel_grid(const float* xyz, int n, float leaf, float* out) {
    if (n <= 0) return 0;
    float mn[3] = {xyz[0], xyz[1], xyz[2]}, mx[3] = {xyz[0], xyz[1], xyz[2]};
    for (int i = 1; i < n; ++i)
        for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], xyz[3 * i + a]); mx[a] = std::max(mx[a], xyz[3 * i + a]); }
    const float inv = 1.0f / leaf;
    {   /* "Leaf size is too small for the input dataset. Integer indices would overflow." */
        const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1, dz = (long long)((mx[2] - mn[2]) * inv) + 1;
        if ((double)dx * (double)dy * (double)dz > 2147483647.0) return -1;
    }
    int min_b[3], div_b[3];
    for (int a = 0; a < 3; ++a) {
        min_b[a] = static_cast<int>(std::floor(mn[a] * inv));
        div_b[a] = static_cast<int>(std::floor(mx[a] * inv)) - min_b[a] + 1;
    }
    std::vector<std::pair<int, int>> idx(n);
    for (int i = 0; i < n; ++i) {
        const int i0 = static_cast<int>(std::floor(xyz[3 * i] * inv) - static_cast<float>(min_b[0]));
        const int i1 = static_cast<int>(std::floor(xyz[3 * i + 1] * inv) - static_cast<float>(min_b[1]));
        const int i2 = static_cast<int>(std::floor(xyz[3 * i + 2] * inv) - static_cast<float>(min_b[2]));
        idx[i] = {i0 + i1 * div_b[0] + i2 * div_b[0] * div_b[1], i};
    }
    std::stable_sort(idx.begin(), idx.end(), [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.first < b.first; });
    int m = 0;
    for (int i = 0; i < n;) {
        float s[3] = {0.f, 0.f, 0.f};
        int c = 0, j = i;
        for (; j < n && idx[j].first == idx[i].first; ++j, ++c)
            for (int a = 0; a < 3; ++a) s[a] += xyz[3 * idx[j].second + a];
        for (int a = 0; a < 3; ++a) out[3 * m + a] = s[a] / static_cast<float>(c);
        ++m;
        i = j;
    }
    return m;
}

/* Dump for tests: per point pos (3 doubles), value, n_obs and the newest-first feature ids (up to 20, -1 padded). */
void flo_vmap_dump_points(const flo_vmap* vm, double* pos, float* value, int* n_obs, int* obs20) {
    for (size_t j = 0; j < vm->pts.size(); ++j) {
        std::memcpy(pos + 3 * j, vm->pts[j].pos, 3 * sizeof(double));
        value[j] = vm->pts[j].value;
        n_obs[j] = (int)vm->pts[j].obs.size();
        for (int q = 0; q < 20; ++q) obs20[20 * j + q] = q < (int)vm->pts[j].obs.size() ? vm->pts[j].obs[q] : -1;
    }
}
/* per feature: px (2), f (3), R (9), t (3) = 17 doubles; score; level, id, img */
void flo_vmap_dump_features(const flo_vmap* vm, double* geo17, float* score, int* level_id_img) {
    for (size_t j = 0; j < vm->fts.size(); ++j) {
        const VFeature& f = vm->fts[j];
        double* g = geo17 + 17 * j;
        g[0] = f.px[0]; g[1] = f.px[1];
        std::memcpy(g + 2, f.f, 3 * sizeof(double));
        std::memcpy(g + 5, f.R, 9 * sizeof(double));
        std::memcpy(g + 14, f.t, 3 * sizeof(double));
        score[j] = f.score;
        level_id_img[3 * j] = f.level; level_id_img[3 * j + 1] = f.id; level_id_img[3 * j + 2] = f.img;
    }
}

}  // extern "C"
