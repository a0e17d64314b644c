// Drives flb::display_keypatch (fastlivo_b200_adapters.hpp) with a mock cv::Mat (.data, .cols, .rows, .step) and a
// recording put_text (tests/test_adapter_keypatch.py).
//   argv[1] == "nohandle": a failing call (no handle) throws flb::Error and draws no text; no device is touched.
//   argv[1] == "device": on a 64 x 48 camera with identity extrinsics and state, a strided img_cp (step 3W + 16):
//     zero patches leave the frame unchanged, return 0 and draw no text; with patches the frame equals
//     flb_keypatch_image's with the pose from the device state, the row padding is untouched, and the text is
//     "25 HZ" at (20, 20) for time = 0.04, drawn once.
// Exit 0 when all hold.
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct Mat {   // the cv::Mat members the adapter reads
    unsigned char* data;
    int cols, rows;
    size_t step;
};

struct Recorder {
    std::vector<std::string> texts;
    std::vector<float> xs, ys;
    void operator()(Mat&, const std::string& t, float x, float y) { texts.push_back(t); xs.push_back(x); ys.push_back(y); }
};

static int no_handle() {
    std::vector<unsigned char> buf(64 * 48 * 3);
    Mat m{buf.data(), 64, 48, 64 * 3};
    int calls = 0;
    try {
        flb::display_keypatch(nullptr, m, 0.04, [&](Mat&, const std::string&, float, float) { ++calls; });
        return 1;
    } catch (const flb::Error&) {
    }
    return calls == 0 ? 0 : 1;
}

static int device() {
    const int W = 64, H = 48;
    flb_handle* h = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &h) != FLB_OK) {
        fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr));
        return 3;
    }
    try {
        flb_camera cam{};
        cam.width = W; cam.height = H; cam.fx = cam.fy = 40.0; cam.cx = 32.0; cam.cy = 24.0;
        flb::check(h, flb_camera_set(h, &cam));
        std::vector<unsigned char> frame((size_t)W * H * 3);
        for (size_t i = 0; i < frame.size(); ++i) frame[i] = (unsigned char)(i * 37 + 11);
        flb::check(h, flb_image_upload_bgr(h, frame.data(), W, H, 3 * W, FLB_GRAY_CV4));
        flb_vmap_params vp{};
        vp.grid_size = 8;
        vp.outlier_threshold = 100.0;
        for (int i = 0; i < 3; ++i) { vp.Rcl[4 * i] = 1.0; vp.R_LI[4 * i] = 1.0; }
        flb::check(h, flb_vmap_reset(h, &vp));
        flb_state18 x{};
        for (int i = 0; i < 3; ++i) x.rot[4 * i] = 1.0;
        for (int i = 0; i < 18; ++i) x.cov[19 * i] = 1e-4;
        flb::check(h, flb_state_upload(h, &x, &x));
        const size_t step = 3 * W + 16;
        std::vector<unsigned char> img(step * H, 0xA5);
        for (int r = 0; r < H; ++r) std::memcpy(&img[r * step], &frame[(size_t)r * W * 3], (size_t)W * 3);
        const std::vector<unsigned char> before = img;
        Mat m{img.data(), W, H, step};
        Recorder rec;
        std::vector<double> pos;
        std::vector<float> patch;
        std::vector<int> level;
        flb::check(h, flb_patches_upload(h, pos.data(), patch.data(), level.data(), 0));
        if (flb::display_keypatch(h, m, 0.04, std::ref(rec)) != 0 || !rec.texts.empty() || img != before) return 5;
        pos = {0.0, 0.0, 2.0, 0.5, 0.25, 2.0, -0.75, 0.5, 2.0, 1.55, 1.1, 2.0};
        patch.assign(4 * 192, 0.f);
        level.assign(4, 0);
        flb::check(h, flb_patches_upload(h, pos.data(), patch.data(), level.data(), 4));
        if (flb::display_keypatch(h, m, 0.04, std::ref(rec)) != 4) return 6;
        if (rec.texts.size() != 1 || rec.texts[0] != "25 HZ" || rec.xs[0] != 20.f || rec.ys[0] != 20.f) return 7;
        std::vector<unsigned char> want((size_t)W * H * 3);
        int n = 0;
        flb::check(h, flb_keypatch_image(h, nullptr, nullptr, want.data(), 3 * W, &n));
        bool drawn = false;
        for (int r = 0; r < H; ++r) {
            if (std::memcmp(&img[r * step], &want[(size_t)r * W * 3], (size_t)W * 3) != 0) return 8;
            if (std::memcmp(&img[r * step], &frame[(size_t)r * W * 3], (size_t)W * 3) != 0) drawn = true;
            for (size_t k = (size_t)W * 3; k < step; ++k)
                if (img[r * step + k] != 0xA5) return 9;
        }
        if (!drawn || n != 4) return 10;
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 4;
    }
    flb_destroy(h);
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 2 && std::string(argv[1]) == "nohandle") return no_handle();
    if (argc >= 2 && std::string(argv[1]) == "device") return device();
    return 2;
}
