// Drives flb::upload_camera_frame (fastlivo_b200_adapters.hpp) with a mock cv::Mat (.data, .cols, .rows, .step) and
// reads the image set back with flb_image_download.  argv[1]: input blob, int32 camera W, H, frame width, height,
// step (bytes per row), gray rule, then height x step bytes; argv[2]: output blob, the gray image (W*H bytes) then the
// colour frame (W*H*3 bytes) (tests/test_adapter_image.py).
#include <cstdio>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct Mat {   // the cv::Mat members the adapter reads
    unsigned char* data;
    int cols, rows;
    size_t step;
};

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int hdr[6];
    if (fread(hdr, sizeof(int), 6, f) != 6) return 2;
    const int W = hdr[0], H = hdr[1];
    std::vector<unsigned char> px((size_t)hdr[3] * hdr[4]);
    if (fread(px.data(), 1, px.size(), f) != px.size()) return 2;
    fclose(f);
    flb_handle* h = nullptr;
    flb_config cfg{};
    if (flb_create(&cfg, &h) != FLB_OK) {
        fprintf(stderr, "flb_create: %s\n", flb_last_error(nullptr));
        return 3;
    }
    std::vector<unsigned char> gray((size_t)W * H), bgr((size_t)W * H * 3);
    try {
        flb_camera cam{};
        cam.width = W;
        cam.height = H;
        cam.fx = cam.fy = 0.6 * W;
        cam.cx = 0.5 * W;
        cam.cy = 0.5 * H;
        flb::check(h, flb_camera_set(h, &cam));
        const Mat img{px.data(), hdr[2], hdr[3], (size_t)hdr[4]};
        flb::upload_camera_frame(h, img, hdr[5]);
        int w = 0, hh = 0;
        flb::check(h, flb_image_download(h, gray.data(), bgr.data(), W * H, &w, &hh));
        if (w != W || hh != H) return 5;
    } catch (const flb::Error& e) {
        fprintf(stderr, "flb error %d: %s\n", e.code, e.what());
        return 4;
    }
    FILE* o = fopen(argv[2], "wb");
    fwrite(gray.data(), 1, gray.size(), o);
    fwrite(bgr.data(), 1, bgr.size(), o);
    fclose(o);
    flb_destroy(h);
    return 0;
}
