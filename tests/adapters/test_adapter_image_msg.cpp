// Drives flb::camera_encoding and flb::upload_camera_msg (fastlivo_b200_adapters.hpp) with a mock sensor_msgs::Image
// (.encoding, .width, .height, .step, .data) (tests/test_adapter_image_msg.py).
//   argv[1] == "map": checks every encoding string's FLB_ENC_* and the throw on strings the device does not take; no
//   device is touched.  Exit 0 when all hold.
//   otherwise argv[1]: input blob, int32 camera W, H, message width, height, step, then the encoding string's length
//   and bytes, then height x step bytes; argv[2]: output blob, the gray image (W*H bytes) then the colour frame.
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/fastlivo_b200.h"
#include "../../fast-livo_b200/adapters/fastlivo_b200_adapters.hpp"

struct ImageMsg {   // the sensor_msgs::Image members the adapter reads
    std::string encoding;
    unsigned width, height, step;
    std::vector<unsigned char> data;
};

static int check_map() {
    const struct { const char* s; int enc; } known[] = {
        {"bgr8", FLB_ENC_BGR8}, {"rgb8", FLB_ENC_RGB8}, {"mono8", FLB_ENC_MONO8}, {"bgra8", FLB_ENC_BGRA8},
        {"rgba8", FLB_ENC_RGBA8}, {"bayer_rggb8", FLB_ENC_BAYER_RGGB8}, {"bayer_bggr8", FLB_ENC_BAYER_BGGR8},
        {"bayer_gbrg8", FLB_ENC_BAYER_GBRG8}, {"bayer_grbg8", FLB_ENC_BAYER_GRBG8}};
    for (const auto& k : known)
        if (flb::camera_encoding(k.s) != k.enc) { fprintf(stderr, "%s -> %d\n", k.s, flb::camera_encoding(k.s)); return 1; }
    const char* refused[] = {"mono16", "bgr16", "yuv422", "bayer_rggb16", "BGR8", "jpeg", "", "8UC3"};
    for (const char* s : refused) {
        try {
            flb::camera_encoding(s);
            fprintf(stderr, "'%s' did not throw\n", s);
            return 1;
        } catch (const flb::Error& e) {
            if (e.code != FLB_ERR_INVALID) return 1;
        }
    }
    // a message with an unknown encoding throws before the handle is used (a null handle would fail any ABI call)
    ImageMsg msg{"yuv422", 32, 16, 64, std::vector<unsigned char>(64 * 16)};
    try {
        flb::upload_camera_msg(nullptr, msg, FLB_GRAY_CV4);
        return 1;
    } catch (const flb::Error& e) {
        if (e.code != FLB_ERR_INVALID) return 1;
    }
    return 0;
}

int main(int argc, char** argv) {
    if (argc >= 2 && std::string(argv[1]) == "map") return check_map();
    if (argc < 3) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    int hdr[6];
    if (fread(hdr, sizeof(int), 6, f) != 6) return 2;
    const int W = hdr[0], H = hdr[1];
    ImageMsg msg;
    msg.encoding.resize(hdr[5]);
    if (fread(&msg.encoding[0], 1, hdr[5], f) != (size_t)hdr[5]) return 2;
    msg.width = hdr[2]; msg.height = hdr[3]; msg.step = hdr[4];
    msg.data.resize((size_t)msg.step * msg.height);
    if (fread(msg.data.data(), 1, msg.data.size(), f) != msg.data.size()) return 2;
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
        flb::upload_camera_msg(h, msg, FLB_GRAY_CV4);
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
