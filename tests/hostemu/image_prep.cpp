// TEST INFRASTRUCTURE -- compiles the per-pixel math of flb_image_upload_bgr (bgr_to_gray and mean2x2 in
// fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_image_prep.py, composed per frame
// as k_image_prep composes it.  This library is NEVER loaded by the product; it exists only under tests/.
#include <cstddef>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// gray[i] = bgr_to_gray of the n pixels bgr[3 i .. 3 i + 2]
void emu_bgr_to_gray(const unsigned char* bgr, long long n, int rule, unsigned char* gray) {
    for (long long i = 0; i < n; ++i) gray[i] = (unsigned char)bgr_to_gray(bgr[3 * i], bgr[3 * i + 1], bgr[3 * i + 2], rule);
}

// The camera-size colour frame (W x H x 3) and gray image of a BGR frame of width x height pixels, stride bytes per
// row: W = width (no resize) or width / 2 (halve = 1: every channel the mean2x2 of its 2x2 source block).
void emu_image_prep(const unsigned char* src, int width, int height, int stride, int halve, int rule, unsigned char* bgr,
                    unsigned char* gray) {
    const int W = halve ? width / 2 : width, H = halve ? height / 2 : height;
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            unsigned c[3];
            for (int ch = 0; ch < 3; ++ch) {
                if (halve) {
                    const unsigned char* s0 = src + (size_t)(2 * y) * stride + 6 * (size_t)x + ch;
                    const unsigned char* s1 = s0 + stride;
                    c[ch] = mean2x2(s0[0], s0[3], s1[0], s1[3]);
                } else {
                    c[ch] = src[(size_t)y * stride + 3 * (size_t)x + ch];
                }
                bgr[((size_t)y * W + x) * 3 + ch] = (unsigned char)c[ch];
            }
            gray[(size_t)y * W + x] = (unsigned char)bgr_to_gray(c[0], c[1], c[2], rule);
        }
}

}  // extern "C"
