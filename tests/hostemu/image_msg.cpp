// TEST INFRASTRUCTURE -- compiles the per-pixel rules of flb_image_upload_msg (enc_byte, bayer_bgr, mean2x2,
// linear_tap, linear_v and bgr_to_gray in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of
// tests/test_image_msg.py, composed per frame as k_bayer_bgr, k_image_prep and k_image_resize_linear compose them.
// This library is NEVER loaded by the product; it exists only under tests/.
#include <cmath>
#include <cstddef>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// The demosaiced BGR8 frame (w x h x 3) of a dense w x h Bayer mosaic.
void emu_bayer_bgr(const unsigned char* m, int w, int h, int enc, unsigned char* bgr) {
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            unsigned b, g, r;
            bayer_bgr(m, w, h, enc, x, y, b, g, r);
            unsigned char* o = bgr + ((size_t)y * w + x) * 3;
            o[0] = (unsigned char)b; o[1] = (unsigned char)g; o[2] = (unsigned char)r;
        }
}

// linear_tap of every output index d < n from a source axis of s: o[d], a0[d], a1[d].
void emu_linear_taps(int n, int s, int* o, int* a0, int* a1) {
    for (int d = 0; d < n; ++d) {
        const LinearTap t = linear_tap(d, n, s);
        o[d] = t.o; a0[d] = t.a0; a1[d] = t.a1;
    }
}

// The camera-size (W x H) colour frame and gray image of a width x height frame in `enc`, `step` bytes a row.
void emu_image_msg(const unsigned char* src, int width, int height, int step, int enc, int W, int H, int rule, unsigned char* bgr,
                   unsigned char* gray) {
    // the frame as dense BGR8 (what every output kernel reads through enc_byte, a Bayer mosaic after k_bayer_bgr)
    const int P = enc_bpp(enc);
    std::vector<unsigned char> dense((size_t)width * height * P), dec((size_t)width * height * 3);
    for (int y = 0; y < height; ++y)
        for (size_t i = 0; i < (size_t)width * P; ++i) dense[(size_t)y * width * P + i] = src[(size_t)y * step + i];
    if (enc >= kEncBayerRggb8) {
        emu_bayer_bgr(dense.data(), width, height, enc, dec.data());
    } else {
        for (size_t p = 0; p < (size_t)width * height; ++p)
            for (int ch = 0; ch < 3; ++ch) dec[3 * p + ch] = dense[p * P + enc_byte(enc, ch)];
    }
    const unsigned char* d = dec.data();
    for (int y = 0; y < H; ++y) {
        const LinearTap ty = linear_tap(y, H, height);
        for (int x = 0; x < W; ++x) {
            const LinearTap tx = linear_tap(x, W, width);
            unsigned c[3];
            for (int ch = 0; ch < 3; ++ch) {
                if (width == W && height == H) {
                    c[ch] = d[((size_t)y * width + x) * 3 + ch];
                } else if (width == 2 * W && height == 2 * H) {
                    const unsigned char* s0 = d + ((size_t)(2 * y) * width + 2 * x) * 3 + ch;
                    const unsigned char* s1 = s0 + (size_t)width * 3;
                    c[ch] = mean2x2(s0[0], s0[3], s1[0], s1[3]);
                } else {
                    const int x1 = tx.o + 1 < width ? tx.o + 1 : width - 1, y1 = ty.o + 1 < height ? ty.o + 1 : height - 1;
                    auto at = [&](int yy, int xx) { return (int)d[((size_t)yy * width + xx) * 3 + ch]; };
                    const int s0 = at(ty.o, tx.o) * tx.a0 + at(ty.o, x1) * tx.a1;
                    const int s1 = at(y1, tx.o) * tx.a0 + at(y1, x1) * tx.a1;
                    c[ch] = linear_v(s0, s1, ty.a0, ty.a1);
                }
                bgr[((size_t)y * W + x) * 3 + ch] = (unsigned char)c[ch];
            }
            gray[(size_t)y * W + x] = (unsigned char)bgr_to_gray(c[0], c[1], c[2], rule);
        }
    }
}

}  // extern "C"
