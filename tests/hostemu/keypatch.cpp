// TEST INFRASTRUCTURE -- compiles the per-patch and per-pixel rules of flb_keypatch_image (keypatch_round,
// keypatch_in_disk and keypatch_colour in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of
// tests/test_keypatch.py, composed per frame as k_kp_stamp and k_kp_compose compose them.
// This library is NEVER loaded by the product; it exists only under tests/.
#include <cstddef>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

// The W x H BGR8 frame `img` with the disks of n centres (float pixel coordinates, x y) and errors drawn into `out`.
void emu_keypatch(const unsigned char* img, int W, int H, const float* cxy, const float* err, int n, unsigned char* out) {
    std::vector<int> owner((size_t)W * H, -1);
    for (int i = 0; i < n; ++i) {                              // k_kp_stamp: the highest index that covers a pixel
        int cx, cy;
        if (!keypatch_round(cxy[2 * i], &cx) || !keypatch_round(cxy[2 * i + 1], &cy)) continue;
        for (int dy = -kKeypatchRadius; dy <= kKeypatchRadius; ++dy)
            for (int dx = -kKeypatchRadius; dx <= kKeypatchRadius; ++dx) {
                const int x = cx + dx, y = cy + dy;
                if (keypatch_in_disk(dx, dy) && x >= 0 && x < W && y >= 0 && y < H) {
                    int& o = owner[(size_t)y * W + x];
                    o = o > i ? o : i;
                }
            }
    }
    for (size_t p = 0; p < (size_t)W * H; ++p) {              // k_kp_compose
        if (owner[p] < 0) {
            for (int c = 0; c < 3; ++c) out[3 * p + c] = img[3 * p + c];
        } else {
            keypatch_colour(err[owner[p]], out + 3 * p);
        }
    }
}

// keypatch_round of each double: ok[i] = drawn, r[i] = the rounded coordinate.
void emu_keypatch_round(const double* v, int n, int* r, int* ok) {
    for (int i = 0; i < n; ++i) ok[i] = keypatch_round(v[i], &r[i]) ? 1 : 0;
}

}  // extern "C"
