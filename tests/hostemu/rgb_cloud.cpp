// TEST INFRASTRUCTURE -- compiles flb_rgb_cloud's per-point rules (rgb_flag_point, rgb_scatter_point, rgb_save_slot and
// rgb_save_expand in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_rgb_cloud.py,
// composed as the device composes them: k_rgb_flags, an exclusive sum over the flags (cub's), k_rgb_scatter into the
// frame's records and a chunked save, k_rgb_save_pack.  The save's chunks are separate allocations of 2^chunk_log2
// records, so a small chunk size exercises the chunk addressing.  Each loop iteration is one thread.  This library is
// NEVER loaded by the product; it exists only under tests/.
#include <cstring>
#include <vector>

#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

namespace {
struct EmuSave {
    int chunk_log2 = 0;
    long long n = 0;
    std::vector<rgb_word4*> chunks;
};
}  // namespace

extern "C" {

void* emu_save_new(int chunk_log2) {
    EmuSave* s = new EmuSave;
    s->chunk_log2 = chunk_log2;
    return s;
}

void emu_save_free(void* sv) {
    EmuSave* s = static_cast<EmuSave*>(sv);
    for (rgb_word4* c : s->chunks) delete[] c;
    delete s;
}

long long emu_save_size(void* sv) { return static_cast<EmuSave*>(sv)->n; }

// cam: width, height as doubles, then fx, fy, cx, cy, d0..d4.  The n world points xyz coloured from the W x H x 3 frame
// bgr at (Rcw, Pcw): writes the records (8 words each) to out32 and returns their count; save != NULL appends them.
int emu_rgb_cloud(const double* camv, const double* Rcw, const double* Pcw, const unsigned char* bgr, const float* xyz, int n,
                  unsigned* out32, void* save) {
    CamModel cam;
    cam.width = (int)camv[0]; cam.height = (int)camv[1];
    cam.fx = camv[2]; cam.fy = camv[3]; cam.cx = camv[4]; cam.cy = camv[5];
    for (int i = 0; i < 5; ++i) cam.d[i] = camv[6 + i];
    cam.jfx = cam.jfy = 0.0;
    std::vector<unsigned> bgra(n);
    std::vector<int> flag(n + 1), pos(n + 1);
    for (int i = 0; i <= n; ++i)                                         // k_rgb_flags
        flag[i] = i == n ? 0 : rgb_flag_point(cam, Rcw, Pcw, bgr, xyz + 3 * (size_t)i, &bgra[i]);
    int run = 0;
    for (int i = 0; i <= n; ++i) { pos[i] = run; run += flag[i]; }      // exclusive sum
    const int m = pos[n];
    EmuSave* s = static_cast<EmuSave*>(save);
    rgb_word4* const* table = nullptr;
    if (s && m > 0) {
        const long long need = s->n + m;
        while ((long long)s->chunks.size() << s->chunk_log2 < need) s->chunks.push_back(new rgb_word4[(size_t)1 << s->chunk_log2]);
        table = s->chunks.data();
    }
    rgb_word4* out = reinterpret_cast<rgb_word4*>(out32);
    for (int i = 0; i < n; ++i)                                          // k_rgb_scatter
        if (flag[i]) rgb_scatter_point(xyz + 3 * (size_t)i, bgra[i], pos[i], out, table, s ? s->n : 0, s ? s->chunk_log2 : 0);
    if (table) s->n += m;
    return m;
}

// k_rgb_save_pack over records first .. first + count - 1 of the save, 8 words each into out32.
void emu_save_download(void* sv, long long first, int count, unsigned* out32) {
    EmuSave* s = static_cast<EmuSave*>(sv);
    rgb_word4* out = reinterpret_cast<rgb_word4*>(out32);
    for (int i = 0; i < count; ++i) rgb_save_expand(*rgb_save_slot(s->chunks.data(), first + i, s->chunk_log2), out + 2 * (size_t)i);
}

}  // extern "C"
