// TEST INFRASTRUCTURE -- compiles the intensity rules of the LiDAR clouds (lidar_intensity, xyzi_record48,
// xyzi_scatter_point, save_slot, xyzi_save_expand and vg_leaf_mean in fast-livo_b200/csrc/flb_device.cuh) with g++ for
// the CPU-only tests of tests/test_intensity_cloud.py, composed as the device composes them: the decode route of
// flb_lidar_upload_intensity (k_lidar_flags' keep rule, the exclusive sum, k_lidar_scatter with k_lidar_intensity, and
// one stable sort of the points and one of the intensities on the same time keys), k_lidar_points48, k_vg_intensity
// over sorted leaf keys, k_xyzi_scatter into the frame's records and a chunked save, and k_xyzi_save_pack.  The save's
// chunks are separate allocations of 2^chunk_log2 records, so a small chunk size exercises the chunk addressing.  Each
// loop iteration is one thread.  This library is NEVER loaded by the product; it exists only under tests/.
#include <algorithm>
#include <numeric>
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

// fmt: kind, step, off_x, off_y, off_z, off_time, off_tag, off_line, n_scans, point_filter_num; off_int: the intensity
// field or -1.  out48: n 48-byte records.  Returns the kept count.
int emu_lidar_points48(const int* fmt, int off_int, double blind, const unsigned char* raw, int n, unsigned* out48) {
    LidarFmt f{};
    f.kind = fmt[0], f.step = fmt[1], f.off_x = fmt[2], f.off_y = fmt[3], f.off_z = fmt[4], f.off_time = fmt[5];
    f.off_tag = fmt[6], f.off_line = fmt[7], f.n_scans = fmt[8], f.filter_num = fmt[9], f.blind = blind;
    f.off_int = off_int < 0 ? (int)kLidarIntZero : off_int;
    if (n > 0 && f.kind == kLidarXt32) f.time_head = lidar_ld64f(raw + f.off_time);
    std::vector<int> vnum(n, 0), kept(n, 0), pos(n, 0);
    if (f.kind == kLidarLivox) {
        for (int i = 0; i < n; ++i) vnum[i] = lidar_livox_valid(raw + (size_t)i * f.step, i, f) ? 1 : 0;
        std::partial_sum(vnum.begin(), vnum.end(), vnum.begin());
    }
    std::vector<LidarPoint> dec(n);
    for (int i = 0; i < n; ++i) {                                  // k_lidar_flags
        const unsigned char* r = raw + (size_t)i * f.step;
        const LidarPoint q = lidar_decode(r, f);
        bool keep;
        if (f.kind == kLidarLivox) {
            const int vn = vnum[i], vp = i > 0 ? vnum[i - 1] : 0;
            keep = false;
            if (lidar_livox_candidate(vn != vp, (unsigned)vn, f)) {
                float px = 0.f, py = 0.f, pz = 0.f;
                const int vpp = i > 1 ? vnum[i - 2] : 0;
                if (i > 0 && lidar_livox_candidate(vp != vpp, (unsigned)vp, f)) {
                    const LidarPoint b = lidar_decode(r - f.step, f);
                    px = b.x, py = b.y, pz = b.z;
                }
                keep = lidar_livox_keep(q, px, py, pz, f.blind);
            }
        } else {
            keep = lidar_pc2_keep(q, i, f);
        }
        dec[i] = q;
        kept[i] = keep ? 1 : 0;
    }
    std::exclusive_scan(kept.begin(), kept.end(), pos.begin(), 0);
    const int m = n > 0 ? pos[n - 1] + kept[n - 1] : 0;
    std::vector<LidarPoint> cloud(m);
    std::vector<float> inten(m);
    std::vector<unsigned> keys(m);
    for (int i = 0; i < n; ++i)                                    // k_lidar_scatter, k_lidar_intensity
        if (kept[i]) {
            cloud[pos[i]] = dec[i];
            keys[pos[i]] = lidar_time_key(dec[i].t);
            inten[pos[i]] = lidar_intensity(raw + (size_t)i * f.step, f);
        }
    // two stable sorts on the same keys: the same permutation
    std::vector<int> order(m), order_i(m);
    std::iota(order.begin(), order.end(), 0);
    std::iota(order_i.begin(), order_i.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    std::stable_sort(order_i.begin(), order_i.end(), [&](int a, int b) { return keys[a] < keys[b]; });
    rgb_word4* out = reinterpret_cast<rgb_word4*>(out48);
    for (int j = 0; j < m; ++j) {                                  // k_lidar_points48
        const LidarPoint& q = cloud[order[j]];
        xyzi_record48(float_as_u32(q.x), float_as_u32(q.y), float_as_u32(q.z), float_as_u32(inten[order_i[j]]), float_as_u32(q.t),
                      out + 3 * (size_t)j);
    }
    return m;
}

// k_vg_heads, the exclusive sum and k_vg_intensity over n sorted leaf keys (vals_sorted: the input index of each
// entry).  Writes each leaf's mean at its rank; returns the leaf count.
int emu_vg_intensity(const unsigned* keys_sorted, const int* vals_sorted, int n, const float* inten, float* out) {
    int rank = 0;
    for (int i = 0; i < n; ++i)
        if (i == 0 || keys_sorted[i] != keys_sorted[i - 1]) out[rank++] = vg_leaf_mean(inten, keys_sorted, vals_sorted, i, n);
    return rank;
}

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

// k_xyzi_scatter: the n points xyz with their intensities as 48-byte records into out48 (12 words each); save != NULL
// appends their save records.
void emu_xyzi_cloud(const float* xyz, const float* inten, int n, unsigned* out48, void* save) {
    EmuSave* s = static_cast<EmuSave*>(save);
    rgb_word4* const* table = nullptr;
    if (s && n > 0) {
        const long long need = s->n + n;
        while ((long long)s->chunks.size() << s->chunk_log2 < need) s->chunks.push_back(new rgb_word4[(size_t)1 << s->chunk_log2]);
        table = s->chunks.data();
    }
    rgb_word4* out = reinterpret_cast<rgb_word4*>(out48);
    for (int i = 0; i < n; ++i) xyzi_scatter_point(xyz + 3 * (size_t)i, inten + i, i, out, table, s ? s->n : 0, s ? s->chunk_log2 : 0);
    if (table) s->n += n;
}

// k_xyzi_save_pack: save records first .. first + count - 1 as 48-byte records
void emu_save_download(void* sv, long long first, int count, unsigned* out48) {
    EmuSave* s = static_cast<EmuSave*>(sv);
    rgb_word4* out = reinterpret_cast<rgb_word4*>(out48);
    for (int i = 0; i < count; ++i) xyzi_save_expand(*save_slot(s->chunks.data(), first + i, s->chunk_log2), out + 3 * (size_t)i);
}

}  // extern "C"
