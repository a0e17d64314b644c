// TEST INFRASTRUCTURE -- compiles the reclaim rules of the device visual map (vm_point_word_feature, vm_feature_live,
// vm_feature_remap, vm_slot_free, vm_image_slot in fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of
// tests/test_vmap_reclaim.py, applied in the order the reclaim kernels of flb_vmap.cuh apply them (each loop below is
// one kernel, its iterations the threads).  This library is NEVER loaded by the product; it exists only under tests/.
#include "../../fast-livo_b200/csrc/flb_device.cuh"
#include <cstring>
#include <vector>

using namespace flb;

extern "C" {

// One reclaim over n_points points (n_obs; obs20: newest-first ids, 20 per point) and n_feats features (feat_img: their
// image slots), `tail` slots handed out, `pinned` the current frame's slot (-1: none).  Out: rank[n_feats + 1], obs20
// remapped in place, feat_img[0..n_live) the survivors' slots in order, free_stack[0..*n_free) (top last).  Returns n_live.
int emu_vm_reclaim(int n_points, const int* n_obs, int* obs20, int n_feats, int* feat_img, int tail, int pinned, int* rank, int* free_stack,
                   int* n_free) {
    std::vector<VmPoint> pts((size_t)n_points);
    std::memset(pts.data(), 0, pts.size() * sizeof(VmPoint));
    for (int j = 0; j < n_points; ++j) {
        pts[j].n_obs = n_obs[j];
        for (int q = 0; q <= kVmMaxObs; ++q) pts[j].obs[q] = q < kVmMaxObs ? obs20[20 * j + q] : 0x7fffffff;   // stale entries stay unread
        pts[j].pad = -7;
    }
    // k_vm_rc_mark: one 32-bit word of the point array per thread
    std::vector<int> flag((size_t)n_feats + 1, 0);
    const int* words = reinterpret_cast<const int*>(pts.data());
    for (size_t w = 0; w < (size_t)n_points * kVmPointWords; ++w) {
        const size_t j = w / kVmPointWords;
        const int f = vm_point_word_feature(words + j * kVmPointWords, (int)(w - j * kVmPointWords));
        if (f >= 0) flag[f] = 1;
    }
    int run = 0;                                                       // the exclusive scan (cub on the device)
    for (int f = 0; f <= n_feats; ++f) { rank[f] = run; run += flag[f]; }
    // k_vm_rc_compact (ascending f: rank[f] <= f, so in place is safe here)
    std::vector<int> slot_live((size_t)std::max(tail, 1), 0);
    for (int f = 0; f < n_feats; ++f) {
        if (!vm_feature_live(rank, f)) continue;
        slot_live[feat_img[f]] = 1;
        feat_img[vm_feature_remap(rank, f)] = feat_img[f];
    }
    // k_vm_rc_remap
    int* wr = reinterpret_cast<int*>(pts.data());
    for (size_t w = 0; w < (size_t)n_points * kVmPointWords; ++w) {
        const size_t j = w / kVmPointWords;
        const int f = vm_point_word_feature(wr + j * kVmPointWords, (int)(w - j * kVmPointWords));
        if (f >= 0) wr[w] = vm_feature_remap(rank, f);
    }
    for (int j = 0; j < n_points; ++j)
        for (int q = 0; q < kVmMaxObs; ++q) obs20[20 * j + q] = q < pts[j].n_obs ? pts[j].obs[q] : -1;
    // k_vm_rc_slots: order-preserving compaction of the free slots, lowest on top
    std::vector<int> fl((size_t)std::max(tail, 1), 0);
    int total = 0;
    for (int s = 0; s < tail; ++s) total += (fl[s] = vm_slot_free(slot_live.data(), pinned, s) ? 1 : 0);
    for (int s = 0, r = 0; s < tail; ++s)
        if (fl[s]) free_stack[total - 1 - r++] = s;
    *n_free = total;
    return rank[n_feats];
}

// The slots the next n committed keyframes get (vm_commit_image): the free-slot stack's top while it holds any, then the tail.
void emu_vm_next_slots(int n_free, const int* free_stack, int tail, int n, int* out) {
    for (int i = 0; i < n; ++i) {
        out[i] = vm_image_slot(n_free, free_stack, tail);
        if (n_free > 0) --n_free;
        else ++tail;
    }
}

}  // extern "C"
