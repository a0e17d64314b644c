// TEST INFRASTRUCTURE -- compiles the sparse cell index of the device map (cell keys, hash probe, knn5_grid<true> in
// fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_map_sparse_index.py.  This library
// is NEVER loaded by the product; it exists only under tests/.
#include "../../fast-livo_b200/csrc/flb_device.cuh"
#include <vector>

using namespace flb;

// host build of the hash table over points sorted by cell key (the device's k_sparse_count_cells / k_sparse_insert:
// >= 2x slots, linear probing from cell_hash)
static std::vector<SparseCell> sparse_table(const unsigned long long* keys_sorted, int M, unsigned& mask) {
    int occupied = 0;
    for (int i = 0; i < M; ++i) occupied += (i == 0 || keys_sorted[i - 1] != keys_sorted[i]);
    size_t slots = 16;
    while (slots < 2 * (size_t)occupied) slots <<= 1;
    std::vector<SparseCell> t(slots, SparseCell{kNoCell, -1, -1});
    mask = (unsigned)(slots - 1);
    for (int i = 0; i < M;) {
        int e = i;
        while (e < M && keys_sorted[e] == keys_sorted[i]) ++e;
        unsigned h = cell_hash(keys_sorted[i]) & mask;
        while (t[h].key != kNoCell) h = (h + 1) & mask;
        t[h] = SparseCell{keys_sorted[i], i, e};
        i = e;
    }
    return t;
}

extern "C" {

// cell keys of points (gridf: ox, oy, oz, cell, inv_cell, max_d2), as k_sparse_cell_keys forms them
void emu_sparse_keys(const float* gridf, const float* xyz, int n, unsigned long long* keys) {
    for (int i = 0; i < n; ++i)
        keys[i] = cell_key((int)floorf((xyz[3 * i] - gridf[0]) * gridf[4]), (int)floorf((xyz[3 * i + 1] - gridf[1]) * gridf[4]),
                           (int)floorf((xyz[3 * i + 2] - gridf[2]) * gridf[4]));
}

// [start, end) of the cells (n x 3 ints, relative to the anchor) in the sparse index of the sorted keys
void emu_sparse_find(const unsigned long long* keys_sorted, int M, const int* cells, int n, int* se) {
    unsigned mask;
    const std::vector<SparseCell> t = sparse_table(keys_sorted, M, mask);
    for (int i = 0; i < n; ++i) sparse_find(t.data(), mask, cells[3 * i], cells[3 * i + 1], cells[3 * i + 2], se[2 * i], se[2 * i + 1]);
}

void emu_knn_sparse(const float* gridf /*ox,oy,oz,cell,inv_cell,max_d2*/, int max_ring, const unsigned long long* keys_sorted,
                    const float* pts4, int M, const float* q, int nq, int* pos, float* d2) {
    GridDesc g{};
    g.ox = gridf[0]; g.oy = gridf[1]; g.oz = gridf[2]; g.cell = gridf[3]; g.inv_cell = gridf[4]; g.max_d2 = gridf[5];
    g.max_ring = max_ring;
    unsigned mask;
    const std::vector<SparseCell> t = sparse_table(keys_sorted, M, mask);
    g.nx = (int)mask;
    const map_pt* pts = reinterpret_cast<const map_pt*>(pts4);
    for (int i = 0; i < nq; ++i) {
        Top5 r;
        int rows[18];
        knn5_grid<true>(g, reinterpret_cast<const int*>(t.data()), pts, q[3 * i], q[3 * i + 1], q[3 * i + 2], r, rows, 1);
        for (int j = 0; j < kMatch; ++j) { pos[5 * i + j] = r.i[j]; d2[5 * i + j] = r.d[j]; }
    }
}

}  // extern "C"
