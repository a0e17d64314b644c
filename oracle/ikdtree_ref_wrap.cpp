// TEST INFRASTRUCTURE -- not product code.  Only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may load the library this
// file builds (oracle/_ref/libikdtree_ref.so).
//
// Thin C-ABI wrapper around the reference's OWN k-d tree
// (the reference's include/ikd-Tree/ikd_Tree.{h,cpp}, compiled unmodified from
// where it lies through oracle/shim/, see oracle/Makefile).  It exposes exactly
// the two calls the hot path makes:
//   KD_TREE::Build          (reference src/laserMapping.cpp:1411-1419)
//   KD_TREE::Nearest_Search (reference src/laserMapping.cpp:1543,
//                            include/ikd-Tree/ikd_Tree.cpp:350-380)
// ikd-Tree returns neighbour POINT COPIES, not indices (ikd_Tree.h:177); we
// stash each map point's index in the bits of its `curvature` field (never
// touched by the tree) so callers can recover indices.
#include "ikd_Tree.h"
#include <omp.h>
#include <cstdint>

extern "C" {

// Heap-allocate and never destroy: KD_TREE embeds a 1M-entry MANUAL_Q
// (ikd_Tree.h:17,82) and its destructor joins a thread whose entry point has no
// `return` (ikd_Tree.cpp:182-185, UB) -- so the tree is deliberately leaked.
void* ikdref_build(const float* xyz, int M, int stride_floats) {
    KD_TREE* tree = new KD_TREE(0.5f, 0.6f, 0.2f);
    PointVector pts((size_t)M);
    for (int i = 0; i < M; ++i) {
        PointType p;
        p.x = xyz[(size_t)i * stride_floats + 0];
        p.y = xyz[(size_t)i * stride_floats + 1];
        p.z = xyz[(size_t)i * stride_floats + 2];
        int32_t idx = i;
        std::memcpy(&p.curvature, &idx, 4);
        pts[i] = p;
    }
    tree->Build(pts);
    return tree;
}

int ikdref_size(void* t) { return static_cast<KD_TREE*>(t)->size(); }

// q: nq x 3 floats.  idx: nq x k (filled with -1 where fewer than k found),
// d2: nq x k (INFINITY where missing), in the ascending order Nearest_Search
// returns.  nthreads mirrors the reference's omp_set_num_threads(MP_PROC_NUM)
// (src/laserMapping.cpp:1516-1518).
int ikdref_knn(void* t, const float* q, int nq, int k, int* idx, float* d2, int nthreads) {
    KD_TREE* tree = static_cast<KD_TREE*>(t);
    if (nthreads < 1) nthreads = 1;
    omp_set_num_threads(nthreads);
#pragma omp parallel for
    for (int i = 0; i < nq; ++i) {
        PointType p;
        p.x = q[3 * (size_t)i + 0];
        p.y = q[3 * (size_t)i + 1];
        p.z = q[3 * (size_t)i + 2];
        PointVector near;
        std::vector<float> dist;
        tree->Nearest_Search(p, k, near, dist);
        for (int j = 0; j < k; ++j) {
            if (j < (int)near.size()) {
                int32_t id;
                std::memcpy(&id, &near[j].curvature, 4);
                idx[(size_t)i * k + j] = id;
                d2[(size_t)i * k + j] = dist[j];
            } else {
                idx[(size_t)i * k + j] = -1;
                d2[(size_t)i * k + j] = INFINITY;
            }
        }
    }
    return 0;
}

// --- map maintenance (SURVEY.md section 8 row f1) -------------------------------------------------
// KD_TREE::Add_Points(PointToAdd, downsample_on = true)  (ikd_Tree.cpp:382-457; called from
// map_incremental, src/laserMapping.cpp:692-706), with set_downsample_param(filter_size_map).
int ikdref_add_points(void* t, const float* xyz, int n, float downsample_size) {
    KD_TREE* tree = static_cast<KD_TREE*>(t);
    tree->set_downsample_param(downsample_size);
    PointVector pts((size_t)n);
    for (int i = 0; i < n; ++i) {
        PointType p;
        p.x = xyz[3 * (size_t)i]; p.y = xyz[3 * (size_t)i + 1]; p.z = xyz[3 * (size_t)i + 2];
        int32_t idx = -1 - i;
        std::memcpy(&p.curvature, &idx, 4);
        pts[i] = p;
    }
    return tree->Add_Points(pts, true);
}

// KD_TREE::Delete_Point_Boxes (ikd_Tree.cpp:501-521; lasermap_fov_segment, src/laserMapping.cpp:363-421).
// boxes: nb x 6 floats (min xyz, max xyz).
int ikdref_delete_boxes(void* t, const float* boxes, int nb) {
    KD_TREE* tree = static_cast<KD_TREE*>(t);
    std::vector<BoxPointType> v((size_t)nb);
    for (int i = 0; i < nb; ++i)
        for (int k = 0; k < 3; ++k) { v[i].vertex_min[k] = boxes[6 * i + k]; v[i].vertex_max[k] = boxes[6 * i + 3 + k]; }
    return tree->Delete_Point_Boxes(v);
}

// All live points of the tree (KD_TREE::flatten, ikd_Tree.cpp:1247-1273).  Returns the count; fills at
// most `capacity` points.
int ikdref_flatten(void* t, float* xyz, int capacity) {
    KD_TREE* tree = static_cast<KD_TREE*>(t);
    PointVector st;
    tree->flatten(tree->Root_Node, st, NOT_RECORD);
    const int n = (int)st.size();
    for (int i = 0; i < n && i < capacity; ++i) { xyz[3 * (size_t)i] = st[i].x; xyz[3 * (size_t)i + 1] = st[i].y; xyz[3 * (size_t)i + 2] = st[i].z; }
    return n;
}

}  // extern "C"
