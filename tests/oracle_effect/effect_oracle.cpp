// TEST INFRASTRUCTURE -- the oracle (oracle/flo_*.cpp, compiled unchanged) plus one accessor the tests of
// flb_effect_cloud need: laserCloudOri of the last pass a flo_lio handle ran.  struct flo_lio is private to
// oracle/flo_oracle.cpp, so this translation unit includes that file to see it; tests/effect_oracle.py compiles it
// with the other oracle sources into a library of its own and drives the handles it creates.  Never loaded by the
// product.
#include "../../oracle/flo_oracle.cpp"

extern "C" {

// The serial compaction of flo_lio_pass (src/laserMapping.cpp:1588-1600) over the arrays the last pass on L left:
// point_selected_surf[i] && res_last[i] <= 2.0, ascending, into ori (may be NULL; room for N).  flo_lio_update and
// flo_ikfom_update only run passes, so after either it is the last pass's set.  Returns the count; 0 before any pass.
int flo_lio_last_ori(const flo_lio* L, int* ori) {
    int n = 0;
    for (int i = 0; i < L->N; ++i)
        if (L->selected[i] && (L->res_last[i] <= 2.0)) {
            if (ori) ori[n] = i;
            ++n;
        }
    return n;
}

}  // extern "C"
