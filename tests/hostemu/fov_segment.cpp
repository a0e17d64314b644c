// TEST INFRASTRUCTURE -- compiles the cube step of flb_map_fov_segment (fov_segment_step and box_contains in
// fast-livo_b200/csrc/flb_device.cuh) with g++ for the CPU-only tests of tests/test_fov_segment.py, carried from call to
// call as k_fov_step carries it (the record a call leaves holds the next call's cube).  This library is NEVER loaded by
// the product; it exists only under tests/.
#include "../../fast-livo_b200/csrc/flb_device.cuh"

using namespace flb;

extern "C" {

int emu_fov_record_bytes() { return (int)sizeof(FovRecord); }

// rec: the record of the previous call (all zeros before the first); overwritten with this call's.  Returns n_boxes.
int emu_fov_step(FovRecord* rec, const double* pos, double cube_len, float det_range, float mov_threshold) {
    const FovCube in = rec->cube;
    fov_segment_step(in, pos, cube_len, det_range, mov_threshold, *rec);
    return rec->n_boxes;
}

// Points (n x 3) inside any of the first nb boxes, as k_fov_flags flags them.
int emu_fov_count(const float* xyz, int n, const float* boxes, int nb, unsigned char* flags) {
    int c = 0;
    for (int i = 0; i < n; ++i) {
        bool del = false;
        for (int b = 0; b < nb; ++b)
            if (box_contains(boxes + 6 * b, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2])) del = true;
        flags[i] = del ? 1 : 0;
        c += del ? 1 : 0;
    }
    return c;
}

}  // extern "C"
