// TEST INFRASTRUCTURE -- the CPU checker of the local-map cube that flb_map_fov_segment tracks: lasermap_fov_segment
// (hku-mars/FAST-LIVO @ dcebf84, src/laserMapping.cpp:361-421) up to its Delete_Point_Boxes call, stated on its own
// terms and independently of the product's fov_segment_step.  The arithmetic follows the cited lines: the sensor
// position is double, the cube's faces are float (BoxPointType), a face gap is the float of a double difference, the
// trigger distance is a float product, the jump is chosen in double and stored as float, and the cube moves in float.
// Built with -ffp-contract=off (the reference's x86-64 build has no FMA contraction) by __graft_entry__.build(), or by
// tests/fov_oracle.py when that library is missing or older than this file.
#include <cmath>
#include <cstring>

namespace {

struct Cube {
    float lo[3], hi[3];     // LocalMap_Points.vertex_min / vertex_max (:361)
    bool placed;            // Localmap_Initialized (:362)
};

struct Config {
    double side;            // cube_side_length (:1118)
    float range;            // DET_RANGE (:83)
    float ratio;            // MOV_THRESHOLD (:90)
};

struct Checker {
    Config cfg;
    Cube cube;
};

// Distance from the sensor coordinate p to a face, as :388-389 store it.
float face_gap(double p, float face) { return (float)std::fabs(p - (double)face); }

// The jump of a move (:396): the larger of the margin-derived length and range * (ratio - 1), chosen in double.
float jump_length(const Config& c) {
    const double from_margin = (c.side - 2.0 * (double)c.ratio * (double)c.range) * 0.5 * 0.9;
    const double from_range = (double)(c.range * (c.ratio - 1.0f));
    return (float)(from_margin < from_range ? from_range : from_margin);
}

// One call at sensor position p.  Writes the slabs the cube leaves behind (cub_needrm) to out, returns their number.
int step(Checker& k, const double* p, float* out) {
    Cube& c = k.cube;
    if (!c.placed) {                                   // first call: centre the cube on the sensor (:376-384)
        for (int a = 0; a < 3; ++a) {
            c.lo[a] = (float)(p[a] - k.cfg.side / 2.0);
            c.hi[a] = (float)(p[a] + k.cfg.side / 2.0);
        }
        c.placed = true;
        return 0;
    }
    // per axis: -1 the sensor is near the low face, +1 near the high face (the low face is tested first, :399 / :405)
    const float trigger = k.cfg.ratio * k.cfg.range;
    int side[3];
    bool moves = false;
    for (int a = 0; a < 3; ++a) {
        const bool near_lo = face_gap(p[a], c.lo[a]) <= trigger, near_hi = face_gap(p[a], c.hi[a]) <= trigger;
        side[a] = near_lo ? -1 : (near_hi ? 1 : 0);
        moves = moves || side[a] != 0;
    }
    if (!moves) return 0;                              // :393
    const float jump = jump_length(k.cfg);
    const Cube before = c;
    int n = 0;
    for (int a = 0; a < 3; ++a) {
        if (side[a] == 0) continue;
        float* slab = out + 6 * n++;                   // the old cube, cut down to the part left behind on axis a
        std::memcpy(slab, before.lo, sizeof(before.lo));
        std::memcpy(slab + 3, before.hi, sizeof(before.hi));
        if (side[a] < 0) {                             // the cube shifts towards -a and leaves its high slab
            c.lo[a] = before.lo[a] - jump;
            c.hi[a] = before.hi[a] - jump;
            slab[a] = before.hi[a] - jump;
        } else {                                       // towards +a, leaving its low slab
            c.lo[a] = before.lo[a] + jump;
            c.hi[a] = before.hi[a] + jump;
            slab[3 + a] = before.lo[a] + jump;
        }
    }
    return n;
}

}  // namespace

extern "C" {

void* fovo_create(double cube_len, float det_range, float mov_threshold) {
    Checker* k = new Checker{};
    k->cfg = Config{cube_len, det_range, mov_threshold};
    return k;
}
void fovo_destroy(void* k) { delete static_cast<Checker*>(k); }
void fovo_reset(void* k) { static_cast<Checker*>(k)->cube.placed = false; }

// One call at pos.  boxes: up to 3 x {min xyz, max xyz}; local_box: the cube after the call {min xyz, max xyz}.
// Returns the number of boxes.
int fovo_step(void* kv, const double* pos, float* boxes, float* local_box) {
    Checker* k = static_cast<Checker*>(kv);
    const int n = step(*k, pos, boxes);
    std::memcpy(local_box, k->cube.lo, sizeof(k->cube.lo));
    std::memcpy(local_box + 3, k->cube.hi, sizeof(k->cube.hi));
    return n;
}

}  // extern "C"
