"""CPU tier: the cube step of flb_map_fov_segment (fov_segment_step in flb_device.cuh, compiled for the host from
tests/hostemu/fov_segment.cpp) against the oracle's restatement of lasermap_fov_segment (tests/oracle_fov), bit for
bit over seeded trajectories; the oracle against an independent numpy float32 / float64 restatement; and the facts of
the shipped configuration (cube_side_length 20, DET_RANGE 300, MOV_THRESHOLD 1.5): the cube moves on every frame."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import fov_oracle
from conftest import bits

f32, f64 = np.float32, np.float64


class FovCube(C.Structure):
    _fields_ = [("vmin", C.c_float * 3), ("vmax", C.c_float * 3), ("initialized", C.c_int), ("pad", C.c_int)]


class FovRecord(C.Structure):
    _fields_ = [("cube", FovCube), ("n_boxes", C.c_int), ("n_deleted", C.c_int), ("boxes", C.c_float * 18)]


@pytest.fixture(scope="module")
def fov_emu(tmp_path_factory):
    """tests/hostemu/fov_segment.cpp built for the host (into a temporary directory)."""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "fov_segment.cpp")
    so = str(tmp_path_factory.mktemp("fov_emu") / "libfov_segment.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emu_fov_step.argtypes = [C.POINTER(FovRecord), C.c_void_p, C.c_double, C.c_float, C.c_float]
    L.emu_fov_count.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    assert L.emu_fov_record_bytes() == C.sizeof(FovRecord)
    return L


class EmuTracker:
    def __init__(self, L, cube_len, det_range=300.0, mov_threshold=1.5):
        self.L, self.prm, self.rec = L, (float(cube_len), float(det_range), float(mov_threshold)), FovRecord()

    def step(self, pos):
        p = np.ascontiguousarray(pos, f64)
        n = self.L.emu_fov_step(C.byref(self.rec), p.ctypes.data_as(C.c_void_p), *self.prm)
        boxes = np.array(self.rec.boxes[:], f32).reshape(3, 6)
        assert (boxes[n:] == 0).all()                 # unused slots: the empty box
        c = self.rec.cube
        return boxes[:n], np.array(list(c.vmin) + list(c.vmax), f32)


class NumpyTracker:
    """lasermap_fov_segment restated in numpy: float32 vertices and threshold, float64 pose and mov_dist expression."""

    def __init__(self, cube_len, det_range=300.0, mov_threshold=1.5):
        self.cube_len, self.det, self.mov = f64(cube_len), f32(det_range), f32(mov_threshold)
        self.vmin = self.vmax = None

    def step(self, pos):
        pos = np.asarray(pos, f64)
        if self.vmin is None:
            self.vmin = (pos - self.cube_len / 2.0).astype(f32)
            self.vmax = (pos + self.cube_len / 2.0).astype(f32)
            return np.zeros((0, 6), f32), np.concatenate([self.vmin, self.vmax])
        thr = self.mov * self.det                                           # float32 product
        d0 = np.abs(pos - self.vmin.astype(f64)).astype(f32)
        d1 = np.abs(pos - self.vmax.astype(f64)).astype(f32)
        if not ((d0 <= thr) | (d1 <= thr)).any():
            return np.zeros((0, 6), f32), np.concatenate([self.vmin, self.vmax])
        a = (float(self.cube_len) - 2.0 * float(self.mov) * float(self.det)) * 0.5 * 0.9
        b = float(self.det * (self.mov - f32(1)))
        mov_dist = f32(b if a < b else a)
        nmin, nmax, boxes = self.vmin.copy(), self.vmax.copy(), []
        for i in range(3):
            lo, hi = self.vmin.copy(), self.vmax.copy()
            if d0[i] <= thr:
                nmin[i] = nmin[i] - mov_dist
                nmax[i] = nmax[i] - mov_dist
                lo[i] = self.vmax[i] - mov_dist
            elif d1[i] <= thr:
                nmin[i] = nmin[i] + mov_dist
                nmax[i] = nmax[i] + mov_dist
                hi[i] = self.vmin[i] + mov_dist
            else:
                continue
            boxes.append(np.concatenate([lo, hi]))
        self.vmin, self.vmax = nmin, nmax
        return np.array(boxes, f32).reshape(-1, 6), np.concatenate([self.vmin, self.vmax])


def random_walk(seed, n, step, start=(0.0, 0.0, 0.0), jumps=True):
    rng = np.random.default_rng(seed)
    d = rng.normal(0, step, (n, 3))
    if jumps:
        d[rng.random(n) < 0.1] *= 20.0                    # the odd jump
    return np.asarray(start, f64) + np.cumsum(d, axis=0)


def face_crossings(seed, reach=400.0, step=3.0):
    """From the start, out and back along +x, -x, +y, -y, +z, -z, with noise: a 1000 m cube moves across every face."""
    rng = np.random.default_rng(seed)
    p = np.array([12.3, -4.56, 1.25])
    out = [p.copy()]
    for ax in range(3):
        for sgn in (1.0, -1.0):
            for _ in range(2):
                for _ in range(int(reach / step)):
                    p = p + rng.normal(0, 0.3, 3)
                    p[ax] += sgn * step
                    out.append(p.copy())
                sgn = -sgn
    return np.array(out)


CASES = {
    "shipped_walk": (fov_oracle.SHIPPED, lambda s: random_walk(s, 300, 2.0)),
    "shipped_far": (fov_oracle.SHIPPED, lambda s: random_walk(s, 200, 5.0, start=(-3.2e3, 1.7e4, 55.5))),
    "cube200": ((200.0, 300.0, 1.5), lambda s: random_walk(s, 300, 4.0)),
    "cube1000_faces": ((1000.0, 300.0, 1.5), face_crossings),
    "cube1000_small_det": ((1000.0, 100.0, 1.5), face_crossings),
}


def run(tracker, traj):
    return [tracker.step(p) for p in traj]


def same(a, b):
    return a.shape == b.shape and (bits(a) == bits(b)).all()


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_step_matches_oracle(fov_emu, case, seed):
    prm, make = CASES[case]
    traj = make(seed)
    want = run(fov_oracle.Tracker(*prm), traj)
    got = run(EmuTracker(fov_emu, *prm), traj)
    assert len(got) == len(want)
    for k, ((bg, lg), (bw, lw)) in enumerate(zip(got, want)):
        assert same(bg, bw) and same(lg, lw), k
    moved = sum(len(b) > 0 for b, _ in want)
    assert moved > 0


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_matches_numpy(case):
    prm, make = CASES[case]
    traj = make(7)
    for k, ((bo, lo), (bn, ln)) in enumerate(zip(run(fov_oracle.Tracker(*prm), traj), run(NumpyTracker(*prm), traj))):
        assert same(bo, bn) and same(lo, ln), k


def test_face_trajectory_moves_every_way():
    """The 1000 m trajectory moves the cube both ways along every axis."""
    prm, make = CASES["cube1000_faces"]
    t = fov_oracle.Tracker(*prm)
    prev = None
    dirs = set()
    for p in make(0):
        _, local = t.step(p)
        if prev is not None:
            for ax in range(3):
                if local[ax] != prev[ax]:
                    dirs.add((ax, np.sign(local[ax] - prev[ax])))
        prev = local
    assert dirs == {(ax, s) for ax in range(3) for s in (-1.0, 1.0)}


def threshold_positions(cube_len, det, mov):
    """Positions that put dist_to_map_edge (float of a double difference) exactly on the float threshold, just inside
    its rounding interval, and one float step beyond, towards the cube's lower x face."""
    thr = f32(mov) * f32(det)
    start = np.array([0.37, -1.91, 2.5])
    vmin0 = f64(f32(start[0] - cube_len / 2.0))
    half_ulp = float(np.spacing(thr)) / 2.0
    xs = {"exact": vmin0 + float(thr), "rounds_onto": vmin0 + float(thr) + 0.4 * half_ulp,
          "rounds_past": vmin0 + float(thr) + 3.0 * half_ulp}
    return start, thr, {k: np.array([x, start[1], start[2]]) for k, x in xs.items()}


@pytest.mark.parametrize("prm", [(1000.0, 300.0, 1.5), (1000.0, 313.7, 1.3), (2e4, 3.0e3, 1.5)])
def test_threshold_boundary(fov_emu, prm):
    start, thr, cases = threshold_positions(*prm)
    for name, pos in cases.items():
        o, e, nt = fov_oracle.Tracker(*prm), EmuTracker(fov_emu, *prm), NumpyTracker(*prm)
        _, cube0 = o.step(start)
        e.step(start)
        nt.step(start)
        (bo, lo), (be, le), (bn, ln) = o.step(pos), e.step(pos), nt.step(pos)
        assert same(bo, be) and same(lo, le) and same(bo, bn) and same(lo, ln), name
        d = f32(abs(pos[0] - f64(cube0[0])))
        if name == "rounds_past":
            assert d > thr and len(bo) == 0 and same(lo, cube0)
        else:
            # on the threshold: the cube moves toward -x, and the box is the old cube's +x slab
            assert d == thr and len(bo) == 1 and lo[0] < cube0[0] and bo[0][3] == cube0[3] and bo[0][0] > cube0[0]


def test_shipped_config_facts():
    """cube_side_length 20 with DET_RANGE 300 and MOV_THRESHOLD 1.5: the threshold 450 m is beyond the 10 m half side,
    so every frame after the first moves the cube by mov_dist = max(-396, 150) = 150 m along all three axes, and frame
    2's boxes each cover the whole start cube and frame 3's lie 140-160 m from the start.  From frame 4 on the cube swings
    between 290-310 m and 440-460 m from the start on every axis, and each frame's boxes lie 290 m or more from it: three
    boxes a frame while the sensor stays within 10 m of where it started."""
    cube_len, det, mov = fov_oracle.SHIPPED
    assert f32(mov) * f32(det) == f32(450.0)
    assert max((cube_len - 2.0 * mov * det) * 0.5 * 0.9, det * (mov - 1)) == 150.0
    for seed in range(3):
        start = np.array([seed * 7.0, -3.0, 0.5])
        traj = start + np.random.default_rng(seed).uniform(-9.5, 9.5, (200, 3))
        traj[0] = start
        t = fov_oracle.Tracker(*fov_oracle.SHIPPED)
        b1, start_cube = t.step(traj[0])
        assert len(b1) == 0
        assert (start_cube[3:] - start_cube[:3] == f32(cube_len)).all()
        for k, p in enumerate(traj[1:], start=2):
            boxes, local = t.step(p)
            assert len(boxes) == 3, k
            if k == 2:
                for b in boxes:
                    assert (b[:3] <= start_cube[:3]).all() and (b[3:] >= start_cube[3:]).all()
            # distance from the start to each box (the largest per-axis gap between the start and the box's extent)
            gap = [np.maximum(np.maximum(b[:3] - start, start - b[3:]), 0.0).max() for b in boxes]
            if k == 3:
                assert min(gap) >= 139.99 and max(gap) <= 160.01, k
            elif k >= 4:
                assert min(gap) >= 289.99, k


def test_shipped_config_drive():
    """The same configuration on a drive along +x at 1 m a frame: once the sensor is more than 10 m past the swing, both
    x faces are beyond 450 m and the cube stops moving along x for good; y and z keep their two boxes a frame."""
    traj = np.array([[float(k), 0.3, -0.2] for k in range(60)])
    t = fov_oracle.Tracker(*fov_oracle.SHIPPED)
    out = run(t, traj)
    n = [len(b) for b, _ in out]
    first2 = n.index(2)
    assert n[0] == 0 and set(n[1:first2]) == {3} and set(n[first2:]) == {2}
    assert len({float(local[0]) for _, local in out[first2:]}) == 1


def test_box_predicate_half_open(fov_emu):
    """box_contains (k_box_flags and k_fov_flags) is min <= p < max on every axis."""
    box = np.array([[-1.0, 0.0, 2.0, 1.0, 0.5, 3.0]], f32)
    rng = np.random.default_rng(3)
    edges = np.array([[-1, 0, 2], [1, 0, 2], [-1, 0.5, 2], [0, 0, 3], [0, 0.25, 2.5], [np.nextafter(f32(1), f32(0)), 0, 2]], f32)
    pts = np.concatenate([edges, rng.uniform(-2, 4, (4000, 3)).astype(f32)])
    flags = np.zeros(len(pts), np.uint8)
    n = fov_emu.emu_fov_count(pts.ctypes.data_as(C.c_void_p), len(pts), box.ctypes.data_as(C.c_void_p), 1,
                              flags.ctypes.data_as(C.c_void_p))
    want = ((pts >= box[0, :3]) & (pts < box[0, 3:])).all(1)
    assert (flags.astype(bool) == want).all() and n == want.sum()
    assert list(flags[:6]) == [1, 0, 0, 0, 1, 1]
    empty = np.zeros((1, 6), f32)                         # the unused-slot box holds nothing
    assert fov_emu.emu_fov_count(pts.ctypes.data_as(C.c_void_p), len(pts), empty.ctypes.data_as(C.c_void_p), 1,
                                 flags.ctypes.data_as(C.c_void_p)) == 0
