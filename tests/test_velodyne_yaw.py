"""CPU tier of flb_lidar_upload_velodyne.  Three statements of velodyne_handler's non-feature branch without per-point
times (reference src/preprocess.cpp:376-428) and the stable time sort (src/laserMapping.cpp:551) must agree byte for
byte on every synthetic spin and layout: the checker (tests/oracle_pre/velo_oracle.cpp, the reference's sequential
per-ring walk), a numpy restatement that runs the walk as a log-step parallel scan, and the product's per-record device
math compiled for the host (tests/hostemu/velodyne_yaw.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pre_oracle
import velo_oracle
from velo_util import LAYOUTS, assert_time_bound, lidar_format_of, spin

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "velodyne_golden.npz")
OMEGA = 0.361 * 10
WRAP = 360.0 / OMEGA


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/velodyne_yaw.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("velodyne_yaw") / "libvelodyne_yaw.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "velodyne_yaw.cpp")])
    L = C.CDLL(so)
    L.emu_velo_process.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.emu_velo_compose.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_velo_apply.argtypes = [C.c_void_p, C.c_float]
    L.emu_velo_apply.restype = C.c_float
    L.emu_velo_step.argtypes = [C.c_double, C.c_double, C.c_void_p]
    L.emu_velo_yaw.argtypes = [C.c_float, C.c_float]
    L.emu_velo_yaw.restype = C.c_double
    return L


def emu_process(L, fmt, records):
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // fmt["point_step"]
    out = np.zeros((max(n, 1), 4), np.float32)
    bad, bad_ring = C.c_int(), C.c_int()
    m = L.emu_velo_process(velo_oracle.fmt_ints(fmt).ctypes.data, fmt["blind"], rec.ctypes.data if n else None, n, out.ctypes.data,
                       C.byref(bad), C.byref(bad_ring))
    return (None if m < 0 else out[:m]), bad.value, bad_ring.value


# ------------------------------------------------------------------------------------------------ numpy restatement
def _apply(m, x):
    with np.errstate(invalid="ignore"):
        return np.where(x > m[0], m[1], m[2])


def _compose(first, then):
    return (first[0], _apply(then, first[1]), _apply(then, first[2]))


def numpy_process(fmt, records):
    """The same result without a loop over the records: the rings' walks as one Hillis-Steele scan in ring order."""
    step = fmt["point_step"]
    raw = np.frombuffer(records, np.uint8).reshape(-1, step)
    n = len(raw)

    def col(off, dtype):
        return np.ascontiguousarray(raw[:, off:off + np.dtype(dtype).itemsize]).view(dtype)[:, 0]

    x, y, z = col(fmt["off_x"], "<f4"), col(fmt["off_y"], "<f4"), col(fmt["off_z"], "<f4")
    ring = col(fmt["off_ring"], "<u2").astype(np.int64)
    assert (ring < fmt["n_scans"]).all()
    yaw = np.arctan2(y.astype(np.float64), x.astype(np.float64)).astype(np.float32).astype(np.float64) * 57.2957
    o = np.argsort(ring, kind="stable")
    rs, ys = ring[o], yaw[o]
    head = np.r_[True, rs[1:] != rs[:-1]] if n else np.zeros(0, bool)
    yaw_fp = ys[np.maximum.accumulate(np.where(head, np.arange(n), 0))] if n else ys
    with np.errstate(invalid="ignore"):
        base = np.where(ys <= yaw_fp, ((yaw_fp - ys) / OMEGA).astype(np.float32), ((yaw_fp - ys + 360.0) / OMEGA).astype(np.float32))
    m = [base, (base.astype(np.float64) + WRAP).astype(np.float32), base.copy()]
    for k in range(3):
        m[k][head] = 0.0
    d = 1
    while d < n:
        c, a, b = _compose((m[0][:-d], m[1][:-d], m[2][:-d]), (m[0][d:], m[1][d:], m[2][d:]))
        m = [np.r_[m[0][:d], c], np.r_[m[1][:d], a], np.r_[m[2][:d], b]]
        d *= 2
    ts = _apply(m, np.float32(0)).astype(np.float32)
    t = np.empty(n, np.float32)
    t[o] = ts
    first = np.zeros(n, bool)
    first[o[head]] = True
    with np.errstate(invalid="ignore"):
        r2 = ((x * x + y * y) + z * z).astype(np.float64)
        keep = ~first & (np.arange(n) % fmt["point_filter_num"] == 0) & (r2 > np.float64(fmt["blind"]) ** 2)
    cloud = np.stack([x, y, z, t], 1)[keep]
    return cloud[np.argsort(cloud[:, 3], kind="stable")]


# ------------------------------------------------------------------------------------------------ the spins
@pytest.mark.parametrize("pfn", [1, 2, 3])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_three_statements_agree(flb, emu, layout, pfn):
    for seed in (1, 2):
        rec, fmt = spin(flb, layout, seed, pfn)
        assert not velo_oracle.midpoint_flags(fmt, rec).any()      # the defined yaw is the same on every conforming atan2
        ref, yaw_times = velo_oracle.process(fmt, rec)
        assert yaw_times and len(ref) > 1000
        assert np.isfinite(ref).all()
        assert numpy_process(fmt, rec).tobytes() == ref.tobytes()
        got, bad, _ = emu_process(emu, fmt, rec)
        assert got.tobytes() == ref.tobytes() and bad == 0


def test_spins_cover_the_branches(flb):
    """What the synthetic spin is meant to reach: +-180, the spin's own wrap, spurious wraps from jitter, NaN records
    blocking a wrap, -0.0, an empty and a one-record ring."""
    rec, fmt = spin(flb, "xyzirt", 1, 1)
    a = np.frombuffer(rec, flb.synth.VELODYNE_LAYOUTS["xyzirt"][0])
    rings, counts = np.unique(a["ring"], return_counts=True)
    assert 1 not in rings and counts.min() == 1
    assert np.signbit(a["y"][a["y"] == 0]).any() and np.signbit(a["x"][a["x"] == 0]).any()
    assert np.isnan(a["x"]).sum() > 100
    yaw = np.degrees(np.arctan2(a["y"].astype(np.float64), a["x"].astype(np.float64)))
    assert (yaw > 179).any() and (yaw < -179).any()
    cloud, _ = velo_oracle.process(fmt, rec, sort=False)
    assert cloud[:, 3].max() > WRAP                          # a ring's time_last wrapped once the spin passed yaw_fp
    walk = {}                                                # the per-ring walk again, counting its wraps
    spurious = 0
    for i, r in enumerate(a["ring"]):
        y = velo_oracle.yaw(a["x"][i], a["y"][i])
        if r not in walk:
            walk[r] = (y, np.float32(0))
            continue
        yfp, last = walk[r]
        base = np.float32((yfp - y) / OMEGA) if y <= yfp else np.float32((yfp - y + 360.0) / OMEGA)
        wrapped = base < last
        t = np.float32(np.float64(base) + WRAP) if wrapped else base
        spurious += bool(wrapped and last - base < 1.0)       # a jitter of a fraction of a degree, not a full turn
        walk[r] = (yfp, t)
    assert spurious > 10


def test_golden(flb, emu):
    g = np.load(GOLDEN)
    for name in sorted({k.split("__")[0] for k in g.files}):
        layout, seed, pfn = name.split("-")
        rec, fmt = flb.synth.make_velodyne_spin(layout, int(seed[1:]), point_filter_num=int(pfn[1:]), n_scans=16, n_cols=60)
        assert rec == g[name + "__records"].tobytes()        # the generator has not drifted
        assert velo_oracle.process(fmt, rec)[0].tobytes() == g[name + "__cloud"].tobytes()
        assert emu_process(emu, fmt, rec)[0].tobytes() == g[name + "__cloud"].tobytes()
        assert numpy_process(fmt, rec).tobytes() == g[name + "__cloud"].tobytes()


def test_timed_layouts_take_the_time_route(flb):
    """With times the yaw is never used: the aligned layout is flb_lidar_upload's Velodyne rule, the packed one reads its
    time at byte 18."""
    rec, fmt = spin(flb, "xyzirt", 3, 2, timed=True)
    ref, yaw_times = velo_oracle.process(fmt, rec)
    assert not yaw_times
    assert ref.tobytes() == pre_oracle.process(lidar_format_of(fmt), rec).tobytes()
    rec22, fmt22 = spin(flb, "packed22", 3, 2, timed=True)
    a, b = (np.frombuffer(r, flb.synth.VELODYNE_LAYOUTS[k][0]) for r, k in ((rec, "xyzirt"), (rec22, "packed22")))
    assert a["time"].tobytes() == b["time"].tobytes() and a["x"].tobytes() == b["x"].tobytes()
    assert velo_oracle.process(fmt22, rec22)[0].tobytes() == ref.tobytes()


# ------------------------------------------------------------------------------------------------ the scan operator
def test_operator_is_associative(emu):
    rng = np.random.default_rng(5)
    special = np.float32([np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 99.72299])
    vals = np.where(rng.random((20000, 3, 3)) < 0.4, rng.choice(special, (20000, 3, 3)),
                    rng.uniform(-200, 200, (20000, 3, 3))).astype(np.float32)
    xs = np.where(rng.random(20000) < 0.3, rng.choice(special, 20000), rng.uniform(-200, 200, 20000)).astype(np.float32)
    ab, bc, l, r = (np.zeros(3, np.float32) for _ in range(4))
    for (f, g, h), x in zip(vals, xs):
        f, g, h = (np.ascontiguousarray(v) for v in (f, g, h))
        emu.emu_velo_compose(f.ctypes.data, g.ctypes.data, ab.ctypes.data)
        emu.emu_velo_compose(ab.ctypes.data, h.ctypes.data, l.ctypes.data)
        emu.emu_velo_compose(g.ctypes.data, h.ctypes.data, bc.ctypes.data)
        emu.emu_velo_compose(f.ctypes.data, bc.ctypes.data, r.ctypes.data)
        assert l.tobytes() == r.tobytes()
        # composition is application in order
        seq = emu.emu_velo_apply(h.ctypes.data, emu.emu_velo_apply(g.ctypes.data, emu.emu_velo_apply(f.ctypes.data, x)))
        assert np.float32(emu.emu_velo_apply(l.ctypes.data, x)).tobytes() == np.float32(seq).tobytes()


# ------------------------------------------------------------------------------------------------ hand-built cases
def records(flb, rows, layout="xyzirt"):
    """rows of (x, y, ring)"""
    dt, off_time = flb.synth.VELODYNE_LAYOUTS[layout]
    a = np.zeros(len(rows), dt)
    for i, (x, y, r) in enumerate(rows):
        a["x"][i], a["y"][i], a["z"][i], a["ring"][i] = x, y, 0.0, r
    fmt = dict(point_step=dt.itemsize, off_x=0, off_y=4, off_z=8, off_time=off_time, off_ring=dt.fields["ring"][1], n_scans=4,
               point_filter_num=1, blind=0.5)
    return a.tobytes(), fmt


def deg(d, r=10.0):
    return (r * np.cos(np.radians(d)), r * np.sin(np.radians(d)))


def all_three(emu, fmt, rec, sort=False):
    """The checker (unsorted unless `sort`), and the sorted results of all three."""
    ref = velo_oracle.process(fmt, rec, sort=sort)[0]
    srt = velo_oracle.process(fmt, rec)[0]
    assert numpy_process(fmt, rec).tobytes() == srt.tobytes()
    assert emu_process(emu, fmt, rec)[0].tobytes() == srt.tobytes()
    return ref


def t_of(yaw, yaw_fp, last):
    base = np.float32((yaw_fp - yaw) / OMEGA) if yaw <= yaw_fp else np.float32((yaw_fp - yaw + 360.0) / OMEGA)
    return np.float32(np.float64(base) + WRAP) if base < last else base


@pytest.mark.parametrize("layout", LAYOUTS)
def test_first_record_of_a_ring_is_never_kept(flb, emu, layout):
    rows = [(*deg(30 - 2 * i), i % 2) for i in range(8)]     # rings 0, 1, 0, 1, ...: records 0 and 1 are the heads
    rec, fmt = records(flb, rows, layout)
    for pfn, want in ((1, [2, 3, 4, 5, 6, 7]), (2, [2, 4, 6]), (3, [3, 6])):
        f = dict(fmt, point_filter_num=pfn)
        got = all_three(emu, f, rec)
        xs = np.float32([rows[i][0] for i in want])
        assert got[:, 0].tolist() == xs.tolist(), pfn       # the head used up its index: record 2 is the next kept at pfn 2


def test_equal_yaw_wrap_nan_and_negative_zero(flb, emu):
    yfp = velo_oracle.yaw(*np.float32(deg(10)))
    y_eq = velo_oracle.yaw(*np.float32(deg(10)))
    y5 = velo_oracle.yaw(*np.float32(deg(5)))
    y0 = velo_oracle.yaw(*np.float32(deg(0)))
    assert y_eq == yfp
    rows = [(*deg(10), 0), (*deg(10), 0), (*deg(5), 0), (*deg(10), 0),          # head; yaw == yaw_fp; 5 degrees on; a wrap
            (*deg(10), 1), (*deg(0), 1), (np.nan, np.nan, 1), (*deg(5), 1),     # head; 10 on; NaN; would wrap, but cannot
            (-10.0, 0.0, 2), (-10.0, -0.0, 2), (-0.0, -0.0, 2)]                   # head at +pi; -pi; atan2(-0, -0) = -pi
    rec, fmt = records(flb, rows)
    got = all_three(emu, fmt, rec)
    t = got[:, 3]
    t1 = t_of(y_eq, yfp, np.float32(0))
    t2 = t_of(y5, yfp, t1)
    t3 = t_of(y_eq, yfp, t2)
    assert t1 == 0 and 0 < t2 < t3 and t3 == np.float32(WRAP)
    assert t[:3].tolist() == [t1, t2, t3]
    yfp1 = velo_oracle.yaw(*np.float32(deg(10)))
    t5 = t_of(y0, yfp1, np.float32(0))
    t7 = np.float32((yfp1 - y5) / OMEGA)                      # below t5, yet no wrap after the NaN
    assert t7 < t5 and t[3:5].tolist() == [t5, t7]
    y_pi = velo_oracle.yaw(np.float32(-10.0), np.float32(0.0))
    y_mpi = velo_oracle.yaw(np.float32(-10.0), np.float32(-0.0))
    assert y_pi > 179.9 and y_mpi == -y_pi and velo_oracle.yaw(np.float32(-0.0), np.float32(-0.0)) == y_mpi
    assert np.float32((y_pi - y_mpi) / OMEGA) in t[5:].tolist()
    assert len(t) == 6                                        # out: the three heads, the NaN, (-0, -0, 0) inside blind


def test_bad_ring(flb, emu):
    rec, fmt = records(flb, [(*deg(1), 0), (*deg(2), 1), (*deg(3), 4), (*deg(4), 7)])
    with pytest.raises(velo_oracle.BadRing) as e:
        velo_oracle.process(fmt, rec)
    assert e.value.record == 2
    assert emu_process(emu, fmt, rec)[2] == 2
    # with times the ring is never read
    a = np.frombuffer(rec, flb.synth.VELODYNE_LAYOUTS["xyzirt"][0]).copy()
    a["time"] = [1e-5, 2e-5, 3e-5, 4e-5]
    assert not velo_oracle.process(fmt, a.tobytes())[1]


def test_yaw_rounding_modes(flb):
    """The defined yaw and libm's atan2f agree on most records and differ by at most one float ulp of the angle where they
    do not; the kept points and their count are the same, the times within a float ulp of the angle scaled to ms."""
    rec, fmt = spin(flb, "xyzirt", 1, 1)
    a, _ = velo_oracle.process(fmt, rec, velo_oracle.YAW_DEFINED)
    b, _ = velo_oracle.process(fmt, rec, velo_oracle.YAW_ATAN2F)
    assert len(a) == len(b)
    ia, ib = np.lexsort((a[:, 2], a[:, 1], a[:, 0])), np.lexsort((b[:, 2], b[:, 1], b[:, 0]))
    assert a[ia, :3].tobytes() == b[ib, :3].tobytes()
    assert_time_bound(a[ia, 3], b[ib, 3])
