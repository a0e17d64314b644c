"""CPU tier of flb_lidar_upload / flb_imu_undistort_lidar's window.  Three statements of Preprocess::process's non-feature
branches (reference src/preprocess.cpp), the stable time sort (src/laserMapping.cpp:551) and UndistortPcl's window
(src/IMU_Processing.cpp:634) must agree byte for byte on every synthetic driver message: the checker
(tests/oracle_pre/pre_oracle.cpp, a serial loop like the reference), a vectorised numpy restatement written here, and the
product's per-record device math compiled for the host (tests/hostemu/lidar_decode.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pre_oracle
from lidar_util import CASES, case_id, message, rounding_message, scan_end_offset

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "lidar_golden.npz")
SIZES = [0, 1, 2, 255, 256, 257, 5000]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/lidar_decode.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("lidar_decode") / "liblidar_decode.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "lidar_decode.cpp")])
    L = C.CDLL(so)
    L.emu_lidar_decode.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.emu_lidar_window.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double]
    return L


def emu_decode(L, fmt, records):
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // fmt["point_step"]
    ints = np.array([fmt[k] for k in pre_oracle.FIELDS], np.int32)
    out = np.zeros((max(n, 1), 4), np.float32)
    bad, was_sorted = C.c_int(), C.c_int()
    m = L.emu_lidar_decode(ints.ctypes.data, fmt["blind"], rec.ctypes.data if n else None, n, out.ctypes.data, C.byref(bad), C.byref(was_sorted))
    return out[:m], bad.value, was_sorted.value


def numpy_process(fmt, records):
    """The same arithmetic without a loop over the records."""
    step, kind, pfn, blind = fmt["point_step"], fmt["kind"], fmt["point_filter_num"], np.float64(fmt["blind"])
    raw = np.frombuffer(records, np.uint8).reshape(-1, step)
    n = len(raw)

    def col(off, dtype):
        return np.ascontiguousarray(raw[:, off:off + np.dtype(dtype).itemsize]).view(dtype)[:, 0]

    xyz = np.stack([col(fmt["off_x"], "<f4"), col(fmt["off_y"], "<f4"), col(fmt["off_z"], "<f4")], 1)
    idx = np.arange(n)
    with np.errstate(all="ignore"):
        r2 = ((xyz[:, 0] * xyz[:, 0] + xyz[:, 1] * xyz[:, 1]) + xyz[:, 2] * xyz[:, 2]).astype(np.float64)
    if kind == 1:
        tag = col(fmt["off_tag"], "u1") & 0x30
        valid = (idx >= 1) & (col(fmt["off_line"], "u1").astype(np.int64) < fmt["n_scans"]) & ((tag == 0x10) | (tag == 0x00))
        valid_num = np.cumsum(valid)
        cand = valid & (valid_num % pfn == 0)
        prev = np.zeros_like(xyz)
        prev[1:][cand[:-1]] = xyz[:-1][cand[:-1]]
        moved = (np.abs(xyz - prev).astype(np.float64) > 1e-7).any(1)
        keep = cand & moved & (r2 > blind * blind)
        t = col(fmt["off_time"], "<u4").astype(np.float32) / np.float32(1000000)
    elif kind == 3:
        keep = (idx % pfn == 0) & ~(r2 < blind * blind)
        t = col(fmt["off_time"], "<u4").astype(np.float32) * np.float32(1.e-6)
    elif kind == 2:
        keep = (idx % pfn == 0) & (r2 > blind * blind)
        t = col(fmt["off_time"], "<f4") * np.float32(1.e-3)
    else:
        keep = (idx % pfn == 0) & (r2 > blind)
        ts = col(fmt["off_time"], "<f8")
        t = ((ts - (ts[0] if n else 0.0)) * 1000.0).astype(np.float32)
    cloud = np.concatenate([xyz[keep], t[keep, None]], 1).astype(np.float32)
    return cloud[np.argsort(cloud[:, 3], kind="stable")]


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_three_statements_agree(flb, emu, case):
    for n in SIZES:
        rec, fmt = message(flb, case, n)
        ref = pre_oracle.process(fmt, rec)
        assert ref.tobytes() == numpy_process(fmt, rec).tobytes(), n
        got, bad, was_sorted = emu_decode(emu, fmt, rec)
        assert got.tobytes() == ref.tobytes(), n
        assert bad == 0
        unsorted_in = pre_oracle.process(fmt, rec, sort=False)
        assert was_sorted == int((np.diff(unsorted_in[:, 3]) >= 0).all())


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_golden(flb, emu, case):
    g = np.load(GOLDEN)
    rec, fmt = message(flb, case, 1000)
    name = case_id(case)
    assert rec == g[name + "__records"].tobytes()            # the generator has not drifted
    assert pre_oracle.process(fmt, rec).tobytes() == g[name + "__cloud"].tobytes()
    assert emu_decode(emu, fmt, rec)[0].tobytes() == g[name + "__cloud"].tobytes()


def test_messages_cover_the_branches(flb):
    """The synthetic messages reach what they are meant to reach."""
    rec, fmt = flb.synth.make_lidar_message("livox", 1, 24000)
    a = np.frombuffer(rec, flb.synth.LIVOX_POINT)
    assert set(np.unique(a["tag"] & 0x30)) == {0x00, 0x10, 0x20, 0x30} and (a["tag"] & 0xCF).any()
    assert (a["line"] >= fmt["n_scans"]).any()
    cloud = pre_oracle.process(fmt, rec)
    assert (np.diff(cloud[:, 3]) == 0).sum() > 1000                                # lines fired together
    assert not (np.abs(cloud[:, :3]).sum(1) == 0).any()                            # no-return points are dropped
    assert ((cloud[:, :3].astype(np.float64) ** 2).sum(1) > fmt["blind"] ** 2 * 0.999).all()
    rec_o, fmt_o = flb.synth.make_lidar_message("ouster", 1, 24000)
    assert (np.diff(pre_oracle.process(fmt_o, rec_o, sort=False)[:, 3]) < 0).any()   # the sort has work to do
    assert pre_oracle.process(*reversed(flb.synth.make_lidar_message("velodyne_notime", 1, 100))) is None


def test_livox_record_zero_and_duplicate_after_untaken_record(flb, emu):
    P = flb.synth.LIVOX_POINT
    a = np.zeros(6, P)
    a["x"], a["y"], a["z"] = [5, 5, 7, 7, 7, 7], 1.0, 0.5
    a["offset_time"] = np.arange(6) * 1000
    a["tag"] = [0x10, 0x10, 0x10, 0x20, 0x10, 0x10]          # record 3 is not valid
    fmt = dict(kind=1, point_step=20, off_time=0, off_x=4, off_y=8, off_z=12, off_tag=17, off_line=18, n_scans=6,
               point_filter_num=1, blind=0.5)
    for f in (pre_oracle.process, numpy_process, lambda fm, r: emu_decode(emu, fm, r)[0]):
        c = f(fmt, a.tobytes())
        # 0: never visited.  1: compared with zeros (record 0 was not taken), kept.  2: moved, kept.  3: invalid.
        # 4: repeats record 3, which was not taken, so it is compared with zeros and kept.  5: repeats record 4, dropped.
        assert c[:, 3].tolist() == [np.float32(1000) / np.float32(1e6), np.float32(2000) / np.float32(1e6), np.float32(4000) / np.float32(1e6)]
        assert c[:, 0].tolist() == [5.0, 7.0, 7.0]
    fmt2 = dict(fmt, point_filter_num=2)                     # valid_num: 1, 2, (invalid), 3, 4 -> records 2 and 5 are taken
    for f in (pre_oracle.process, numpy_process, lambda fm, r: emu_decode(emu, fm, r)[0]):
        c = f(fmt2, a.tobytes())
        assert c[:, 3].tolist() == [np.float32(2000) / np.float32(1e6), np.float32(5000) / np.float32(1e6)]   # 5 repeats 4, which was not taken


def test_xt32_blind_is_not_squared(flb, emu):
    a = np.zeros(3, flb.synth.XT32_POINT)
    a["x"] = [0.7, 0.85, 2.0]                                # squares 0.49, 0.7225, 4: blind 0.64 keeps the last two
    a["timestamp"] = 1.7e9 + np.arange(3) * 1e-4
    fmt = dict(kind=4, point_step=32, off_x=0, off_y=4, off_z=8, off_time=16, off_tag=0, off_line=0, n_scans=32,
               point_filter_num=1, blind=0.64)
    for f in (pre_oracle.process, numpy_process, lambda fm, r: emu_decode(emu, fm, r)[0]):
        assert f(fmt, a.tobytes())[:, 0].tolist() == [np.float32(0.85), 2.0]
    fmt_v = dict(fmt, kind=2, point_step=24, off_time=20)    # the same distances through the Velodyne rule (blind squared)
    b = np.zeros(3, flb.synth.VELODYNE_POINT)
    b["x"], b["time"] = a["x"], [1e-4, 2e-4, 3e-4]
    assert pre_oracle.process(fmt_v, b.tobytes())[:, 0].tolist() == [np.float32(0.7), np.float32(0.85), 2.0]


def test_non_finite_kept_value_is_flagged(flb, emu):
    rec, fmt = flb.synth.make_lidar_message("ouster", 4, 300)
    a = np.frombuffer(rec, flb.synth.OUSTER_POINT).copy()
    a["x"][30] = np.inf                                      # record 30 is taken (30 % 3 == 0)
    assert emu_decode(emu, fmt, a.tobytes())[1] == 1
    a["x"][30] = 1.0
    a["x"][31] = np.nan                                      # record 31 is not
    assert emu_decode(emu, fmt, a.tobytes())[1] == 0


@pytest.mark.parametrize("case", [CASES[0], CASES[3]], ids=case_id)
def test_window(flb, emu, case):
    rec, fmt = message(flb, case, 5000)
    p48 = pre_oracle.process48(fmt, rec)
    cloud = np.ascontiguousarray(p48[:, [0, 1, 2, 9]])
    n, last = len(cloud), cloud[-1, 3]
    for begin in (0, 17, n):
        for off in (0.0, -1.0, float(cloud[n // 3, 3]), float(last), np.nextafter(np.float64(last), 0.0), 1e9):
            want = len(pre_oracle.window(p48, begin, off))
            assert emu.emu_lidar_window(cloud.ctypes.data, begin, n, off) == want
            assert want == int((cloud[begin:, 3].astype(np.float64) <= off).sum())
    # a scan-end pcl_offset_time that rounds below the last time leaves the last point(s) out (:628-634)
    rec, fmt = rounding_message(flb, case, 5000)
    p48 = pre_oracle.process48(fmt, rec)
    cloud = np.ascontiguousarray(p48[:, [0, 1, 2, 9]])
    n, last = len(cloud), cloud[-1, 3]
    _, off = scan_end_offset(1.7e9, last)
    assert off < float(last)
    want = len(pre_oracle.window(p48, 0, off))
    assert want < n and want == int((cloud[:, 3].astype(np.float64) <= off).sum())
    assert emu.emu_lidar_window(cloud.ctypes.data, 0, n, off) == want
