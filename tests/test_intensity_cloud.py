"""CPU tier of the LiDAR clouds' intensity (flb_lidar_upload_intensity, flb_lidar_download_points, flb_scan_from_undistorted's
leaf mean, flb_world_cloud_points and flb_lidar_save_*), from the rules the device applies compiled for the host
(tests/hostemu/intensity_cloud.cpp): the decode route with its intensity and the two stable sorts on one set of time keys,
the 48-byte pcl::PointXYZINormal records, the voxel grid's all-data intensity mean and the chunked save with its
expansion.  The records must be byte-identical to the checker's pl_surf (tests/oracle_pre/intensity_oracle.cpp: each
handler with its intensity line), and to records packed in numpy, on seeded messages and clouds from synth.py: equal-time ties
with differing intensities, leaves of one point and of many, a NaN intensity, and save slices across chunk boundaries."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pre_oracle
from intensity_oracle import XYZINORMAL_POINT
from intensity_oracle import process as oracle_process
from conftest import bits

HERE = os.path.dirname(os.path.abspath(__file__))
# the intensity field of each synthetic kind: Livox reflectivity (u8), the others' float32 intensity
OFF_INTENSITY = {"livox": 16, "ouster": 16, "velodyne": 12, "xt32": 12}


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("intensity_emu") / "libintensity_cloud.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "intensity_cloud.cpp")])
    L = C.CDLL(so)
    L.emu_lidar_points48.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_int, C.c_void_p]
    L.emu_vg_intensity.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_save_new.restype = C.c_void_p
    L.emu_save_free.argtypes = [C.c_void_p]
    L.emu_save_size.argtypes = [C.c_void_p]
    L.emu_save_size.restype = C.c_longlong
    L.emu_xyzi_cloud.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.emu_save_download.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    return L


def with_intensity(flb, kind, seed, n, pfn, unsorted, ties=False, nan=False):
    """A synth.py message whose intensities are set from a seeded generator.  ties: Ouster-like records whose times tie
    in groups (the Livox lines share their time already).  nan: one kept point's intensity is a NaN."""
    rec, fmt = flb.synth.make_lidar_message(kind, seed, n, point_filter_num=pfn, unsorted=unsorted)
    dt = {"livox": flb.synth.LIVOX_POINT, "ouster": flb.synth.OUSTER_POINT, "velodyne": flb.synth.VELODYNE_POINT,
          "xt32": flb.synth.XT32_POINT}[kind]
    a = np.frombuffer(rec, dt).copy()
    rng = np.random.default_rng(77 + seed)
    if kind == "livox":
        a["reflectivity"] = rng.integers(0, 256, len(a))
    else:
        a["intensity"] = rng.uniform(0, 255, len(a)).astype(np.float32)
        if nan:
            a["intensity"][::97] = np.nan
    if ties and kind == "ouster":
        a["t"] = (np.arange(len(a)) // 8)[::-1] * 1000                       # reversed groups of 8 equal times
    return a.tobytes(), fmt


CASES = [("livox", 1, 1, None), ("livox", 3, 3, True), ("ouster", 1, 3, None), ("ouster", 2, 1, False), ("velodyne", 2, 2, True),
         ("xt32", 1, 3, None), ("xt32", 2, 1, True)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-s{c[1]}-f{c[2]}-{c[3]}")
@pytest.mark.parametrize("n", [0, 1, 257, 5000])
def test_decode_records_match_oracle(flb, emu, case, n):
    kind, seed, pfn, unsorted = case
    rec, fmt = with_intensity(flb, kind, seed, n, pfn, unsorted, nan=(seed == 2))
    for off in (OFF_INTENSITY[kind], -1):
        ref = oracle_process(fmt, rec, off)
        got = np.zeros(max(n, 1), XYZINORMAL_POINT)
        ints = np.array([int(fmt[k]) for k in pre_oracle.FIELDS], np.int32)
        raw = np.frombuffer(rec, np.uint8)
        m = emu.emu_lidar_points48(_p(ints), off, float(fmt["blind"]), _p(raw) if raw.size else None, n, _p(got))
        assert m == len(ref)
        assert got[:m].tobytes() == ref.tobytes()
        if off == -1:
            assert (bits(ref["intensity"]) == 0).all()
        # the checker's x, y, z, curvature are the plain upload's (pre_oracle.process48 without an intensity)
        plain = pre_oracle.process48(fmt, rec)
        assert bits(ref.view(np.float32).reshape(-1, 12)[:, [0, 1, 2, 9]]).tobytes() == bits(plain[:, [0, 1, 2, 9]]).tobytes()


def test_equal_times_keep_record_order_with_their_intensity(flb, emu):
    rec, fmt = with_intensity(flb, "ouster", 5, 4096, 1, False, ties=True)
    ref = oracle_process(fmt, rec, 16)
    t = ref["curvature"]
    assert (np.diff(t) >= 0).all() and (np.diff(t) == 0).sum() > 1000        # ties
    ties = np.flatnonzero(np.diff(t) == 0)
    assert (ref["intensity"][ties] != ref["intensity"][ties + 1]).any()          # whose intensities differ
    got = np.zeros(4096, XYZINORMAL_POINT)
    ints = np.array([int(fmt[k]) for k in pre_oracle.FIELDS], np.int32)
    raw = np.frombuffer(rec, np.uint8)
    m = emu.emu_lidar_points48(_p(ints), 16, float(fmt["blind"]), _p(raw), 4096, _p(got))
    assert got[:m].tobytes() == ref.tobytes()


def leaf_order(xyz, leaf):
    """voxel_grid_dev's leaf keys and the stable sort of the input by them (input order within a leaf): the defined
    order of tests/test_voxel_grid.py's oracle."""
    inv = np.float32(1.0) / np.float32(leaf)
    lo = np.floor(xyz.min(0) * inv).astype(np.int64)
    hi = np.floor(xyz.max(0) * inv).astype(np.int64)
    div = hi - lo + 1
    ijk = np.floor(xyz * inv).astype(np.int64) - lo
    key = (ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]).astype(np.uint32)
    order = np.argsort(key, kind="stable").astype(np.int32)
    return np.ascontiguousarray(key[order]), order


def leaf_means(values, key_sorted, order):
    """Each leaf's float32 sum in sorted order over float32(count), in numpy."""
    heads = np.flatnonzero(np.r_[True, key_sorted[1:] != key_sorted[:-1]])
    ends = np.r_[heads[1:], len(key_sorted)]
    out = []
    for a, b in zip(heads, ends):
        s = np.float32(0)
        for j in order[a:b]:
            s = np.float32(s + values[j])
        out.append(np.float32(s / np.float32(b - a)))
    return np.array(out, np.float32).reshape((len(out),) + values.shape[1:])


@pytest.mark.parametrize("leaf", [0.2, 0.5, 3.0])
def test_voxel_intensity_mean(flb, po, emu, leaf):
    xyz = flb.synth.make_frame("T1")["scan_body"][:6000]
    rng = np.random.default_rng(int(leaf * 10))
    inten = rng.uniform(0, 255, len(xyz)).astype(np.float32)
    inten[17] = np.nan
    key_sorted, order = leaf_order(xyz, leaf)
    # the grouping is the oracle's: the same sums give po.voxel_grid's centroids bit for bit
    cen = np.stack([leaf_means(xyz[:, k], key_sorted, order) for k in range(3)], 1)
    assert (bits(cen) == bits(po.voxel_grid(xyz, leaf))).all()
    ref = leaf_means(inten, key_sorted, order)
    counts = np.diff(np.r_[np.flatnonzero(np.r_[True, key_sorted[1:] != key_sorted[:-1]]), len(key_sorted)])
    assert (counts == 1).any() and counts.max() > 3                            # leaves of one point and of many
    assert np.isnan(ref).sum() == 1
    got = np.zeros(len(xyz), np.float32)
    m = emu.emu_vg_intensity(_p(key_sorted), _p(order), len(xyz), _p(inten), _p(got))
    assert m == len(ref) and (bits(got[:m]) == bits(ref)).all()


def pack_records(xyz, inten):
    out = np.zeros(len(xyz), XYZINORMAL_POINT)
    out["x"], out["y"], out["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    out["w"] = 1.0
    out["intensity"] = inten
    return out


def test_world_records_and_save(flb, emu):
    rng = np.random.default_rng(3)
    save = emu.emu_save_new(7)                                                  # 128-record chunks
    frames = []
    try:
        for k, n in enumerate([0, 1, 127, 128, 300, 1000]):
            xyz = rng.normal(0, 30, (n, 3)).astype(np.float32)
            inten = rng.uniform(0, 255, n).astype(np.float32)
            if n > 10:
                inten[5] = np.nan
            out = np.zeros(max(n, 1), XYZINORMAL_POINT)
            emu.emu_xyzi_cloud(_p(xyz), _p(inten), n, _p(out), save)
            ref = pack_records(xyz, inten)
            assert out[:n].tobytes() == ref.tobytes()
            frames.append(ref)
        allrec = np.concatenate(frames)
        assert emu.emu_save_size(save) == len(allrec)
        for first, count in [(0, len(allrec)), (100, 200), (127, 2), (255, 129), (len(allrec) - 1, 1), (5, 0)]:
            got = np.zeros(max(count, 1), XYZINORMAL_POINT)
            emu.emu_save_download(save, first, count, _p(got))
            assert got[:count].tobytes() == allrec[first:first + count].tobytes()
    finally:
        emu.emu_save_free(save)
