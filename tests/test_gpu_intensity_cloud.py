"""GPU tier: intensity through the device chain of a LiDAR frame.  flb_lidar_upload_intensity /
flb_lidar_upload_velodyne_intensity / the feature calls -> flb_lidar_download_points against the checker's time-sorted
pl_surf byte for byte; flb_imu_undistort_lidar -> flb_world_cloud -> flb_world_cloud_points (publish_frame_world's
pcl_wait_pub) against the checker's window; flb_scan_from_undistorted's leaf mean; the effect cloud's intensities; the
LiDAR save (pcl_wait_save_lidar); and every refusal.  Expected values come from tests/oracle_pre and numpy only."""
import ctypes as C

import numpy as np
import pytest

import intensity_oracle
import pre_oracle
from conftest import bits
from imu_util import product_inputs
from lidar_util import c_format, rounding_message, scan_end_offset
from test_intensity_cloud import OFF_INTENSITY, XYZINORMAL_POINT, leaf_means, leaf_order, oracle_process, with_intensity

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
VELO_FIELDS = ("point_step", "off_x", "off_y", "off_z", "off_time", "off_ring", "n_scans", "point_filter_num")


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def velo_format(flb, fmt):
    f = flb.capi.VelodyneFormat()
    for k in VELO_FIELDS + ("blind",):
        setattr(f, k, fmt[k])
    return f


def same(a, b):
    """Bit-equal floats, except that a NaN matches any NaN: an average that meets a NaN gives the device's canonical NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and (bits(a[~nan]) == bits(b[~nan])).all()


def records48(xyzt, inten):
    out = np.zeros(len(xyzt), XYZINORMAL_POINT)
    out["x"], out["y"], out["z"], out["curvature"] = xyzt[:, 0], xyzt[:, 1], xyzt[:, 2], xyzt[:, 3]
    out["w"] = 1.0
    out["intensity"] = inten
    return out


def xyzt_bytes(recs):
    return np.ascontiguousarray(recs.view(np.float32).reshape(-1, 12)[:, [0, 1, 2, 9]]).tobytes()


# ------------------------------------------------------------------------------------------------ the raw cloud
ROUTES = [("livox", 1, 1, None), ("livox", 3, 3, True), ("ouster", 1, 3, None), ("ouster", 2, 1, False), ("velodyne", 1, 3, None),
          ("velodyne", 2, 2, True), ("xt32", 1, 3, None), ("xt32", 2, 1, True)]


@pytest.mark.parametrize("case", ROUTES, ids=lambda c: f"{c[0]}-s{c[1]}-f{c[2]}-{c[3]}")
@pytest.mark.parametrize("absent", [False, True])
def test_download_points_match_oracle(flb, case, absent):
    kind, seed, pfn, unsorted = case
    rec, fmt = with_intensity(flb, kind, seed, 24000, pfn, unsorted, nan=(seed == 2))
    off = -1 if absent else OFF_INTENSITY[kind]
    ref = oracle_process(fmt, rec, off)
    h = flb.Handle(device=0)
    raw = np.frombuffer(rec, np.uint8)
    n, last = h.lidar_upload_intensity(c_format(flb, fmt), raw, off)
    got = h.lidar_download_points()
    assert n == len(ref) == len(got) > 100
    assert got.tobytes() == ref.tobytes()
    assert last == (ref["curvature"][-1] if n else 0)
    h.lidar_upload(c_format(flb, fmt), raw)                    # the plain call: the same x, y, z, curvature bytes
    assert h.lidar_download().tobytes() == xyzt_bytes(got)
    expect_error(flb, ERR_STATE, h.lidar_download_points)       # ... and no intensity
    h.close()


@pytest.mark.parametrize("layout,timed", [("xyzirt", False), ("packed22", False), ("packed22", True), ("xyzir32", False)])
def test_velodyne_routes(flb, layout, timed):
    rec, fmt = flb.synth.make_velodyne_spin(layout, seed=3, timed=timed)
    off = flb.synth.VELODYNE_LAYOUTS[layout][0].fields["intensity"][1]
    xyzt, inten = intensity_oracle.process_velodyne(fmt, rec, off)
    h = flb.Handle(device=0)
    raw = np.frombuffer(rec, np.uint8)
    n, _, yaw = h.lidar_upload_velodyne_intensity(velo_format(flb, fmt), raw, off)
    assert yaw == (not timed or fmt["off_time"] < 0)
    got = h.lidar_download_points()
    assert n == len(xyzt) > 1000
    assert got.tobytes() == records48(xyzt, inten).tobytes()
    h.lidar_upload_velodyne(velo_format(flb, fmt), raw)
    assert h.lidar_download().tobytes() == xyzt_bytes(got)
    n, _, _ = h.lidar_upload_velodyne_intensity(velo_format(flb, fmt), raw, -1)
    assert (bits(h.lidar_download_points()["intensity"]) == 0).all()
    h.close()


@pytest.mark.parametrize("kind", ["livox", "ouster", "velodyne"])
def test_feature_calls_carry_zero_intensity(flb, kind):
    rec, fmt = flb.synth.make_feature_scan(kind, 1, nan_returns=False)     # a NaN return would be refused as not finite
    raw = np.frombuffer(rec, np.uint8)
    h = flb.Handle(device=0)
    if kind == "velodyne":
        vfmt = dict(fmt, off_ring=fmt["off_line"])
        n = h.lidar_upload_velodyne_features(velo_format(flb, vfmt), raw)[0]
    else:
        n = h.lidar_upload_features(c_format(flb, fmt), raw)[0]
    got = h.lidar_download_points()
    assert n == len(got) > 100
    assert xyzt_bytes(got) == h.lidar_download().tobytes()
    assert (bits(got["intensity"]) == 0).all() and (bits(got["w"]) == bits(np.float32(1))).all()
    h.close()


# ------------------------------------------------------------------------------------------------ window -> world cloud
def shifted_imu(flb, seed, beg):
    fi = flb.synth.make_imu_frame(seed=seed, n_points=0)
    shift = beg - fi["pcl_beg_time"]
    v_imu = fi["v_imu"].copy()
    v_imu[:, 0] += shift
    return dict(fi, v_imu=v_imu, last_lidar_end_time=fi["last_lidar_end_time"] + shift)


def test_world_cloud_points_follow_the_window(flb, frames):
    """Two camera updates (windows that start mid-cloud), then a scan end whose pcl_offset_time drops the last points."""
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    rec, fmt = rounding_message(flb, ("ouster", 1, 1, None), 24000)
    a = np.frombuffer(rec, flb.synth.OUSTER_POINT).copy()
    a["intensity"] = np.random.default_rng(5).uniform(0, 255, len(a)).astype(np.float32)
    rec = a.tobytes()
    ref = oracle_process(fmt, rec, 16)
    p48 = np.ascontiguousarray(ref.view(np.float32).reshape(-1, 12))
    beg = 1.7e9
    end, off_end = scan_end_offset(beg, p48[-1, 9])
    fi = shifted_imu(flb, 33, beg)
    h = flb.Handle(device=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    h.lidar_upload_intensity(c_format(flb, fmt), np.frombuffer(rec, np.uint8), 16)
    index_now, t_prev, takes = 0, beg, []
    for off, t_end, is_end in ((0.0, beg + 0.005, False), (0.0, beg + 0.010, False), (off_end, end, True)):
        win = pre_oracle.window(p48, index_now, off)
        taken, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], t_prev, t_end, off, is_end, download=False)
        assert taken == len(win)
        takes.append(taken)
        for R, p in ((f["R_true"], f["p_true"]), (None, None)):
            n = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, R, p)
            got = h.world_cloud_points()
            assert n == taken == len(got)
            xyz = h.world_cloud_download()
            assert np.ascontiguousarray(got.view(np.float32).reshape(-1, 12)[:, :3]).tobytes() == xyz.tobytes()
            assert (bits(got["intensity"]) == bits(win[:, 8])).all()
            assert (bits(got["w"]) == bits(np.float32(1))).all()
            assert not got["normal"].any() and not got["curvature"].any() and not got["pad"].any()
        index_now = 0 if is_end else index_now + taken
        t_prev = t_end
    assert takes[0] > 0 and takes[1] == 0 and 0 < takes[2] < len(p48) - takes[0]
    h.close()


def device_scan(flb, h, f, leaf, n=None, seed=9):
    """An Ouster message made of the frame's body points (all kept, in order), with random intensities, uploaded and
    undistorted whole, then filtered into the scan.  Returns (undistorted xyz, intensities, leaf count)."""
    body = f["scan_body"] if n is None else f["scan_body"][:n]
    a = np.zeros(len(body), flb.synth.OUSTER_POINT)
    a["x"], a["y"], a["z"] = body[:, 0], body[:, 1], body[:, 2]
    a["t"] = np.arange(len(body)) * (90_000_000 // max(len(body), 1))          # ns, in order, within the scan
    inten = np.random.default_rng(seed).uniform(0, 255, len(body)).astype(np.float32)
    inten[3] = np.nan
    a["intensity"] = inten
    fmt = dict(kind=3, point_step=48, off_x=0, off_y=4, off_z=8, off_time=20, off_tag=0, off_line=0, n_scans=64, point_filter_num=1,
               blind=0.0)
    fi = flb.synth.make_imu_frame(seed=seed, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    assert h.lidar_upload_intensity(c_format(flb, fmt), np.frombuffer(a.tobytes(), np.uint8), 16)[0] == len(body)
    taken, xyz, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True)
    assert taken == len(body)
    return xyz, inten, h.scan_from_undistorted(leaf)


@pytest.mark.parametrize("name,leaf", [("T0", 0.15), ("C2", 0.15), ("C2", 0.5)])
def test_scan_leaf_mean(flb, po, frames, name, leaf):
    f = frames(name)
    prm = flb.capi.lio_params(f, 3)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    xyz, inten, m = device_scan(flb, h, f, leaf)
    key_sorted, order = leaf_order(xyz, leaf)
    ref = leaf_means(inten, key_sorted, order)
    assert m == len(ref) == len(po.voxel_grid(xyz, leaf))
    assert h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_true"], f["p_true"]) == m
    got = h.world_cloud_points()
    assert same(got["intensity"], ref) and np.isnan(ref).sum() == 1
    assert np.ascontiguousarray(got.view(np.float32).reshape(-1, 12)[:, :3]).tobytes() == h.world_cloud_download().tobytes()
    h.close()


def test_effect_cloud_intensity(flb, frames):
    f = frames("T1")
    prm = flb.capi.lio_params(f, 3)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.map_upload(f["map_xyz"])
    xyz, inten, m = device_scan(flb, h, f, 0.15)
    assert h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_true"], f["p_true"]) == m
    scan_int = h.world_cloud_points()["intensity"]
    R, p = f["R_true"], f["p_true"]
    g = h.lio_pass(prm, R, p, True)
    assert h.effect_cloud(prm, R, p) == g["n"] > 50
    got = h.effect_cloud_download_points()
    assert np.ascontiguousarray(got.view(np.float32).reshape(-1, 12)[:, :3]).tobytes() == h.effect_cloud_download().tobytes()
    assert (bits(got["intensity"]) == bits(scan_int[g["sel_idx"]])).all()
    assert not got["curvature"].any()
    # one more scan install keeps the pass's rows (and intensities) capturable
    h2 = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h2.map_upload(f["map_xyz"])
    device_scan(flb, h2, f, 0.15)
    g2 = h2.lio_pass(prm, R, p, True)
    h2.scan_upload(f["scan_body"][:100])
    assert h2.effect_cloud(prm, R, p) == g2["n"]
    assert h2.effect_cloud_download_points().tobytes() == got.tobytes()
    # a host-uploaded scan carries no intensity
    h2.lio_pass(prm, R, p, True)
    h2.effect_cloud(prm, R, p)
    expect_error(flb, ERR_STATE, h2.effect_cloud_download_points)
    h.close()
    h2.close()


# ------------------------------------------------------------------------------------------------ the LiDAR save
def test_lidar_save(flb, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    rec, fmt = with_intensity(flb, "ouster", 4, 400_000, 1, None)
    h = flb.Handle(device=0)
    fi = flb.synth.make_imu_frame(seed=4, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    h.lidar_upload_intensity(c_format(flb, fmt), np.frombuffer(rec, np.uint8), 16)
    h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True, download=False)
    expect_error(flb, ERR_STATE, h.lidar_save_size)
    expect_error(flb, ERR_INVALID, h.lidar_save_begin, 0)
    h.rgb_save_begin(10)                                        # the RGB save is independent
    n = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
    assert n > 300_000
    cap = 4 * n + n // 2
    h.lidar_save_begin(cap)
    expect_error(flb, ERR_STATE, h.lidar_save_begin, 5)
    frames_rec = []
    for k in range(5):                                          # four frames fit (past one 2^20 chunk), the fifth is dropped
        p = np.asarray(f["p_true"]) + [0.1 * k, 0.0, 0.0]
        h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], p)
        if k == 2:                                              # no download: the append alone
            assert h.world_cloud_points(download=False) == n
            frames_rec.append(None)
        else:
            frames_rec.append(h.world_cloud_points())
    assert len(frames_rec[4]) == n                              # a dropped frame's cloud is still built
    sz = h.lidar_save_size()
    assert sz["n"] == 4 * n and sz["dropped"] == n and 4 * n > (1 << 20)
    assert h.rgb_save_size() == dict(n=0, dropped=0, device_bytes=0)
    allrec = h.lidar_save_download()
    assert len(allrec) == 4 * n
    # frame k's save records are its published records
    assert allrec[:n].tobytes() == frames_rec[0].tobytes()
    assert allrec[n:2 * n].tobytes() == frames_rec[1].tobytes()
    assert allrec[3 * n:].tobytes() == frames_rec[3].tobytes()
    for first, count in [(0, 1), ((1 << 20) - 3, 7), (2 * n - 5, 300_000), (4 * n - 1, 1), (7, 0)]:
        assert h.lidar_save_download(first, count).tobytes() == allrec[first:first + count].tobytes()
    expect_error(flb, ERR_INVALID, h.lidar_save_download, 4 * n - 1, 2)
    h.lidar_save_end()
    expect_error(flb, ERR_STATE, h.lidar_save_size)
    assert h.rgb_save_size()["n"] == 0                          # still open
    h.rgb_save_end()
    h.lidar_save_end()                                          # no save open: nothing to do
    h.close()


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(flb, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    h = flb.Handle(device=0)
    expect_error(flb, ERR_STATE, h.lidar_download_points)                        # no cloud
    rec, fmt = with_intensity(flb, "ouster", 1, 5000, 3, None)
    raw = np.frombuffer(rec, np.uint8)
    cf = c_format(flb, fmt)
    h.lidar_upload_intensity(cf, raw, 16)
    ref = h.lidar_download_points()
    for off in (13, 46, 48, -2, -100):                                           # misaligned, past the step, negative
        expect_error(flb, ERR_INVALID, h.lidar_upload_intensity, cf, raw, off)
    assert h.lidar_download_points().tobytes() == ref.tobytes()                  # a refusal keeps the cloud
    lrec, lfmt = with_intensity(flb, "livox", 1, 5000, 1, None)
    expect_error(flb, ERR_INVALID, h.lidar_upload_intensity, c_format(flb, lfmt), np.frombuffer(lrec, np.uint8), 20)
    h.lidar_upload_intensity(c_format(flb, lfmt), np.frombuffer(lrec, np.uint8), 17)   # a u8 at any byte
    vrec, vfmt = flb.synth.make_velodyne_spin("packed22", seed=2)
    vf = velo_format(flb, vfmt)
    expect_error(flb, ERR_INVALID, h.lidar_upload_velodyne_intensity, vf, np.frombuffer(vrec, np.uint8), 19)
    h.lidar_upload_velodyne_intensity(vf, np.frombuffer(vrec, np.uint8), 13)     # any alignment
    # host-uploaded sources carry none
    fi = flb.synth.make_imu_frame(seed=2, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    pts = np.concatenate([f["scan_body"], np.linspace(0, 90, len(f["scan_body"]), dtype=np.float32)[:, None]], 1)
    h.imu_undistort(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], pts, offset_index=3, download=False)
    h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
    expect_error(flb, ERR_STATE, h.world_cloud_points)
    h.scan_from_undistorted(0.2)
    h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_true"], f["p_true"])
    expect_error(flb, ERR_STATE, h.world_cloud_points)
    h.scan_upload(f["scan_body"])
    h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_true"], f["p_true"])
    expect_error(flb, ERR_STATE, h.world_cloud_points)
    expect_error(flb, ERR_INVALID, h.world_cloud, prm, 7, f["R_true"], f["p_true"])
    expect_error(flb, ERR_STATE, h.world_cloud_points)                           # no world cloud after a failure
    expect_error(flb, ERR_STATE, h.effect_cloud_download_points)                 # no effect cloud
    L = h.L
    n = C.c_int()
    assert L.flb_world_cloud_points(h.h, None, -1, C.byref(n)) == ERR_INVALID
    assert L.flb_lidar_download_points(h.h, None, 5, C.byref(n)) == ERR_INVALID
    assert L.flb_effect_cloud_download_points(h.h, None, -1, C.byref(n)) == ERR_INVALID
    expect_error(flb, ERR_STATE, h.lidar_save_download, 0, 0)
    h.lidar_save_end()
    h.close()
