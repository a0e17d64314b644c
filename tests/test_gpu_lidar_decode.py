"""GPU tier: the driver's LiDAR message on the device.  flb_lidar_upload (Preprocess::process's non-feature branches,
reference src/preprocess.cpp, and the time sort of src/laserMapping.cpp:551) against the checker
(tests/oracle_pre/pre_oracle.cpp) byte for byte, and flb_imu_undistort_lidar (UndistortPcl's window,
src/IMU_Processing.cpp:624-646, then flb_imu_undistort on the device cloud) against flb_imu_undistort of the checker's
windowed 48-byte points on a second handle: everything downstream must be byte-identical."""
import numpy as np
import pytest

import pre_oracle
from imu_util import product_inputs
from lidar_util import CASES, c_format, case_id, message, rounding_message, scan_end_offset

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
SIZES = [0, 1, 2, 255, 256, 257, 24000, 262144]


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value
    assert str(e.value)


def upload_and_check(flb, h, rec, fmt, source="pageable"):
    ref = pre_oracle.process(fmt, rec)
    a = np.frombuffer(rec, np.uint8)
    if source == "pinned":
        a = h.pinned_like(a)
    n, last = h.lidar_upload(c_format(flb, fmt), a, len(rec) // fmt["point_step"])
    assert n == len(ref)
    got = h.lidar_download()
    assert got.tobytes() == ref.tobytes()
    assert np.float32(last).tobytes() == (ref[-1, 3] if n else np.float32(0)).tobytes()
    return ref


# ------------------------------------------------------------------------------------------------ decode + sort
@pytest.mark.parametrize("source", ["pageable", "pinned"])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_upload_equals_oracle(flb, case, source):
    """Every kind, sorted and unsorted times (both sort paths), a 48-byte step with padding (Ouster), every size."""
    h = flb.Handle(device=0)
    for n in SIZES:
        rec, fmt = message(flb, case, n)
        upload_and_check(flb, h, rec, fmt, source)
    h.close()


def test_both_sort_paths_are_taken(flb):
    sorted_in = pre_oracle.process(*reversed(message(flb, CASES[0], 24000)), sort=False)
    unsorted_in = pre_oracle.process(*reversed(message(flb, CASES[2], 24000)), sort=False)
    assert (np.diff(sorted_in[:, 3]) >= 0).all() and (np.diff(sorted_in[:, 3]) == 0).any()
    assert (np.diff(unsorted_in[:, 3]) < 0).any()


# ------------------------------------------------------------------------------------------------ the chain
def livox_from_body(flb, body, seed):
    """A Livox message whose points are `body` (so that the LIO update downstream has a map to match), six lines fired
    together over 100 ms, with a few invalid tags."""
    n = len(body)
    a = np.zeros(n, flb.synth.LIVOX_POINT)
    a["x"], a["y"], a["z"] = body[:, 0], body[:, 1], body[:, 2]
    a["offset_time"] = ((np.arange(n) // 6) * (100e6 / max(n // 6, 1))).astype(np.uint32)
    a["line"] = np.arange(n) % 6
    a["tag"] = np.where(np.random.default_rng(seed).random(n) < 0.05, 0x20, 0x10)
    fmt = dict(kind=1, point_step=20, off_time=0, off_x=4, off_y=8, off_z=12, off_tag=17, off_line=18, n_scans=6,
               point_filter_num=1, blind=0.5)
    return a.tobytes(), fmt


def downstream(flb, h, f, prm, leaf=0.5):
    n = h.scan_from_undistorted(leaf)
    nw = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
    wc = h.world_cloud_download().tobytes()
    x = flb.capi.State18.from_frame(f)
    rep = h.lio_update(prm, x, x.copy())
    return dict(n=n, order=h.debug_scan_order().tobytes(), nw=nw, wc=wc, x=bytes(x), rep=bytes(rep))


@pytest.mark.parametrize("download", [True, False])
@pytest.mark.parametrize("name", ["T0", "C2"])
def test_chain_equals_host_route(flb, frames, name, download):
    f = frames(name)
    prm = flb.capi.lio_params(f, 3)
    rec, fmt = livox_from_body(flb, np.asarray(f["scan_body"], np.float32), 5)
    p48 = pre_oracle.process48(fmt, rec)
    fi = flb.synth.make_imu_frame(seed=31, n_points=0)
    end, off = scan_end_offset(fi["pcl_beg_time"], p48[-1, 9])
    res = []
    for device in (True, False):
        h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
        h.map_upload(f["map_xyz"])
        P, Cc, x = product_inputs(flb, fi)
        h.state_upload(x, x.copy())
        if device:
            upload_and_check(flb, h, rec, fmt)
            taken, out, poses = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, off, True, download=download)
        else:
            win = pre_oracle.window(p48, 0, off)
            taken = len(win)
            out, poses = h.imu_undistort(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, win, offset_index=9, download=download)
        xs, _, _ = h.state_download()
        r = dict(taken=taken, out=None if out is None else out.tobytes(), poses=poses.tobytes(), carry=bytes(Cc), xs=bytes(xs))
        r.update(downstream(flb, h, f, prm))
        res.append(r)
        h.close()
    assert res[0]["taken"] > 100 and res[0]["n"] > 5
    for key in res[1]:
        assert res[0][key] == res[1][key], key


# ------------------------------------------------------------------------------------------------ split scan
def host_undistort(h, P, Cc, v_imu, t_beg, t_end, win):
    if len(win) == 0:
        return h.imu_undistort(P, Cc, v_imu, t_beg, t_end, np.zeros((0, 4), np.float32), offset_index=3)
    return h.imu_undistort(P, Cc, v_imu, t_beg, t_end, win, offset_index=9)


def test_split_scan_cursor_and_rounding(flb):
    """Two camera updates (pcl_offset_time 0.0: only points at time <= 0 are taken, once), then the scan end with a
    pcl_offset_time that rounds below the last time: n_taken and the cursor follow the reference's loop, the last
    point(s) stay out and the cursor's reset drops them."""
    rec, fmt = rounding_message(flb, ("ouster", 1, 3, None), 24000)
    p48 = pre_oracle.process48(fmt, rec)
    beg = 1.7e9
    end, off_end = scan_end_offset(beg, p48[-1, 9])
    assert off_end < float(p48[-1, 9])
    fi = flb.synth.make_imu_frame(seed=33, n_points=0)
    shift = beg - fi["pcl_beg_time"]
    v_imu = fi["v_imu"].copy()
    v_imu[:, 0] += shift
    fi = dict(fi, last_lidar_end_time=fi["last_lidar_end_time"] + shift)
    a, b = flb.Handle(device=0), flb.Handle(device=0)
    Pa, Ca, x = product_inputs(flb, fi)
    Pb, Cb, _ = product_inputs(flb, fi)
    a.state_upload(x, x.copy())
    b.state_upload(x, x.copy())
    upload_and_check(flb, a, rec, fmt)
    index_now, counts = 0, []
    t_prev = beg
    for off, t_end, is_end in ((0.0, beg + 0.005, False), (0.0, beg + 0.010, False), (off_end, end, True)):
        win = pre_oracle.window(p48, index_now, off)
        taken, out, poses = a.imu_undistort_lidar(Pa, Ca, v_imu, t_prev, t_end, off, is_end)
        out_b, poses_b = host_undistort(b, Pb, Cb, v_imu, t_prev, t_end, win)
        assert taken == len(win)
        assert out.tobytes() == out_b.tobytes() and poses.tobytes() == poses_b.tobytes() and bytes(Ca) == bytes(Cb)
        assert bytes(a.state_download()[0]) == bytes(b.state_download()[0])
        counts.append(taken)
        index_now = 0 if is_end else index_now + taken
        t_prev = t_end
    at_zero = int((p48[:, 9] <= 0).sum())
    assert at_zero > 0 and counts[0] == at_zero and counts[1] == 0
    assert 0 < counts[2] < len(p48) - at_zero                # the rounding left the last point(s) out
    # the scan end reset the cursor: the first window again gives the first count
    assert a.imu_undistort_lidar(Pa, Ca, v_imu, beg, beg + 0.005, 0.0, False)[0] == at_zero
    a.close()
    b.close()


def test_upload_during_enqueued_update(flb, frames):
    """A second message is uploaded while the first one's LIO update is enqueued: the update's posterior, the scan and the
    undistorted cloud are those of a run without the second upload."""
    f = frames("C2")
    prm = flb.capi.lio_params(f, 3)
    rec, fmt = livox_from_body(flb, np.asarray(f["scan_body"], np.float32), 6)
    rec2, fmt2 = message(flb, CASES[3], 131072)
    p48 = pre_oracle.process48(fmt, rec)
    fi = flb.synth.make_imu_frame(seed=35, n_points=0)
    end, off = scan_end_offset(fi["pcl_beg_time"], p48[-1, 9])
    res = []
    for second in (True, False):
        h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
        h.map_upload(f["map_xyz"])
        P, Cc, x = product_inputs(flb, fi)
        h.state_upload(x, x.copy())
        h.lidar_upload(c_format(flb, fmt), np.frombuffer(rec, np.uint8))
        h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, off, True, download=False)
        n = h.scan_from_undistorted(0.5)
        x0 = flb.capi.State18.from_frame(f)
        h.state_upload(x0, x0.copy())
        h.lio_update_enqueue(prm)
        if second:
            ref2 = upload_and_check(flb, h, rec2, fmt2)
        nw = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
        xs, rep, _ = h.state_download()
        res.append((n, nw, h.world_cloud_download().tobytes(), bytes(xs), bytes(rep)))
        if second:
            assert h.lidar_download().tobytes() == ref2.tobytes()
        h.close()
    assert res[0] == res[1] and res[0][0] > 5


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_previous_cloud(flb):
    h = flb.Handle(device=0)
    fi = flb.synth.make_imu_frame(seed=36, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    expect_error(flb, ERR_STATE, h.lidar_download)
    expect_error(flb, ERR_STATE, h.imu_undistort_lidar, P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 100.0, True)
    rec, fmt = message(flb, CASES[0], 5000)
    ref = upload_and_check(flb, h, rec, fmt)
    expect_error(flb, ERR_STATE, h.imu_undistort_lidar, P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 100.0, True)   # no state
    h.state_upload(x, x.copy())
    taken, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], float(ref[100, 3]), False)
    assert 0 < taken < len(ref)
    a = np.frombuffer(rec, np.uint8)
    L = flb.capi.lib()

    def bad(**k):
        return c_format(flb, dict(fmt, **k))

    cases = [bad(kind=0), bad(kind=5), bad(point_filter_num=0), bad(n_scans=0), bad(blind=float("nan")), bad(blind=float("inf")),
             bad(off_z=18), bad(off_z=20), bad(off_x=2), bad(off_x=-4), bad(off_line=20), bad(off_time=18), bad(point_step=0)]
    for c in cases:
        expect_error(flb, ERR_INVALID, h.lidar_upload, c, a)
    assert L.flb_lidar_upload(h.h, None, a.ctypes.data, 10, None, None) == ERR_INVALID and L.flb_last_error(h.h)
    assert L.flb_lidar_upload(h.h, flb.capi.C.byref(c_format(flb, fmt)), None, 10, None, None) == ERR_INVALID
    assert L.flb_lidar_upload(h.h, flb.capi.C.byref(c_format(flb, fmt)), a.ctypes.data, -1, None, None) == ERR_INVALID
    rec_x, fmt_x = message(flb, CASES[7], 1000)
    expect_error(flb, ERR_INVALID, h.lidar_upload, c_format(flb, dict(fmt_x, off_time=20)), np.frombuffer(rec_x, np.uint8))   # f64 at 20
    rec_v, fmt_v = flb.synth.make_lidar_message("velodyne_notime", 1, 1000)
    with pytest.raises(flb.capi.FlbError, match="yaw"):
        h.lidar_upload(c_format(flb, fmt_v), np.frombuffer(rec_v, np.uint8))
    rec_o, fmt_o = message(flb, ("ouster", 1, 1, None), 1000)
    for field, value in (("x", np.inf), ("z", np.nan)):      # a NaN range is not < blind^2, so the Ouster rule keeps the point
        o = np.frombuffer(rec_o, flb.synth.OUSTER_POINT).copy()
        o[field][500] = value
        expect_error(flb, ERR_INVALID, h.lidar_upload, c_format(flb, fmt_o), o.view(np.uint8))
    rec_t, fmt_t = flb.synth.make_lidar_message("velodyne", 1, 1000, point_filter_num=1)
    v = np.frombuffer(rec_t, flb.synth.VELODYNE_POINT).copy()
    v["time"][400] = np.inf
    v["x"][400], v["y"][400] = 5.0, 5.0
    expect_error(flb, ERR_INVALID, h.lidar_upload, c_format(flb, fmt_t), v.view(np.uint8))
    # after all of that the first cloud and its cursor are untouched
    assert h.lidar_download().tobytes() == ref.tobytes()
    rest, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True)
    assert rest == len(ref) - taken
    expect_error(flb, ERR_INVALID, h.imu_undistort_lidar, P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], float("nan"), True)
    h.close()


def test_empty_clouds(flb):
    h = flb.Handle(device=0)
    fi = flb.synth.make_imu_frame(seed=37, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    rec, fmt = message(flb, CASES[0], 1000)
    far = c_format(flb, dict(fmt, blind=1e4))               # everything filtered
    assert h.lidar_upload(far, np.frombuffer(rec, np.uint8))[0] == 0
    assert h.lidar_download().shape == (0, 4)
    taken, out, poses = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 100.0, True)
    assert taken == 0 and len(out) == 0 and len(poses) > 0   # propagation only (:776)
    assert h.scan_from_undistorted(0.5) == 0
    assert h.lidar_upload(c_format(flb, fmt), np.zeros(0, np.uint8), 0)[0] == 0
    h.close()
