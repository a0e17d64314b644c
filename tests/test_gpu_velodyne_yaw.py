"""GPU tier: Velodyne messages in any layout, with the times derived from the yaw angle on the device.
flb_lidar_upload_velodyne (velodyne_handler's non-feature branch, reference src/preprocess.cpp:376-428, and the stable
time sort of src/laserMapping.cpp:551) against the checker (tests/oracle_pre/velo_oracle.cpp) byte for byte with the
project's defined yaw, against the reference as built with libm's atan2f within DESIGN §2's bound, against
flb_lidar_upload where both take the layout, and flb_imu_undistort_lidar on its cloud against flb_imu_undistort of the
checker's window."""
import numpy as np
import pytest

import pre_oracle
import velo_oracle
from imu_util import product_inputs
from lidar_util import c_format, scan_end_offset
from velo_util import LAYOUTS, assert_time_bound, c_velo_format, lidar_format_of, spin

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


def expect_error(flb, code, fn, *a, match=None, **k):
    with pytest.raises(flb.capi.FlbError, match=match) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def upload_and_check(flb, h, rec, fmt, source="pageable", yaw=True):
    ref, yaw_times = velo_oracle.process(fmt, rec)
    assert yaw_times == yaw
    a = np.frombuffer(rec, np.uint8)
    if source == "pinned":
        a = h.pinned_like(a)
    n, last, got_yaw = h.lidar_upload_velodyne(c_velo_format(flb, fmt), a)
    assert (n, got_yaw) == (len(ref), yaw)
    assert h.lidar_download().tobytes() == ref.tobytes()
    assert np.float32(last).tobytes() == (ref[-1, 3] if n else np.float32(0)).tobytes()
    return ref


@pytest.mark.parametrize("pfn", [1, 2, 3])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("size", ["vlp16", "hdl64"])
def test_device_equals_checker(flb, size, layout, pfn):
    h = flb.Handle(device=0)
    for seed in (1, 2):
        rec, fmt = spin(flb, layout, seed, pfn, size)
        assert not velo_oracle.midpoint_flags(fmt, rec).any()
        upload_and_check(flb, h, rec, fmt, "pinned" if seed == 2 else "pageable")
    h.close()


@pytest.mark.parametrize("size", ["vlp16", "hdl64"])
def test_device_against_atan2f(flb, size):
    """The reference as built here (glibc atan2f): the same kept points and count, each time within the bound."""
    h = flb.Handle(device=0)
    for seed in (3, 4):
        rec, fmt = spin(flb, "xyzir32", seed, 1, size)
        h.lidar_upload_velodyne(c_velo_format(flb, fmt), np.frombuffer(rec, np.uint8))
        got = h.lidar_download()
        ref, _ = velo_oracle.process(fmt, rec, velo_oracle.YAW_ATAN2F)
        assert len(got) == len(ref)
        ia, ib = np.lexsort((got[:, 2], got[:, 1], got[:, 0])), np.lexsort((ref[:, 2], ref[:, 1], ref[:, 0]))
        assert got[ia, :3].tobytes() == ref[ib, :3].tobytes()
        assert_time_bound(got[ia, 3], ref[ib, 3])
    h.close()


def test_with_times_equals_lidar_upload(flb):
    """With times the route is flb_lidar_upload's, byte for byte, and the packed layout (time at 18) gives the same cloud."""
    a, b = flb.Handle(device=0), flb.Handle(device=0)
    for pfn in (1, 3):
        rec, fmt = spin(flb, "xyzirt", 5, pfn, "hdl64", timed=True)
        ref = upload_and_check(flb, a, rec, fmt, yaw=False)
        n, last = b.lidar_upload(c_format(flb, lidar_format_of(fmt)), np.frombuffer(rec, np.uint8))
        assert n == len(ref) and b.lidar_download().tobytes() == ref.tobytes()
        assert np.float32(last).tobytes() == ref[-1, 3].tobytes()
        assert ref.tobytes() == pre_oracle.process(lidar_format_of(fmt), rec).tobytes()
        rec22, fmt22 = spin(flb, "packed22", 5, pfn, "hdl64", timed=True)
        assert upload_and_check(flb, a, rec22, fmt22, yaw=False).tobytes() == ref.tobytes()
    a.close()
    b.close()


def test_undistort_after_upload(flb):
    """flb_imu_undistort_lidar on the device cloud equals flb_imu_undistort on the checker's window of 48-byte points."""
    rec, fmt = spin(flb, "packed22", 6, 2)
    ref, _ = velo_oracle.process(fmt, rec)
    p48 = np.zeros((len(ref), 12), np.float32)
    p48[:, [0, 1, 2, 9]] = ref
    fi = flb.synth.make_imu_frame(seed=41, n_points=0)
    end, off = scan_end_offset(fi["pcl_beg_time"], ref[-1, 3])
    a, b = flb.Handle(device=0), flb.Handle(device=0)
    Pa, Ca, x = product_inputs(flb, fi)
    Pb, Cb, _ = product_inputs(flb, fi)
    a.state_upload(x, x.copy())
    b.state_upload(x, x.copy())
    upload_and_check(flb, a, rec, fmt)
    mid = float(ref[len(ref) // 2, 3])
    index_now = 0
    t_prev = fi["pcl_beg_time"]
    for o, t_end, is_end in ((mid, t_prev + mid / 1000.0, False), (off, end, True)):
        win = pre_oracle.window(p48, index_now, o)
        taken, out, poses = a.imu_undistort_lidar(Pa, Ca, fi["v_imu"], t_prev, t_end, o, is_end)
        out_b, poses_b = b.imu_undistort(Pb, Cb, fi["v_imu"], t_prev, t_end, win, offset_index=9)
        assert taken == len(win) > 100
        assert out.tobytes() == out_b.tobytes() and poses.tobytes() == poses_b.tobytes() and bytes(Ca) == bytes(Cb)
        index_now += taken
        t_prev = t_end
    assert bytes(a.state_download()[0]) == bytes(b.state_download()[0])
    a.close()
    b.close()


def test_errors_leave_the_previous_cloud(flb):
    h = flb.Handle(device=0)
    fi = flb.synth.make_imu_frame(seed=42, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    rec, fmt = spin(flb, "xyzirt", 7, 1)
    ref = upload_and_check(flb, h, rec, fmt)
    taken, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], float(ref[100, 3]), False)
    assert 0 < taken < len(ref)
    launches = h.launch_count()
    a = np.frombuffer(rec, np.uint8)

    def bad(**k):
        return c_velo_format(flb, dict(fmt, **k))

    for c in (bad(point_filter_num=0), bad(n_scans=0), bad(blind=float("nan")), bad(blind=float("-inf")), bad(point_step=0),
              bad(off_x=21), bad(off_z=-1), bad(off_time=21), bad(off_time=-2), bad(off_ring=23)):
        expect_error(flb, ERR_INVALID, h.lidar_upload_velodyne, c, a)
    assert h.launch_count() == launches                      # refused before any work
    L = flb.capi.lib()
    C = flb.capi.C
    assert L.flb_lidar_upload_velodyne(h.h, None, a.ctypes.data, 10, None, None, None) == ERR_INVALID and L.flb_last_error(h.h)
    assert L.flb_lidar_upload_velodyne(h.h, C.byref(c_velo_format(flb, fmt)), None, 10, None, None, None) == ERR_INVALID
    assert L.flb_lidar_upload_velodyne(h.h, C.byref(c_velo_format(flb, fmt)), a.ctypes.data, -1, None, None, None) == ERR_INVALID
    # a ring >= n_scans on the yaw route: the message names the ring and the record
    dt = flb.synth.VELODYNE_LAYOUTS["xyzirt"][0]
    v = np.frombuffer(rec, dt).copy()
    v["ring"][5000], v["ring"][9000] = 16, 40
    expect_error(flb, ERR_INVALID, h.lidar_upload_velodyne, c_velo_format(flb, fmt), v.view(np.uint8), match="record 5000 has ring 16")
    # the argument errors and the ring error, which comes back after device work, left the cloud and its cursor as they were
    assert h.lidar_download().tobytes() == ref.tobytes()
    rest, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True)
    assert rest == len(ref) - taken
    # ... which the time route never reads
    v["time"][-1] = 1e-3
    assert h.lidar_upload_velodyne(c_velo_format(flb, fmt), v.view(np.uint8))[2] is False
    upload_and_check(flb, h, rec, fmt)
    taken, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], float(ref[100, 3]), False)
    # a kept value that is not finite: an infinite x (record 0 mod point_filter_num, outside blind), and a ring whose
    # first record has no return, which makes every later time of that ring NaN
    v = np.frombuffer(rec, dt).copy()
    k = next(i for i in range(1000, 2000) if np.isfinite(v["x"][i]))
    v["x"][k] = np.inf
    expect_error(flb, ERR_INVALID, h.lidar_upload_velodyne, c_velo_format(flb, fmt), v.view(np.uint8), match="not finite")
    v = np.frombuffer(rec, dt).copy()
    v["x"][0] = v["y"][0] = np.nan
    assert np.isnan(velo_oracle.process(fmt, v.tobytes())[0][:, 3]).any()
    expect_error(flb, ERR_INVALID, h.lidar_upload_velodyne, c_velo_format(flb, fmt), v.view(np.uint8), match="not finite")
    # after all of that the cloud and its cursor are untouched
    assert h.lidar_download().tobytes() == ref.tobytes()
    rest, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True)
    assert rest == len(ref) - taken
    h.close()


def test_empty_and_tiny_messages(flb):
    h = flb.Handle(device=0)
    rec, fmt = spin(flb, "xyzir32", 8, 1)
    assert h.lidar_upload_velodyne(c_velo_format(flb, fmt), np.zeros(0, np.uint8), 0) == (0, np.float32(0), False)
    assert h.lidar_download().shape == (0, 4)
    step = fmt["point_step"]
    for n in (1, 2, 3, 17, 255, 256, 257):
        upload_and_check(flb, h, rec[:n * step], fmt)
    h.close()
