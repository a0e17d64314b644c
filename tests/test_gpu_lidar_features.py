"""GPU tier: surface features on the device (feature_extract_enable: 1).  flb_lidar_upload_features and
flb_lidar_upload_velodyne_features against the checker (tests/oracle_pre/feat_oracle.cpp) byte for byte over every
scene kind, point_filter_num 1 to 4, disB 0 and non-zero and sizes from an empty message to Ouster-128 and HDL-64
spins; flb_imu_undistort_lidar on the device cloud against flb_imu_undistort of the checker's window; and every error
leaves the previous cloud and cursor in place."""
import numpy as np
import pytest

import feat_oracle
import pre_oracle
from feat_util import DIS_B, FILTERS, SCENES, scene
from imu_util import product_inputs
from lidar_util import c_format, scan_end_offset
from velo_util import c_velo_format

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


def velo_fmt(flb, fmt):
    return c_velo_format(flb, dict(point_step=fmt["point_step"], off_x=fmt["off_x"], off_y=fmt["off_y"], off_z=fmt["off_z"],
                                   off_time=fmt["off_time"], off_ring=fmt["off_line"], n_scans=fmt["n_scans"],
                                   point_filter_num=fmt["point_filter_num"], blind=fmt["blind"]))


def lidar_fmt(flb, fmt):
    return c_format(flb, {k: v for k, v in fmt.items()})


def upload(flb, h, rec, fmt, dis_b=0.0, pinned=False):
    a = np.frombuffer(rec, np.uint8)
    if pinned:
        a = h.pinned_like(a)
    if fmt["kind"] == 2:
        n, last, _ = h.lidar_upload_velodyne_features(velo_fmt(flb, fmt), a, dis_b)
    else:
        n, last = h.lidar_upload_features(lidar_fmt(flb, fmt), a, dis_b)
    return n, last


def upload_and_check(flb, h, rec, fmt, dis_b=0.0, pinned=False):
    ref, _, _, _ = feat_oracle.process(fmt, rec, dis_b)
    assert np.isfinite(ref).all()
    n, last = upload(flb, h, rec, fmt, dis_b, pinned)
    assert n == len(ref)
    assert h.lidar_download().tobytes() == ref.tobytes()
    assert np.float32(last).tobytes() == (ref[-1, 3] if n else np.float32(0)).tobytes()
    return ref


CASES = [(k, kw, pf, db) for k, kw in SCENES for pf in FILTERS for db in DIS_B]


@pytest.mark.parametrize("kind,kw,pf,dis_b", CASES, ids=[f"{k}-{kw['seed']}-{kw.get('timed', '')}-pf{pf}-b{db}" for k, kw, pf, db in CASES])
def test_device_equals_checker(flb, kind, kw, pf, dis_b):
    h = flb.Handle(device=0)
    rec, fmt = scene(kind, point_filter_num=pf, **kw)
    ref, _, _, _ = feat_oracle.process(fmt, rec, dis_b)
    if np.isfinite(ref).all():
        upload_and_check(flb, h, rec, fmt, dis_b, pinned=pf == 2)
    else:       # NaN no-returns that reach pl_surf: refused, as a kept non-finite point is
        with pytest.raises(flb.capi.FlbError, match="not finite") as e:
            upload(flb, h, rec, fmt, dis_b)
        assert e.value.code == ERR_INVALID
    h.close()


@pytest.mark.parametrize("kind,kw", [("ouster", dict(n_scans=128, n_cols=1024)), ("velodyne", dict(n_scans=64, n_cols=1800,
                                      timed=False, nan_returns=False)), ("velodyne", dict(n_scans=64, n_cols=1800, timed=True,
                                      nan_returns=False)), ("livox", dict(n_cols=4000))])
def test_full_size(flb, kind, kw):
    h = flb.Handle(device=0)
    for pf, dis_b in ((1, 0.0), (3, 0.05)):
        rec, fmt = scene(kind, point_filter_num=pf, seed=11, **kw)
        upload_and_check(flb, h, rec, fmt, dis_b)
    h.close()


def test_empty_and_tiny_messages(flb):
    h = flb.Handle(device=0)
    for kind in ("livox", "ouster", "velodyne"):
        rec, fmt = scene(kind, seed=5, nan_returns=False) if kind == "velodyne" else scene(kind, seed=5)
        for n in (0, 1, 2, 7, 40):
            upload_and_check(flb, h, rec[:n * fmt["point_step"]], fmt)
    h.close()


def test_undistort_after_upload(flb):
    """flb_imu_undistort_lidar on the device pl_surf equals flb_imu_undistort on the checker's window of 48-byte points."""
    rec, fmt = scene("ouster", seed=6, point_filter_num=2)
    ref, _, _, _ = feat_oracle.process(fmt, rec, 0.0)
    p48 = np.zeros((len(ref), 12), np.float32)
    p48[:, [0, 1, 2, 9]] = ref
    fi = flb.synth.make_imu_frame(seed=43, n_points=0)
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
    fi = flb.synth.make_imu_frame(seed=44, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    h.state_upload(x, x.copy())
    rec, fmt = scene("livox", seed=7)
    ref = upload_and_check(flb, h, rec, fmt)
    taken, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], float(ref[len(ref) // 3, 3]), False)
    assert 0 < taken < len(ref)
    a = np.frombuffer(rec, np.uint8)

    def expect(fn, *args, match=None):
        with pytest.raises(flb.capi.FlbError, match=match) as e:
            fn(*args)
        assert e.value.code == ERR_INVALID, e.value

    for k in (dict(point_filter_num=0), dict(n_scans=0), dict(n_scans=129), dict(blind=float("nan")), dict(point_step=0),
              dict(off_x=18), dict(off_line=20), dict(kind=4), dict(kind=2), dict(kind=7)):
        expect(h.lidar_upload_features, lidar_fmt(flb, dict(fmt, **k)), a)
    expect(h.lidar_upload_features, lidar_fmt(flb, fmt), a, float("nan"))
    vrec, vfmt = scene("velodyne", seed=8, nan_returns=False)
    expect(h.lidar_upload_velodyne_features, velo_fmt(flb, dict(vfmt, n_scans=129)), np.frombuffer(vrec, np.uint8))
    # a point of pl_surf that is not finite comes back after device work
    v = np.frombuffer(vrec, flb.synth.VELODYNE_POINT).copy()
    v["x"][3000:3040] = np.inf
    assert not np.isfinite(feat_oracle.process(vfmt, v.tobytes())[0]).all()
    expect(h.lidar_upload_velodyne_features, velo_fmt(flb, vfmt), v.view(np.uint8), 0.0, match="not finite")
    # the cloud and its cursor are as they were
    assert h.lidar_download().tobytes() == ref.tobytes()
    rest, _, _ = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True)
    assert rest == len(ref) - taken
    h.close()


def test_golden(flb):
    """The device cloud equals the committed outputs of tests/golden/lidar_features_golden.npz."""
    import json
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lidar_features_golden.npz"))
    h = flb.Handle(device=0)
    names = sorted({k.split("__")[0] for k in z.files})
    assert len(names) == 6
    for name in names:
        fmt = json.loads(bytes(z[name + "__fmt"]).decode())
        dis_b = fmt.pop("dis_b")
        n, _ = upload(flb, h, z[name + "__records"].tobytes(), fmt, dis_b)
        assert h.lidar_download().tobytes() == z[name + "__cloud"].tobytes(), name
    h.close()
