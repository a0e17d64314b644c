"""flb::preprocess and flb::undistort_pcl_from_lidar, the C++ adapters of flb_lidar_upload and flb_imu_undistort_lidar
(tests/adapters/test_adapter_lidar.cpp: mock livox_ros_driver::CustomMsg, sensor_msgs::PointCloud2 with its fields
looked up by name, LidarMeasureGroup).  CPU tier: the program compiles and links against the library.  GPU tier: the
decoded cloud equals the checker's, and a camera update followed by the scan end leaves n_taken, lidar_scan_index_now,
last_update_time and the propagated state as flb_imu_undistort on the checker's windows does."""
import os
import subprocess

import numpy as np
import pytest

import pre_oracle
from imu_util import product_inputs
from lidar_util import message, scan_end_offset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_lidar.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_lidar") / "test_adapter_lidar")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [("livox", 1, 2, None), ("ouster", 1, 3, None), ("xt32", 1, 3, True)], ids=lambda c: c[0])
def test_adapter_equals_oracle_and_host_route(flb, exe, tmp_path, case):
    rec, fmt = message(flb, case, 24000)
    f = flb.synth.make_imu_frame(seed=41, n_points=0)
    beg, img_offset = f["pcl_beg_time"], 0.004
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([len(f["v_imu"]), fmt["kind"], 24000, fmt["point_step"], fmt["off_x"], fmt["off_y"], fmt["off_z"],
                           fmt["off_time"], fmt["n_scans"], fmt["point_filter_num"]], np.int32).tobytes())
        fh.write(np.array([fmt["blind"], beg, img_offset], np.float64).tobytes())
        fh.write(np.ascontiguousarray(f["v_imu"], np.float64).tobytes())
        fh.write(np.concatenate([f["R"].ravel(), f["p"], f["vel"], f["bg"], f["ba"], f["grav"], f["cov"].ravel()]).astype(np.float64).tobytes())
        fh.write(np.concatenate([[f["last_lidar_end_time"]], f["acc_s_last"], f["angvel_last"]]).astype(np.float64).tobytes())
        fh.write(np.concatenate([f["cov_gyr"], f["cov_acc"], f["cov_bias_gyr"], f["cov_bias_acc"], [f["G_m_s2"], f["mean_acc_norm"]],
                                 np.asarray(f["R_LI"]).ravel(), f["t_LI"]]).astype(np.float64).tobytes())
        fh.write(rec)
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    raw = open(out, "rb").read()
    head = np.frombuffer(raw, np.int32, 7)
    last = np.frombuffer(raw, np.float32, 1, 28)[0]
    update_time = np.frombuffer(raw, np.float64, 2, 32)
    state = np.frombuffer(raw, np.float64, 15, 48)
    cloud = np.frombuffer(raw, np.float32, offset=168).reshape(-1, 4)
    p48 = pre_oracle.process48(fmt, rec)
    ref = p48[:, [0, 1, 2, 9]]
    assert head[0] == head[1] == len(ref) and cloud.tobytes() == np.ascontiguousarray(ref).tobytes()
    assert last.tobytes() == ref[-1, 3].tobytes()
    # the reference's bookkeeping on the checker's cloud, and flb_imu_undistort on its windows
    end, off_end = scan_end_offset(beg, ref[-1, 3])
    w0 = pre_oracle.window(p48, 0, 0.0)
    w1 = pre_oracle.window(p48, len(w0), off_end)
    assert head[2:6].tolist() == [len(w0), len(w1), len(w0), 0]
    assert update_time.tolist() == [beg + img_offset, end]
    h = flb.Handle(device=0)
    P, Cc, x = product_inputs(flb, f)
    t_prev = max(beg, 0.0)
    for win, t_end in ((w0, beg + img_offset), (w1, end)):
        h.state_upload(x, x.copy())
        pts, idx = (win, 9) if len(win) else (np.zeros((0, 4), np.float32), 3)
        h.imu_undistort(P, Cc, f["v_imu"], t_prev, t_end, pts, offset_index=idx, download=False)
        x, _, _ = h.state_download()
        t_prev = max(beg, t_end)
    assert head[6] == h.scan_from_undistorted(0.5)
    got = np.concatenate([np.array(x.rot[:]), np.array(x.pos[:]), np.array(x.vel[:])])
    assert got.tobytes() == state.tobytes()
    h.close()
