"""flb::undistort_pcl_on_device + flb::downsample_scan, the C++ adapters of flb_imu_undistort with out_xyz = NULL and
flb_scan_from_undistorted (tests/adapters/test_adapter_scan_filter.cpp, mock sensor_msgs::Imu / PCL / StatesGroup
types).  CPU tier: the program compiles and links against the library.  GPU tier: feats_down_size, the scan order, the
propagated state and the carry equal those of the host chain (flb::undistort_pcl -> flb_voxel_grid -> flb::upload_scan),
byte for byte."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_scan_filter.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_scan_filter") / "test_adapter_scan_filter")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


def _read_chain(raw, off):
    n = int(np.frombuffer(raw, np.int32, 1, off)[0])
    off += 4
    order = np.frombuffer(raw, np.int32, n, off)
    off += 4 * n
    rest = raw[off:off + 8 * (15 + 7)]
    return (n, order.tobytes(), rest), off + 8 * (15 + 7)


@pytest.mark.gpu
@pytest.mark.parametrize("leaf", [0.15, 0.5])
def test_adapter_scan_equals_host_chain(flb, frames, exe, tmp_path, leaf):
    f = flb.synth.make_imu_frame(seed=33, n_points=0)
    body = frames("C2")["scan_body"]
    off = np.sort(np.random.default_rng(33).uniform(0.0, 100.0, len(body)))
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([len(f["v_imu"]), len(body)], np.int32).tobytes())
        fh.write(np.ascontiguousarray(f["v_imu"], np.float64).tobytes())
        fh.write(np.array([f["pcl_beg_time"], f["pcl_end_time"], f["last_lidar_end_time"]], np.float64).tobytes())
        fh.write(np.concatenate([f["R"].ravel(), f["p"], f["vel"], f["bg"], f["ba"], f["grav"], f["cov"].ravel()]).astype(np.float64).tobytes())
        fh.write(np.concatenate([f["acc_s_last"], f["angvel_last"]]).astype(np.float64).tobytes())
        fh.write(np.concatenate([f["cov_gyr"], f["cov_acc"], f["cov_bias_gyr"], f["cov_bias_acc"], [f["G_m_s2"], f["mean_acc_norm"]],
                                 np.asarray(f["R_LI"]).ravel(), f["t_LI"]]).astype(np.float64).tobytes())
        fh.write(np.concatenate([body, off[:, None]], 1).astype(np.float32).tobytes())
        fh.write(np.array([leaf], np.float64).tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    raw = open(out, "rb").read()
    dev, o = _read_chain(raw, 0)
    host, o = _read_chain(raw, o)
    assert o == len(raw)
    assert dev == host and dev[0] > 1000
