"""flb::preprocess_features, the C++ adapter of flb_lidar_upload_features and flb_lidar_upload_velodyne_features
(tests/adapters/test_adapter_features.cpp: a mock livox_ros_driver::CustomMsg, and a mock sensor_msgs::PointCloud2 with
its fields looked up by name and their datatypes checked).  CPU tier: the program compiles and links against the library.
GPU tier: the cloud equals the checker's (with disB = 0, the adapter's value) for every kind, and a wrong datatype, a
missing field and a kind without a feature branch are refused."""
import os
import subprocess

import numpy as np
import pytest

import feat_oracle
from feat_util import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_features.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_features") / "test_adapter_features")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,kw", [("livox", dict(seed=31)), ("ouster", dict(seed=31)),
                                     ("velodyne", dict(seed=31, timed=True, nan_returns=False)),
                                     ("velodyne", dict(seed=32, timed=False, nan_returns=False))],
                         ids=["livox", "ouster", "velodyne-timed", "velodyne-yaw"])
def test_adapter_equals_checker(exe, tmp_path, kind, kw):
    rec, fmt = scene(kind, point_filter_num=2, **kw)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    n = len(rec) // fmt["point_step"]
    off_time = fmt["off_time"] if (kind != "velodyne" or kw["timed"]) else -1
    with open(inp, "wb") as fh:
        fh.write(np.array([fmt["kind"], n, fmt["point_step"], fmt["off_x"], fmt["off_y"], fmt["off_z"], off_time, fmt["off_line"],
                           fmt["n_scans"], fmt["point_filter_num"]], np.int32).tobytes())
        fh.write(np.array([fmt["blind"]], np.float64).tobytes())
        fh.write(rec)
    subprocess.check_call([str(exe), str(inp), str(out)])
    blob = open(out, "rb").read()
    n_points, yaw_times, refused = np.frombuffer(blob[:12], np.int32)
    last = np.frombuffer(blob[12:16], np.float32)[0]
    cloud = np.frombuffer(blob[16:], np.float32).reshape(-1, 4)
    ref, _, _, ref_yaw = feat_oracle.process(dict(fmt, off_time=off_time), rec, 0.0)
    assert refused == (0 if kind == "livox" else 3)
    assert n_points == len(ref) > 0 and bool(yaw_times) == ref_yaw
    assert cloud.tobytes() == ref.tobytes() and last.tobytes() == ref[-1, 3].tobytes()
