"""flb::preprocess_velodyne, the C++ adapter of flb_lidar_upload_velodyne (tests/adapters/test_adapter_velodyne.cpp: a
mock sensor_msgs::PointCloud2 with its fields looked up by name and their datatypes checked).  CPU tier: the program
compiles and links against the library.  GPU tier: the decoded cloud equals the checker's in every layout."""
import os
import subprocess

import numpy as np
import pytest

import velo_oracle
from velo_util import LAYOUTS, spin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_velodyne.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_velodyne") / "test_adapter_velodyne")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("timed", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_adapter_equals_checker(flb, exe, tmp_path, layout, timed):
    rec, fmt = spin(flb, layout, 9, 2, timed=timed)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    n = len(rec) // fmt["point_step"]
    with open(inp, "wb") as fh:
        fh.write(np.array([n, fmt["point_step"], fmt["off_x"], fmt["off_y"], fmt["off_z"], fmt["off_time"], fmt["off_ring"],
                           fmt["n_scans"], fmt["point_filter_num"]], np.int32).tobytes())
        fh.write(np.array([fmt["blind"]], np.float64).tobytes())
        fh.write(rec)
    subprocess.check_call([exe, str(inp), str(out)])
    blob = open(out, "rb").read()
    n_points, yaw_times, refused = np.frombuffer(blob[:12], np.int32)
    last = np.frombuffer(blob[12:16], np.float32)[0]
    cloud = np.frombuffer(blob[16:], np.float32).reshape(-1, 4)
    ref, ref_yaw = velo_oracle.process(fmt, rec)
    assert refused == 1
    assert n_points == len(ref) and bool(yaw_times) == ref_yaw == (not timed or fmt["off_time"] < 0)
    assert cloud.tobytes() == ref.tobytes() and last.tobytes() == ref[-1, 3].tobytes()
