"""flb::preprocess (Livox CustomMsg; PointCloud2 with a FLOAT32, a UINT16 and no intensity field), flb::publish_frame_world
and flb::save_intensity_map, the C++ adapters of the intensity calls (tests/adapters/test_adapter_intensity.cpp, mock
messages and a mock 48-byte pcl::PointXYZINormal cloud).  CPU tier: the program compiles and links against the library.
GPU tier: its clouds equal the checker's pl_surf and the ABI's records byte for byte; a FLOAT32 intensity is kept, any
other reads 0 as in PCL; the map is the two published frames; a save that dropped a frame makes save_intensity_map throw."""
import os
import subprocess

import numpy as np
import pytest

from imu_util import product_inputs
from lidar_util import c_format
from test_intensity_cloud import XYZINORMAL_POINT, oracle_process, with_intensity

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_intensity.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_intensity") / "test_adapter_intensity")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_adapter_clouds_equal_abi(flb, frames, exe, tmp_path):
    lrec, lfmt = with_intensity(flb, "livox", 1, 5000, 1, None)
    orec, ofmt = with_intensity(flb, "ouster", 2, 8192, 1, None, nan=True)
    ofmt = dict(ofmt, point_filter_num=1, blind=0.8)
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    fi = flb.synth.make_imu_frame(seed=6, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    v_imu = np.ascontiguousarray(fi["v_imu"], np.float64)
    pose = np.concatenate([np.ravel(f["R_true"]), f["p_true"]]).astype(np.float64)
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as fh:
        fh.write(np.array([len(lrec) // 20], np.int32).tobytes() + lrec)
        fh.write(np.array([len(orec) // 48], np.int32).tobytes() + orec)
        fh.write(bytes(P) + bytes(Cc) + np.array([len(v_imu)], np.int32).tobytes() + v_imu.tobytes())
        fh.write(np.array([fi["pcl_beg_time"], fi["pcl_end_time"]], np.float64).tobytes() + bytes(x) + bytes(prm) + pose.tobytes())
    subprocess.check_call([exe, inp, out])
    raw = open(out, "rb").read()
    clouds, off = [], 0
    for _ in range(6):
        n = int(np.frombuffer(raw, np.int32, 1, off)[0])
        off += 4
        clouds.append(np.frombuffer(raw, XYZINORMAL_POINT, n, off))
        off += 48 * n
    threw = int(np.frombuffer(raw, np.int32, 1, off)[0])
    A, B, Cu, D, E, F = clouds
    lfmt = dict(lfmt, n_scans=6, blind=0.5, point_filter_num=1)
    assert A.tobytes() == oracle_process(lfmt, lrec, 16).tobytes() and len(A) > 100
    assert B.tobytes() == oracle_process(ofmt, orec, 16).tobytes() and len(B) > 100
    zero = oracle_process(ofmt, orec, -1).tobytes()
    assert Cu.tobytes() == zero and D.tobytes() == zero
    # the ABI on a handle of its own: the same chain, then flb_world_cloud_points
    h = flb.Handle(device=0)
    h.lidar_upload_intensity(c_format(flb, ofmt), np.frombuffer(orec, np.uint8), 16)
    h.state_upload(x, x.copy())
    P2, Cc2, _ = product_inputs(flb, fi)                   # the carry as it was before the program's call
    h.imu_undistort_lidar(P2, Cc2, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True, download=False)
    h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
    ref = h.world_cloud_points()
    h.close()
    assert len(ref) == len(B) and E.tobytes() == ref.tobytes()
    assert F.tobytes() == ref.tobytes() + ref.tobytes()
    assert threw == 1
