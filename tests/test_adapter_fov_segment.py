"""flb::lasermap_fov_segment, the C++ adapter of flb_map_fov_segment (tests/adapters/test_adapter_fov_segment.cpp, mock
Eigen-shaped types).  CPU tier: both overloads compile and link against the library, and a nullptr counter selects the
plain overload.  GPU tier: the 18-DoF overload (position from the device state) and the IKFoM overload (pos_lid) both
give the deleted counts and the map of flb_map_fov_segment at the same positions, byte for byte."""
import os
import subprocess

import numpy as np
import pytest

import fov_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_fov_segment.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_fov_segment") / "test_adapter_fov_segment")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_adapter_matches_c_api(flb, frames, exe, tmp_path):
    f = frames("C2")
    room = np.ascontiguousarray(f["map_xyz"][::8], np.float32)
    m = np.concatenate([room, room + np.float32(-150.0)]).astype(np.float32)   # a copy the third frame's boxes cut
    cube_len = fov_oracle.SHIPPED[0]
    traj = np.asarray(f["p_true"], np.float64) + np.random.default_rng(6).uniform(-2.0, 2.0, (8, 3))
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as fh:
        fh.write(np.array([len(m), len(traj)], np.int32).tobytes() + m.tobytes())
        fh.write(np.array([cube_len], np.float64).tobytes() + traj.tobytes())
    subprocess.check_call([exe, inp, out])
    raw = open(out, "rb").read()
    K = len(traj)
    cnt_a = np.frombuffer(raw, np.int32, K, 0)
    cnt_b = np.frombuffer(raw, np.int32, K, 4 * K)
    off, maps = 8 * K, []
    for _ in range(2):
        n = int(np.frombuffer(raw, np.int32, 1, off)[0])
        maps.append(np.frombuffer(raw, np.float32, 3 * n, off + 4).reshape(n, 3))
        off += 4 + 12 * n
    h = flb.Handle(device=0, cell_size=0.6)
    h.map_upload(m)
    want = [h.map_fov_segment(*fov_oracle.SHIPPED, pos=p)[2] for p in traj]
    ref = h.map_download()
    h.close()
    assert list(cnt_a) == want and list(cnt_b) == want
    assert want[1] > 0 and want[2] > 0                    # the start cube, then the copy 150 m back
    assert maps[0].tobytes() == ref.tobytes() and maps[1].tobytes() == ref.tobytes()
