"""flb::map_incremental, the C++ adapter of flb_map_add_scan (tests/adapters/test_adapter_map_incremental.cpp, mock
Eigen-shaped types).  CPU tier: both overloads compile and link against the library.  GPU tier: the 18-DoF overload (pose
from the device state) and the IKFoM overload (rot.toRotationMatrix(), pos, offset_*_L_I) both give the map
flb_map_add_points gives on the oracle-transformed scan, byte for byte."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_map_incremental.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_map_incremental") / "test_adapter_map_incremental")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


def _read_maps(path):
    raw = open(path, "rb").read()
    maps, off = [], 0
    while off < len(raw):
        m = int(np.frombuffer(raw, np.int32, 1, off)[0])
        off += 4
        maps.append(np.frombuffer(raw, np.float32, 3 * m, off).reshape(m, 3))
        off += 12 * m
    return maps


@pytest.mark.gpu
@pytest.mark.parametrize("name,ds", [("T0", 0.3), ("T1", 0.5)])
def test_adapter_maps_equal_host_path(flb, po, frames, exe, tmp_path, name, ds):
    f = frames(name)
    assert f["cfg"].cell_size == 0.6                     # the program's handle config
    R = np.asarray(f["R_true"], np.float64)
    assert not np.allclose(R, R.T)                        # a transposed pose would show
    p = np.asarray(f["p_true"], np.float64)
    m = np.ascontiguousarray(f["map_xyz"], np.float32)
    s = np.ascontiguousarray(f["scan_body"], np.float32)
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as fh:
        fh.write(np.array([len(m), len(s)], np.int32).tobytes() + m.tobytes() + s.tobytes())
        fh.write(np.concatenate([R.ravel(), p, np.asarray(f["R_LI"], np.float64).ravel(), np.asarray(f["t_LI"], np.float64),
                                 [ds]]).tobytes())
    subprocess.check_call([exe, inp, out])
    a, b = _read_maps(out)
    lio = po.Lio(m[:64], s)
    world = lio.run_pass(po.lio_params(f, 1), R, p, True)["world"]
    h = flb.Handle(device=0, cell_size=0.6)
    h.map_upload(m)
    h.map_add_points(world, ds)
    ref = h.map_download()
    h.close()
    assert a.tobytes() == ref.tobytes() and b.tobytes() == ref.tobytes()
