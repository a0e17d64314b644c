"""flb::publish_effect_world, the C++ adapter of flb_effect_cloud (tests/adapters/test_adapter_effect.cpp, mock
Eigen-shaped types and a mock PCL cloud).  CPU tier: both overloads compile and link against the library.  GPU tier:
after flb::lio_update, the 18-DoF overload (pose from the device state) and the IKFoM overload (rot.toRotationMatrix(),
pos, offset_*_L_I) both fill the cloud with the oracle's last-pass laserCloudOri transformed at that pose, byte for
byte."""
import os
import subprocess

import numpy as np
import pytest

import effect_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_effect.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_effect") / "test_adapter_effect")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


def _read(path):
    raw = open(path, "rb").read()
    clouds, off = [], 0
    for _ in range(2):
        n = int(np.frombuffer(raw, np.int32, 1, off)[0])
        off += 4
        clouds.append(np.frombuffer(raw, np.float32, 3 * n, off).reshape(n, 3))
        off += 12 * n
    post = np.frombuffer(raw, np.float64, 12, off)
    return clouds, post[:9].reshape(3, 3), post[9:]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["T0", "T1"])
def test_adapter_clouds_equal_oracle(flb, po, frames, exe, tmp_path, name):
    from test_gpu_effect_cloud import oracle_world
    f = frames(name)
    assert f["cfg"].cell_size == 0.6                     # the program's handle config
    R = np.asarray(f["R_prop"], np.float64)
    assert not np.allclose(R, R.T)                        # a transposed pose would show
    p = np.asarray(f["p_prop"], np.float64)
    m = np.ascontiguousarray(f["map_xyz"], np.float32)
    s = np.ascontiguousarray(f["scan_body"], np.float32)
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as fh:
        fh.write(np.array([len(m), len(s)], np.int32).tobytes() + m.tobytes() + s.tobytes())
        fh.write(np.concatenate([R.ravel(), p, np.asarray(f["R_LI"], np.float64).ravel(), np.asarray(f["t_LI"], np.float64)]).tobytes())
    subprocess.check_call([exe, inp, out])
    (a, b), Rpost, ppost = _read(out)
    lio = eo.Lio(m, s)
    x = po.State18.make(R, p, cov=np.eye(18) * 1e-3)
    lio.update(po.lio_params(f, 3), x, x.copy())
    ori = lio.last_ori()
    assert len(a) == len(b) == len(ori) > 100
    assert a.tobytes() == oracle_world(po, f, s[ori], Rpost, ppost).tobytes()
    assert b.tobytes() == oracle_world(po, f, s[ori], R, p).tobytes()
