"""flb::upload_camera_msg and flb::camera_encoding, the C++ adapter of flb_image_upload_msg
(tests/adapters/test_adapter_image_msg.cpp, a mock sensor_msgs::Image).  CPU tier: the program compiles and links
against the library, maps every encoding string to its FLB_ENC_* and throws flb::Error on any other string.  GPU tier:
the image set it leaves equals cv2's outputs recorded in tests/golden/image_msg_golden.npz."""
import os
import subprocess

import numpy as np
import pytest

from test_image_msg import golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_image_msg.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_image_msg") / "test_adapter_image_msg")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_encoding_map_and_refusals(exe):
    r = subprocess.run([exe, "map"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bayer_bggr8__w42_oddwh_strided", "mono8__2x", "rgba8__w42_1x_strided", "rgb8__oddwh"])
def test_adapter_image_msg_equals_golden(exe, tmp_path, name):
    rows, (w, h, W, H, enc, bpp), bgr, gray = golden(name)
    encoding = name.split("__")[0].encode()
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([W, H, w, h, rows.shape[1], len(encoding)], np.int32).tobytes())
        fh.write(encoding)
        fh.write(np.ascontiguousarray(rows).tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(out, np.uint8)
    assert raw.size == 4 * W * H
    assert np.array_equal(raw[W * H:].reshape(H, W, 3), bgr)
    assert np.array_equal(raw[:W * H].reshape(H, W), gray)
