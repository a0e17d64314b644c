"""flb::upload_camera_frame, the C++ adapter of flb_image_upload_bgr (tests/adapters/test_adapter_image.cpp, a mock
cv::Mat).  CPU tier: the program compiles and links against the library.  GPU tier: the image set it leaves equals
cv2's outputs recorded in tests/golden/image_golden.npz, at 1x and 2x, with strided rows, for both gray rules."""
import os
import subprocess

import numpy as np
import pytest

from test_image_prep import GOLDEN, cv3_rule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_image.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_image") / "test_adapter_image")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("rule", [0, 1])
@pytest.mark.parametrize("name", ["noise_1x_strided", "texture_2x_strided", "odd_2x_strided"])
def test_adapter_image_equals_golden(exe, tmp_path, name, rule):
    g = np.load(GOLDEN)
    w, h, W, H = (int(v) for v in g[f"{name}__size"])
    rows = g[f"{name}__rows"]
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as fh:
        fh.write(np.array([W, H, w, h, rows.shape[1], rule], np.int32).tobytes())
        fh.write(np.ascontiguousarray(rows).tobytes())
    r = subprocess.run([exe, str(inp), str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(out, np.uint8)
    assert raw.size == 4 * W * H
    bgr = g[f"{name}__bgr"]
    assert np.array_equal(raw[W * H:].reshape(H, W, 3), bgr)
    assert np.array_equal(raw[:W * H].reshape(H, W), g[f"{name}__gray"] if rule == 0 else cv3_rule(bgr))
