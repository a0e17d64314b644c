"""flb::publish_frame_world_rgb and flb::save_rgb_map, the C++ adapters of flb_rgb_cloud and flb_rgb_save_*
(tests/adapters/test_adapter_rgb_cloud.cpp, a mock 32-byte pcl::PointXYZRGB and a mock PCL cloud).  CPU tier: the
program compiles and links against the library.  GPU tier: its frame cloud equals the ABI's records byte for byte, its
map is two such frames, and a save that dropped a frame makes save_rgb_map throw."""
import os
import subprocess

import numpy as np
import pytest

from test_gpu_world_cloud import bgr_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_rgb_cloud.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_rgb_cloud") / "test_adapter_rgb_cloud")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Werror", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_adapter_builds(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_adapter_clouds_equal_abi(flb, exe, tmp_path):
    seq = flb.synth.make_visual_sequence("T0", 1)
    fr, cam = seq["frames"][0], seq["cam"]
    bgr = bgr_of(fr["image"], 0)
    body = np.ascontiguousarray(fr["scan_body"], np.float32)
    inp, out = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    with open(inp, "wb") as fh:
        fh.write(np.array([cam["width"], cam["height"]], np.int32).tobytes())
        fh.write(np.array([cam["fx"], cam["fy"], cam["cx"], cam["cy"], *cam["d"]], np.float64).tobytes())
        fh.write(bgr.tobytes() + np.array([len(body)], np.int32).tobytes() + body.tobytes())
        fh.write(np.concatenate([np.ravel(fr["R"]), fr["p"], np.ravel(seq["R_LI"]), seq["t_LI"], np.ravel(fr["Rcw"]), fr["Pcw"]]).astype(np.float64).tobytes())
    subprocess.check_call([exe, inp, out])
    raw = open(out, "rb").read()
    clouds, off = [], 0
    for _ in range(2):
        n = int(np.frombuffer(raw, np.int32, 1, off)[0])
        off += 4
        clouds.append(np.frombuffer(raw, flb.capi.RGB_POINT, n, off))
        off += 32 * n
    threw = int(np.frombuffer(raw, np.int32, 1, off)[0])
    h = flb.Handle(device=0)
    h.camera_set(cam)
    h.image_upload_bgr(bgr)
    h.scan_upload(body)
    h.world_cloud(flb.capi.lio_params(dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"]), 3), flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
    h.rgb_cloud(fr["Rcw"], fr["Pcw"])
    ref = h.rgb_cloud_download()
    h.close()
    assert len(ref) > 100
    assert clouds[0].tobytes() == ref.tobytes()
    assert clouds[1].tobytes() == ref.tobytes() * 2
    assert threw == 1
