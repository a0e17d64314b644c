"""flb::display_keypatch, the C++ adapter of flb_keypatch_image (tests/adapters/test_adapter_keypatch.cpp, a mock cv::Mat
and a recording put_text).  CPU tier: the program compiles and links against the library, and a failing call throws
flb::Error without drawing text.  GPU tier: zero patches leave img_cp unchanged with no text; with patches img_cp equals
flb_keypatch_image's frame at the row step the Mat gives, and the rate text is drawn once, as display_keypatch draws it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "adapters", "test_adapter_keypatch.cpp")


@pytest.fixture(scope="module")
def exe(flb, tmp_path_factory):
    flb.capi.build()
    out = str(tmp_path_factory.mktemp("adapter_keypatch") / "test_adapter_keypatch")
    subprocess.check_call(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-o", out, SRC,
                           "-L" + os.path.join(ROOT, "fast-livo_b200"), "-lfastlivo_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "fast-livo_b200")])
    return out


def test_failure_draws_no_text(exe):
    r = subprocess.run([exe, "nohandle"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr


@pytest.mark.gpu
def test_adapter_keypatch_on_device(exe):
    r = subprocess.run([exe, "device"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stderr)
