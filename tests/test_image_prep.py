"""CPU tier: the per-pixel math of flb_image_upload_bgr (bgr_to_gray and mean2x2 in flb_device.cuh, compiled for the
host from tests/hostemu/image_prep.cpp and composed per frame as k_image_prep composes it).

- FLB_GRAY_CV4 equals OpenCV's cvtColor(BGR2GRAY) for all 2^24 colours, and the 2x path equals cv2.resize(0.5,
  INTER_LINEAR) on even-sized frames (both need cv2 and are skipped without it).
- FLB_GRAY_CV3 equals its integer formula.  No OpenCV 3 is available to check it against; the formula is OpenCV 3.x's
  fixed-point BGR2GRAY as published in its sources.
- Every case of tests/golden/image_golden.npz (cv2's outputs, recorded with the OpenCV version named in the file)
  equals the host emulation, with no cv2 needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "image_golden.npz")
CV4, CV3 = 0, 1


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/image_prep.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("image_prep") / "libimage_prep.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "image_prep.cpp")])
    L = C.CDLL(so)
    L.emu_bgr_to_gray.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    L.emu_image_prep.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p] * 2
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_gray(L, bgr, rule):
    bgr = np.ascontiguousarray(bgr, np.uint8)
    out = np.zeros(bgr.shape[:-1], np.uint8)
    L.emu_bgr_to_gray(_p(bgr), out.size, rule, _p(out))
    return out


def emu_prep(L, rows, width, height, halve, rule):
    """(colour frame, gray) of a frame held as `rows` (height x stride bytes, pixels first)."""
    rows = np.ascontiguousarray(rows, np.uint8)
    W, H = (width // 2, height // 2) if halve else (width, height)
    bgr = np.zeros((H, W, 3), np.uint8)
    gray = np.zeros((H, W), np.uint8)
    L.emu_image_prep(_p(rows), width, height, rows.shape[1], int(halve), rule, _p(bgr), _p(gray))
    return bgr, gray


def every_colour():
    """All 2^24 BGR colours as a 4096 x 4096 frame."""
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([v & 255, (v >> 8) & 255, v >> 16], -1).astype(np.uint8).reshape(4096, 4096, 3)


def cv3_rule(bgr):
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((1868 * b + 9617 * g + 4899 * r + (1 << 13)) >> 14).astype(np.uint8)


def cv4_rule(bgr):
    b, g, r = (bgr[..., k].astype(np.int64) for k in range(3))
    return ((3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15).astype(np.uint8)


def test_cv4_gray_equals_opencv_for_every_colour(emu):
    cv2 = pytest.importorskip("cv2")
    img = every_colour()
    got = emu_gray(emu, img, CV4)
    assert np.array_equal(got, cv2.cvtColor(img, cv2.COLOR_BGR2GRAY))
    assert np.array_equal(got, cv4_rule(img))


def test_cv3_gray_is_its_integer_formula(emu):
    img = every_colour()
    got = emu_gray(emu, img, CV3)
    assert np.array_equal(got, cv3_rule(img))
    # the two rules are different functions: they disagree by one grey level on some colours, never by more
    d = got.astype(np.int16) - emu_gray(emu, img, CV4)
    assert np.abs(d).max() == 1 and 0 < np.count_nonzero(d) < d.size // 100


@pytest.mark.parametrize("size", [(320, 256), (1280, 1024), (84, 36), (18, 34)])
def test_halving_equals_opencv_resize(emu, size):
    cv2 = pytest.importorskip("cv2")
    w, h = size
    rng = np.random.default_rng(w * h)
    src = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    src[: h // 4] = rng.integers(250, 256, (h // 4, w, 3), dtype=np.uint8)     # near-saturated rows: the rounding at the top
    ref = cv2.resize(src, (int(w * 0.5), int(h * 0.5)), 0, 0, cv2.INTER_LINEAR)
    bgr, gray = emu_prep(emu, src.reshape(h, 3 * w), w, h, True, CV4)
    assert np.array_equal(bgr, ref)
    assert np.array_equal(gray, cv2.cvtColor(ref, cv2.COLOR_BGR2GRAY))


def golden_cases():
    g = np.load(GOLDEN)
    return [str(n) for n in g["names"]]


@pytest.mark.parametrize("rule", [CV4, CV3])
@pytest.mark.parametrize("name", golden_cases())
def test_golden(emu, name, rule):
    g = np.load(GOLDEN)
    w, h, W, H = (int(v) for v in g[f"{name}__size"])
    rows = g[f"{name}__rows"]
    bgr, gray = emu_prep(emu, rows, w, h, (w, h) != (W, H), rule)
    assert np.array_equal(bgr, g[f"{name}__bgr"])
    assert np.array_equal(gray, g[f"{name}__gray"] if rule == CV4 else cv3_rule(g[f"{name}__bgr"]))


def test_golden_file_records_its_opencv():
    g = np.load(GOLDEN)
    assert str(g["cv2_version"]).startswith("4.")
    assert os.path.getsize(GOLDEN) < 1 << 20
