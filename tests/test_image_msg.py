"""CPU tier: the per-pixel rules of flb_image_upload_msg (enc_byte, bayer_bgr, linear_tap, linear_v, mean2x2 and
bgr_to_gray in flb_device.cuh, compiled for the host from tests/hostemu/image_msg.cpp and composed per frame as
k_bayer_bgr, k_image_prep and k_image_resize_linear compose them).

- Every case of tests/golden/image_msg_golden.npz (cv2's cvtColor -> resize -> cvtColor, recorded with the OpenCV
  version named in the file) equals the host emulation byte for byte, with no cv2 needed; FLB_GRAY_CV3 equals its
  integer formula on the colour frame wherever the rule takes it.
- A numpy statement of the demosaic and of the linear resize's fixed-point weights and rounding is a third voice: it
  equals the emulation, and cv2 where cv2 is installed, at sizes up to 2449 x 2049."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from test_image_prep import cv3_rule

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "image_msg_golden.npz")
CV4, CV3 = 0, 1
BAYER = {"bayer_rggb8": 5, "bayer_bggr8": 6, "bayer_gbrg8": 7, "bayer_grbg8": 8}
TILE = {5: "RGGB", 6: "BGGR", 7: "GBRG", 8: "GRBG"}        # the 2x2 tile from its top-left site


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/image_msg.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("image_msg") / "libimage_msg.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "image_msg.cpp")])
    L = C.CDLL(so)
    L.emu_bayer_bgr.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.emu_linear_taps.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_image_msg.argtypes = [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p] * 2
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def golden_names():
    return [str(n) for n in np.load(GOLDEN)["names"]]


def golden(name):
    g = np.load(GOLDEN)
    w, h, W, H, enc, bpp = (int(v) for v in g[f"{name}__size"])
    return g[f"{name}__rows"], (w, h, W, H, enc, bpp), g[f"{name}__bgr"], g[f"{name}__gray"]


def is_linear(w, h, W, H):
    return (w, h) not in ((W, H), (2 * W, 2 * H))


def emu_msg(L, rows, w, h, W, H, enc, rule):
    rows = np.ascontiguousarray(rows, np.uint8)
    bgr = np.zeros((H, W, 3), np.uint8)
    gray = np.zeros((H, W), np.uint8)
    L.emu_image_msg(_p(rows), w, h, rows.shape[1], enc, W, H, rule, _p(bgr), _p(gray))
    return bgr, gray


# ------------------------------------------------------------------------------------------------ numpy statements
def np_demosaic(m, enc):
    """OpenCV's bilinear demosaic as cv_bridge applies it: interior rule, then the outer rows and columns copy rows
    1 and h - 2, columns 1 and w - 2."""
    m = m.astype(np.int32)
    h, w = m.shape
    tile = TILE[enc]
    colour = np.empty((h, w), np.int8)
    for k, c in enumerate(tile):
        colour[k // 2::2, k % 2::2] = "BGR".index(c)
    c, n, s, we, e = m[1:-1, 1:-1], m[:-2, 1:-1], m[2:, 1:-1], m[1:-1, :-2], m[1:-1, 2:]
    cross = (n + s + we + e + 2) >> 2
    diag = (m[:-2, :-2] + m[:-2, 2:] + m[2:, :-2] + m[2:, 2:] + 2) >> 2
    hp, vp = (we + e + 1) >> 1, (n + s + 1) >> 1
    site, left = colour[1:-1, 1:-1], colour[1:-1, :-2]
    g = np.where(site == 1, c, cross)
    b = np.where(site == 0, c, np.where(site == 2, diag, np.where(left == 0, hp, vp)))
    r = np.where(site == 2, c, np.where(site == 0, diag, np.where(left == 2, hp, vp)))
    inner = np.stack([b, g, r], -1)
    yy, xx = np.clip(np.arange(h), 1, h - 2) - 1, np.clip(np.arange(w), 1, w - 2) - 1
    return inner[yy][:, xx].astype(np.uint8)


def np_taps(n, s):
    """OpenCV's INTER_LINEAR taps for output index d < n from a source axis of s: the position in double, rounded to
    float, its fraction in float, the 11-bit weights each rounded half to even on its own, the edges clamped."""
    f32 = np.float32
    o, a0, a1 = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64)
    scale = 1.0 / (n / s)
    for d in range(n):
        f = f32((d + 0.5) * scale - 0.5)
        i = int(math.floor(f))
        f = f32(f - f32(i))
        if i < 0:
            f, i = f32(0), 0
        if i >= s - 1:
            f, i = f32(0), s - 1
        o[d], a0[d], a1[d] = i, int(np.rint(f32(f32(1) - f) * f32(2048))), int(np.rint(f * f32(2048)))
    return o, a0, a1


def np_resize_linear(img, W, H):
    h, w = img.shape[:2]
    xo, xa0, xa1 = np_taps(W, w)
    yo, ya0, ya1 = np_taps(H, h)
    s = img.astype(np.int64)
    hs = s[:, xo] * xa0[None, :, None] + s[:, np.minimum(xo + 1, w - 1)] * xa1[None, :, None]
    s0, s1 = hs[yo], hs[np.minimum(yo + 1, h - 1)]
    b0, b1 = ya0[:, None, None], ya1[:, None, None]
    return ((((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", golden_names())
def test_golden(emu, name):
    rows, (w, h, W, H, enc, bpp), bgr, gray = golden(name)
    got_bgr, got_gray = emu_msg(emu, rows, w, h, W, H, enc, CV4)
    assert np.array_equal(got_bgr, bgr)
    assert np.array_equal(got_gray, gray)
    if not is_linear(w, h, W, H):
        assert np.array_equal(emu_msg(emu, rows, w, h, W, H, enc, CV3)[1], cv3_rule(bgr))


def test_golden_covers_the_issue_sizes():
    g = np.load(GOLDEN)
    sizes = [tuple(int(v) for v in g[f"{n}__size"]) for n in golden_names()]
    assert {s[4] for s in sizes} == set(range(9))
    for enc in range(9):
        mine = [s for s in sizes if s[4] == enc]
        kinds = {(w == W, w == 2 * W, w == 2 * W + 1, h == H, h == 2 * H, h == 2 * H + 1) for w, h, W, H, _, _ in mine}
        assert (True, False, False, True, False, False) in kinds                      # camera size
        assert (False, True, False, False, True, False) in kinds                      # exactly twice
        assert (False, False, True, False, True, False) in kinds                      # odd width
        assert (False, True, False, False, False, True) in kinds                      # odd height
        assert (False, False, True, False, False, True) in kinds                      # both odd
        assert any(W % 4 for _, _, W, _, _, _ in mine) and any(w >= 1283 for w, *_ in mine)
        assert min(w * h for w, h, *_ in mine) == 16 * 16
        assert any(g[f"{n}__rows"].shape[1] > s[0] * s[5] for n, s in zip(golden_names(), sizes) if s[4] == enc)
    assert str(g["cv2_version"]).startswith("4.")
    assert os.path.getsize(GOLDEN) < 1 << 20


@pytest.mark.parametrize("enc", sorted(BAYER.values()))
@pytest.mark.parametrize("size", [(16, 16), (33, 17), (64, 96), (513, 129)])
def test_demosaic_statement(emu, enc, size):
    w, h = size
    m = np.random.default_rng(w * h + enc).integers(0, 256, (h, w), dtype=np.uint8)
    ref = np_demosaic(m, enc)
    got = np.zeros((h, w, 3), np.uint8)
    emu.emu_bayer_bgr(_p(m), w, h, enc, _p(got))
    assert np.array_equal(got, ref)
    cv2 = pytest.importorskip("cv2")
    code = {5: cv2.COLOR_BayerBG2BGR, 6: cv2.COLOR_BayerRG2BGR, 7: cv2.COLOR_BayerGR2BGR, 8: cv2.COLOR_BayerGB2BGR}[enc]
    assert np.array_equal(cv2.cvtColor(m, code), ref)


@pytest.mark.parametrize("n,s", [(320, 641), (256, 513), (1224, 2449), (1024, 2049), (16, 33), (642, 1285), (32, 64), (8, 16)])
def test_linear_taps_statement(emu, n, s):
    o, a0, a1 = (np.zeros(n, np.int32) for _ in range(3))
    emu.emu_linear_taps(n, s, _p(o), _p(a0), _p(a1))
    ro, ra0, ra1 = np_taps(n, s)
    assert np.array_equal(o, ro) and np.array_equal(a0, ra0) and np.array_equal(a1, ra1)


@pytest.mark.parametrize("size", [(641, 512), (640, 513), (97, 65), (1283, 9), (2449, 2049)])
def test_linear_resize_statement(emu, size):
    """The numpy statement, the host emulation and (when installed) cv2 agree on odd-sided BGR frames."""
    w, h = size
    W, H = w // 2, h // 2
    img = np.random.default_rng(w + h).integers(0, 256, (h, w, 3), dtype=np.uint8)
    ref = np_resize_linear(img, W, H)
    got, _ = emu_msg(emu, img.reshape(h, 3 * w), w, h, W, H, 0, CV4)
    assert np.array_equal(got, ref)
    cv2 = pytest.importorskip("cv2")
    assert np.array_equal(cv2.resize(img, (W, H), 0, 0, cv2.INTER_LINEAR), ref)
