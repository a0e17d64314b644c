"""CPU tier: the drawing rules of flb_keypatch_image (LidarSelector::display_keypatch without its text,
src/lidar_selection.cpp:985-1005): keypatch_round, keypatch_in_disk and keypatch_colour in flb_device.cuh, compiled for
the host from tests/hostemu/keypatch.cpp and composed per frame as k_kp_stamp and k_kp_compose compose them.

Every case of tests/golden/keypatch_golden.npz (cv2.circle(img, c, 6, colour, FILLED, LINE_8) in list order, recorded
with the OpenCV version named in the file) is reproduced byte for byte by three restatements: the host emulation, a
numpy statement of the rules, and cv2 itself where it is installed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "keypatch_golden.npz")
LIMIT = 2.0 ** 30
HALF_WIDTH = (6, 5, 5, 5, 4, 3, 0)          # the disk's half-width by |dy|: rows 1 7 9 11 11 11 13 11 11 11 9 7 1 wide
GREEN, BLUE = (0, 255, 0), (255, 0, 0)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/keypatch.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("keypatch") / "libkeypatch.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "keypatch.cpp")])
    L = C.CDLL(so)
    L.emu_keypatch.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.emu_keypatch_round.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def golden_names():
    return [str(n) for n in np.load(GOLDEN)["names"]]


def golden(name):
    """(input frame, centres (n, 2) float32, errors (n,) float32, cv2's drawn frame)."""
    g = np.load(GOLDEN)
    img = g[f"frame{int(g[f'{name}__size'][0])}"]
    return img, g[f"{name}__cxy"], g[f"{name}__err"], img ^ g[f"{name}__diff"]


# ------------------------------------------------------------------------------------------------ restatements
def np_keypatch(img, cxy, err):
    """display_keypatch's circles in numpy: each centre rounded to float then to int half to even (cvRound of
    cv::Point2f), skipped when non-finite or beyond +-2^30; the fixed 113-pixel disk clipped to the frame; the highest
    index wins where disks overlap; green where errors[i] < 8000, blue otherwise (NaN included)."""
    H, W = img.shape[:2]
    owner = np.full((H, W), -1, np.int64)
    c = np.asarray(cxy, np.float64).astype(np.float32)
    for i, (x, y) in enumerate(c):
        if not (np.isfinite(x) and np.isfinite(y) and abs(x) <= LIMIT and abs(y) <= LIMIT):
            continue
        cx, cy = int(np.rint(x)), int(np.rint(y))
        for dy in range(-6, 7):
            hw, yy = HALF_WIDTH[abs(dy)], cy + dy
            x0, x1 = max(cx - hw, 0), min(cx + hw, W - 1)
            if 0 <= yy < H and x0 <= x1:
                owner[yy, x0:x1 + 1] = i
    out = img.copy()
    m = owner >= 0
    green = np.asarray(err, np.float32)[owner[m]] < np.float32(8000)
    out[m] = np.where(green[:, None], np.array(GREEN, np.uint8), np.array(BLUE, np.uint8))
    return out


def emu_keypatch(L, img, cxy, err):
    img = np.ascontiguousarray(img, np.uint8)
    cxy = np.ascontiguousarray(cxy, np.float32)
    err = np.ascontiguousarray(err, np.float32)
    out = np.zeros_like(img)
    L.emu_keypatch(_p(img), img.shape[1], img.shape[0], _p(cxy), _p(err), len(err), _p(out))
    return out


def cv2_keypatch(cv2, img, cxy, err):
    out = img.copy()
    for (x, y), e in zip(cxy, err):
        if np.isfinite(x) and np.isfinite(y) and abs(x) <= LIMIT and abs(y) <= LIMIT:
            cv2.circle(out, (int(np.rint(x)), int(np.rint(y))), 6, GREEN if e < np.float32(8000) else BLUE, -1, 8)
    return out


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("name", golden_names())
def test_golden(emu, name):
    img, cxy, err, want = golden(name)
    assert np.array_equal(emu_keypatch(emu, img, cxy, err), want)
    assert np.array_equal(np_keypatch(img, cxy, err), want)


def test_golden_cv2():
    cv2 = pytest.importorskip("cv2")
    for name in golden_names():
        img, cxy, err, want = golden(name)
        assert np.array_equal(cv2_keypatch(cv2, img, cxy, err), want), name


def test_golden_covers_the_rules():
    """The file pins what it claims: clipped disks on every side, ties, each colour rule and dropped centres."""
    drawn, blues, greens, dropped = 0, 0, 0, 0
    for name in golden_names():
        img, cxy, err, want = golden(name)
        d = (img != want).any(2)
        drawn += int(d.sum())
        greens += int((want[d] == GREEN).all(1).sum())
        blues += int((want[d] == BLUE).all(1).sum())
        dropped += int((~np.isfinite(cxy).all(1) | (np.abs(cxy) > LIMIT).any(1)).sum())
    assert greens > 1000 and blues > 1000 and dropped >= 3 * 6
    img, cxy, err, want = golden("s1_tie+3")
    assert (cxy % 1 == 0.5).all()
    assert set(np.unique(np.where(np.isnan(err), -1, err))) == {-1, np.float32(7999.999), 8000, np.float32(8000.0005)}


def test_single_disk_shape(emu):
    img = np.zeros((31, 33, 3), np.uint8)
    out = emu_keypatch(emu, img, np.array([[16, 15]], np.float32), np.array([0], np.float32))
    rows = (out[..., 1] == 255).sum(1)
    assert rows[rows > 0].tolist() == [1, 7, 9, 11, 11, 11, 13, 11, 11, 11, 9, 7, 1]


def test_round_half_even_and_limits(emu):
    v = np.array([0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 0.49999997, 2.0 ** 30, -2.0 ** 30, 2.0 ** 30 + 64, 3e9, np.inf, -np.inf, np.nan,
                  # doubles that round to a float tie, and one that lands just below it
                  2.5 + 2.0 ** -30, 1e300], np.float64)
    r, ok = np.zeros(len(v), np.int32), np.zeros(len(v), np.int32)
    emu.emu_keypatch_round(_p(v), len(v), _p(r), _p(ok))
    want_ok = [1] * 9 + [1, 0, 0, 0, 0, 1, 0]
    assert ok.tolist() == want_ok
    assert r[:9].tolist() == [0, 2, 2, 0, -2, -2, 0, 2 ** 30, -2 ** 30]
    assert r[9] == 2 ** 30 and r[14] == 2        # 2^30 + 64 is 2^30 in float; 2.5 + 2^-30 is the float 2.5
