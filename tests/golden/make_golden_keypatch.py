"""Generate tests/golden/keypatch_golden.npz: LidarSelector::display_keypatch's circles (src/lidar_selection.cpp:985-1005)
drawn by cv2 in list order, cv2.circle(img, c, 6, colour, -1, 8) with colour (0, 255, 0) where errors[i] < 8000 and
(255, 0, 0) otherwise.  Needs cv2.  Run from the repo root:
    python tests/golden/make_golden_keypatch.py

The reference passes cv::Point2f(pc) to cv::circle, which takes a cv::Point: cvRound of each float, half to even on
x86-64.  cv2's Python binding only takes integer centres, so the float cases are rounded here with np.rint on float32
(round half to even) before cv2 draws them; the integer cases are cv2 alone.  A centre with a non-finite coordinate, or
one that rounds beyond +-2^30, is not drawn: that is the library's definition (OpenCV's clipping overflows there).

Frames: seeded random at 640 x 512 (4 levels per channel, so the file stays small), 97 x 65 and 16 x 16.  Cases,
per frame: integer centres from 7 px outside to 7 px inside every border and corner (one case per offset), overlapping
disks of alternating colour, far and out-of-range centres, and the same border cases with float centres on exact .5
ties, whose errors cycle through 7999.999, 8000, 8000.0005 and NaN.  Each case stores its centres (float32), errors
(float32) and the drawn frame XOR the input frame."""
import os

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.join(ROOT, "tests", "golden", "keypatch_golden.npz")
SIZES = [(640, 512), (97, 65), (16, 16)]
LIMIT = 2.0 ** 30
EDGE_ERRORS = np.array([7999.999, 8000.0, 8000.0005, np.nan], np.float32)


def frame(k, W, H):
    rng = np.random.default_rng(100 + k)
    if W * H > 10000:
        return (rng.integers(0, 4, (H, W, 3)) * 85).astype(np.uint8)
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def draw(img, cxy, err):
    out = img.copy()
    for (x, y), e in zip(cxy, err):
        if not (np.isfinite(x) and np.isfinite(y) and abs(x) <= LIMIT and abs(y) <= LIMIT):
            continue
        c = (int(np.rint(x)), int(np.rint(y)))
        cv2.circle(out, c, 6, (0, 255, 0) if e < np.float32(8000) else (255, 0, 0), -1, 8)
    return out


def border_centres(W, H, d):
    """Four edges and four corners, d px inside (d < 0: outside)."""
    return [(d, H // 2), (W - 1 - d, H // 2), (W // 2, d), (W // 2, H - 1 - d),
            (d, d), (W - 1 - d, d), (d, H - 1 - d), (W - 1 - d, H - 1 - d)]


def cases(W, H, k):
    rng = np.random.default_rng(200 + k)
    for d in range(-7, 8):
        c = np.array(border_centres(W, H, d), np.float32)
        yield f"border{d:+d}", c, np.where(np.arange(len(c)) % 2 == 0, 100.0, 9000.0).astype(np.float32)
        t = c + np.float32(0.5) * np.array([1, -1], np.float32)             # exact .5 ties in both coordinates
        yield f"tie{d:+d}", t, EDGE_ERRORS[np.arange(len(t)) % 4]
    # overlapping disks of alternating colour: a tight cluster, then spread over the frame
    cl = np.array([W / 2, H / 2], np.float32) + rng.integers(-8, 9, (40, 2)).astype(np.float32)
    sp = (rng.random((160, 2)) * [W + 12, H + 12] - 6).astype(np.float32)
    c = np.concatenate([cl, sp])
    yield "overlap", c, np.where(np.arange(len(c)) % 2 == 0, 10.0, 8000.0).astype(np.float32)
    ties = np.concatenate([cl, sp]).round() + np.float32(0.5)
    yield "overlap_tie", ties.astype(np.float32), EDGE_ERRORS[np.arange(len(ties)) % 4]
    far = np.array([[1e6, 3], [3, -1e6], [LIMIT, LIMIT], [-LIMIT, 3], [3, LIMIT], [W // 2, H // 2],
                    [3e9, 3], [3, -3e9], [np.inf, 3], [3, -np.inf], [np.nan, 3], [3, np.nan], [LIMIT + 256, 3],
                    [W // 2 + 4, H // 2 + 1]], np.float32)
    yield "far", far, np.where(np.arange(len(far)) % 2 == 0, 1.0, 9e9).astype(np.float32)


def main():
    data = {"sizes": np.array(SIZES, np.int32), "cv2_version": np.array(cv2.__version__)}
    names = []
    for k, (W, H) in enumerate(SIZES):
        img = frame(k, W, H)
        data[f"frame{k}"] = img
        for name, cxy, err in cases(W, H, k):
            full = f"s{k}_{name}"
            names.append(full)
            data[f"{full}__size"] = np.array([k], np.int32)
            data[f"{full}__cxy"] = cxy
            data[f"{full}__err"] = err
            data[f"{full}__diff"] = draw(img, cxy, err) ^ img
    data["names"] = np.array(names)
    np.savez_compressed(OUT, **data)
    print(f"wrote {OUT}: {len(names)} cases, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
