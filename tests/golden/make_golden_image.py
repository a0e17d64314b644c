"""Generate tests/golden/image_golden.npz: small BGR8 camera frames and what OpenCV makes of them in
LidarSelector::detect (src/lidar_selection.cpp:1029-1037): cv::resize(0.5, INTER_LINEAR) when the frame is twice the
camera's size, then cv::cvtColor(BGR2GRAY).  Needs cv2.  Run from the repo root:
    python tests/golden/make_golden_image.py

Every case holds its source as rows of `stride` bytes, the pixels in the first 3 * width of each row (strided cases
have padding after them), the camera size, and cv2's colour frame (img_rgb) and gray image at that size.  The cameras
are 160 x 128 (the synthetic texture and flat fields), 96 x 64 (random noise) and 42 x 18 (a width that is not a
multiple of 4).  The file stays under 1 MB."""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import fastlivo_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "image_golden.npz")


def texture_bgr():
    """The synthetic scene's texture (T0 frame, 320 x 256) as three distinct channels."""
    img = fastlivo_loader.load().synth.make_frame("T0")["image"]
    return np.ascontiguousarray(np.stack([img, np.roll(img, 5, 1), 255 - np.roll(img, 3, 0)], -1))


def main():
    rng = np.random.default_rng(20261016)
    tex = texture_bgr()
    cases = {
        # name: (camera (W, H), source frame (h, w, 3), padding bytes after each row)
        "noise_1x": ((96, 64), rng.integers(0, 256, (64, 96, 3), dtype=np.uint8), 0),
        "noise_2x": ((96, 64), rng.integers(0, 256, (128, 192, 3), dtype=np.uint8), 0),
        "texture_1x": ((160, 128), np.ascontiguousarray(tex[::2, ::2]), 0),
        "texture_2x_strided": ((160, 128), tex, 13),
        "noise_1x_strided": ((96, 64), rng.integers(0, 256, (64, 96, 3), dtype=np.uint8), 7),
        "flat0_1x": ((160, 128), np.zeros((128, 160, 3), np.uint8), 0),
        "flat255_2x": ((160, 128), np.full((256, 320, 3), 255, np.uint8), 0),
        "odd_1x": ((42, 18), rng.integers(0, 256, (18, 42, 3), dtype=np.uint8), 0),
        "odd_2x_strided": ((42, 18), rng.integers(0, 256, (36, 84, 3), dtype=np.uint8), 5),
    }
    out = {"cv2_version": np.array(cv2.__version__), "names": np.array(sorted(cases))}
    for name, ((W, H), src, pad) in cases.items():
        h, w = src.shape[:2]
        rows = np.zeros((h, 3 * w + pad), np.uint8)
        rows[:, :3 * w] = src.reshape(h, 3 * w)
        rows[:, 3 * w:] = rng.integers(0, 256, (h, pad), dtype=np.uint8)
        img = src
        if (w, h) != (W, H):
            img = cv2.resize(src, (int(w * 0.5), int(h * 0.5)), 0, 0, cv2.INTER_LINEAR)
        assert img.shape == (H, W, 3)
        out[f"{name}__rows"] = rows
        out[f"{name}__size"] = np.array([w, h, W, H], np.int32)
        out[f"{name}__bgr"] = np.ascontiguousarray(img)
        out[f"{name}__gray"] = cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, OpenCV {cv2.__version__})")


if __name__ == "__main__":
    main()
