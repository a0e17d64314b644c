"""Generate tests/golden/image_msg_golden.npz: camera messages in every encoding flb_image_upload_msg takes, and what
cv_bridge and LidarSelector::detect make of them: cv2.cvtColor(frame, code) to BGR8 (cv_bridge::toCvCopy(msg, "bgr8"),
src/laserMapping.cpp:490-493), cv2.resize(0.5, INTER_LINEAR) to (int)(cols * 0.5) x (int)(rows * 0.5) when the size
differs from the camera's, then cv2.cvtColor(BGR2GRAY) (src/lidar_selection.cpp:1029-1037).  Needs cv2.  Run from the
repo root:
    python tests/golden/make_golden_image_msg.py

Every case holds its message as rows of `step` bytes, the pixels first (strided cases have padding after them), the
encoding, the camera size, and cv2's colour frame (img_rgb) and FLB_GRAY_CV4 gray image at that size.  Sizes, for
every encoding: 32 x 16 camera at 1x, 2x, odd width, odd height and both odd; a 42 x 18 camera (a width that is not a
multiple of 4) at 1x and with both sides odd, strided; the smallest camera (16 x 16) at 1x and both odd; and a 642 x 16
camera from a 1285 x 33 frame, wide enough for OpenCV's vector paths.  The file stays under 1 MB."""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import fastlivo_loader  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "image_msg_golden.npz")

# encoding: (FLB_ENC_*, bytes per pixel, cv2 conversion to BGR or None)
ENCODINGS = {
    "bgr8": (0, 3, None),
    "rgb8": (1, 3, cv2.COLOR_RGB2BGR),
    "mono8": (2, 1, cv2.COLOR_GRAY2BGR),
    "bgra8": (3, 4, cv2.COLOR_BGRA2BGR),
    "rgba8": (4, 4, cv2.COLOR_RGBA2BGR),
    "bayer_rggb8": (5, 1, cv2.COLOR_BayerBG2BGR),
    "bayer_bggr8": (6, 1, cv2.COLOR_BayerRG2BGR),
    "bayer_gbrg8": (7, 1, cv2.COLOR_BayerGR2BGR),
    "bayer_grbg8": (8, 1, cv2.COLOR_BayerGB2BGR),
}
# size name: (camera (W, H), frame (w, h), padding bytes after each row, texture source)
SIZES = {
    "1x": ((32, 16), (32, 16), 0, False),
    "2x": ((32, 16), (64, 32), 0, False),
    "oddw": ((32, 16), (65, 32), 0, False),
    "oddh": ((32, 16), (64, 33), 0, False),
    "oddwh": ((32, 16), (65, 33), 0, False),
    "w42_1x_strided": ((42, 18), (42, 18), 7, False),
    "w42_oddwh_strided": ((42, 18), (85, 37), 5, False),
    "min_1x": ((16, 16), (16, 16), 0, False),
    "min_oddwh": ((16, 16), (33, 33), 0, False),
    "wide_oddwh": ((642, 16), (1285, 33), 0, True),
}


def texture(w, h, bpp):
    """The synthetic scene's texture (T0 frame) tiled to h x w, as bpp distinct channels."""
    img = fastlivo_loader.load().synth.make_frame("T0")["image"]
    planes = [img, np.roll(img, 5, 1), 255 - np.roll(img, 3, 0), np.roll(img, 7, 0)][:bpp]
    t = np.stack(planes, -1)
    reps = (-(-h // t.shape[0]), -(-w // t.shape[1]), 1)
    return np.ascontiguousarray(np.tile(t, reps)[:h, :w])


def to_bgr(frame, code):
    return np.ascontiguousarray(frame if code is None else cv2.cvtColor(frame, code))


def main():
    rng = np.random.default_rng(20261017)
    names = []
    out = {"cv2_version": np.array(cv2.__version__)}
    for enc, (flb_enc, bpp, code) in ENCODINGS.items():
        for size, ((W, H), (w, h), pad, tex) in SIZES.items():
            name = f"{enc}__{size}"
            src = texture(w, h, bpp) if tex else rng.integers(0, 256, (h, w, bpp), dtype=np.uint8)
            frame = src[..., 0] if bpp == 1 else src
            bgr = to_bgr(frame, code)
            if (w, h) != (W, H):
                bgr = cv2.resize(bgr, (int(w * 0.5), int(h * 0.5)), 0, 0, cv2.INTER_LINEAR)
            assert bgr.shape == (H, W, 3)
            rows = np.zeros((h, bpp * w + pad), np.uint8)
            rows[:, :bpp * w] = src.reshape(h, bpp * w)
            rows[:, bpp * w:] = rng.integers(0, 256, (h, pad), dtype=np.uint8)
            out[f"{name}__rows"] = rows
            out[f"{name}__size"] = np.array([w, h, W, H, flb_enc, bpp], np.int32)
            out[f"{name}__bgr"] = np.ascontiguousarray(bgr)
            out[f"{name}__gray"] = cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)
            names.append(name)
    out["names"] = np.array(names)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, OpenCV {cv2.__version__})")


if __name__ == "__main__":
    main()
