"""The camera message's conversion on the host vs on the device (DESIGN.md section 8): cv_bridge::toCvCopy(msg, "bgr8")
(src/laserMapping.cpp:490-493) and LidarSelector::detect's resize + cvtColor (src/lidar_selection.cpp:1029-1037).

Workloads (message encoding, message size -> camera size):
  mono8        752 x 480   -> 752 x 480     (NTU_VIRAL's camera)
  rgb8        1280 x 1024  -> 1280 x 1024
  bayer_rggb8 2448 x 2048  -> 1224 x 1024   (MARS_LVIG's halving, the 2x2 area path)
  bayer_rggb8 2449 x 2049  -> 1224 x 1024   (the same with odd sides, the linear path)
The timed step, on the host clock and ending in a synchronise:
  (a) host    cv2.cvtColor to BGR + cv2.resize(INTER_LINEAR) when the size differs, on one host thread
              (cv2.setNumThreads(1)), then flb_image_upload_bgr of the camera-size frame
  (b) device  flb_image_upload_msg of the message's own bytes
The arms alternate frame by frame in one process, one handle each, over --frames distinct frames; their image sets
(flb_image_download) must be byte-identical.  Prints one JSON line per workload and arm: ms per step (median, p10,
p90, the first two frames left out) and the host-to-device bytes per frame; the GPU name, power limit and SM clocks
come from NVML in the same run.  Needs a GPU and cv2.
Usage: python profiles/image_msg_probe.py [--frames 40]  (writes nothing)."""
import argparse
import json
import os
import sys
import time

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fastlivo_loader  # noqa: E402
from image_prep_probe import sm_clocks  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402

WORKLOADS = [("mono8", (752, 480), (752, 480)), ("rgb8", (1280, 1024), (1280, 1024)),
             ("bayer_rggb8", (2448, 2048), (1224, 1024)), ("bayer_rggb8", (2449, 2049), (1224, 1024))]
CODES = {"mono8": cv2.COLOR_GRAY2BGR, "rgb8": cv2.COLOR_RGB2BGR, "bayer_rggb8": cv2.COLOR_BayerBG2BGR}


def host_route(msg, encoding, W, H):
    bgr = cv2.cvtColor(msg, CODES[encoding])
    if bgr.shape[:2] != (H, W):
        bgr = cv2.resize(bgr, (W, H), 0, 0, cv2.INTER_LINEAR)
    return bgr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    args = ap.parse_args()
    cv2.setNumThreads(1)
    flb = fastlivo_loader.load()
    print(json.dumps(dict(nvml_gpu(), host="cv2 " + cv2.__version__ + ", 1 thread")), flush=True)
    image = flb.synth.make_frame("T0")["image"]
    for encoding, (w, h), (W, H) in WORKLOADS:
        rng = np.random.default_rng(w + h)
        msgs = []
        for _ in range(args.frames):
            bgr = flb.synth.texture_bgr(image, w, h) ^ rng.integers(0, 8, (h, w, 3), dtype=np.uint8)
            msgs.append(flb.synth.mono_message(bgr) if encoding == "mono8" else flb.synth.bayer_message(bgr, encoding)
                        if encoding.startswith("bayer") else np.ascontiguousarray(bgr[..., ::-1]))
        cam = dict(width=W, height=H, fx=0.6 * W, fy=0.6 * W, cx=0.5 * W, cy=0.5 * H, d=[0.0] * 5)
        hs = {}
        for arm in ("host", "device"):
            hs[arm] = flb.Handle(device=0)
            hs[arm].camera_set(cam)
        ms = {"host": [], "device": []}
        equal = True
        for k, msg in enumerate(msgs):
            res = {}
            for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                hd = hs[arm]
                hd.synchronize()
                t0 = time.perf_counter()
                if arm == "host":
                    hd.image_upload_bgr(host_route(msg, encoding, W, H))
                else:
                    hd.image_upload_msg(msg, encoding)
                hd.synchronize()
                t1 = time.perf_counter()
                if k > 1:
                    ms[arm].append(1e3 * (t1 - t0))
                g, c = hd.image_download()
                res[arm] = (g.tobytes(), c.tobytes())
            equal = equal and res["host"] == res["device"]
        for hd in hs.values():
            hd.close()
        bpp = 1 if encoding != "rgb8" else 3
        for arm in ("host", "device"):
            v = np.array(ms[arm])
            h2d = 3 * W * H if arm == "host" else bpp * w * h
            print(json.dumps({"encoding": encoding, "message": [w, h], "camera": [W, H], "arm": arm, "h2d_bytes_per_frame": h2d,
                              "steps": len(v), "ms_median": round(float(np.median(v)), 4),
                              "ms_p10": round(float(np.percentile(v, 10)), 4), "ms_p90": round(float(np.percentile(v, 90)), 4),
                              "outputs_equal": equal}), flush=True)
        assert equal, f"{encoding} {w}x{h}: the two arms differ"
    print(json.dumps(sm_clocks()), flush=True)


if __name__ == "__main__":
    main()
