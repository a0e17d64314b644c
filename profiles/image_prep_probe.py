"""The camera step of a frame with the frame prepared on the host vs on the device (DESIGN.md section 8): LidarSelector::
detect's resize + cvtColor (src/lidar_selection.cpp:1029-1037) and publish_frame_world_rgb's colouring (src/
laserMapping.cpp:727-744).

Per configuration (C2: 640 x 512 camera, C4: 1280 x 1024) and source size (1x: the camera's, 2x: twice it), a handle
holds the frame's world cloud (flb_world_cloud of the scan, untimed).  The timed step, on the host clock and ending in a
synchronise:
  (a) host    cv2.resize + cv2.cvtColor (or their numpy restatement when cv2 is not importable) + flb_image_upload of the
              gray image + flb_colorize_cloud with the host colour frame (its own upload)
  (b) device  flb_image_upload_bgr of the raw frame + flb_colorize_cloud(bgr = NULL)
The arms alternate frame by frame in one process, one handle each, over --frames distinct frames; the gray images
(flb_image_download) and the colours must be byte-identical.  Prints one JSON line per configuration, source size and
arm: ms per step (median, p10, p90, the first frame of each arm left out) and the host-to-device bytes per frame; the GPU
name, power limit and SM clocks come from NVML in the same run.
Usage: python profiles/image_prep_probe.py [--frames 40]  (needs a GPU; writes nothing)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fastlivo_loader  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402

try:
    import cv2
except ImportError:
    cv2 = None


def sm_clocks():
    """Current SM and memory clocks (MHz) of GPU 0 through NVML (read only)."""
    nv = C.CDLL("libnvidia-ml.so.1")
    nv.nvmlInit_v2()
    dev = C.c_void_p()
    nv.nvmlDeviceGetHandleByIndex_v2(0, C.byref(dev))
    sm, mem = C.c_uint(), C.c_uint()
    nv.nvmlDeviceGetClockInfo(dev, 1, C.byref(sm))                 # NVML_CLOCK_SM
    nv.nvmlDeviceGetClockInfo(dev, 2, C.byref(mem))                # NVML_CLOCK_MEM
    nv.nvmlShutdown()
    return dict(sm_clock_mhz=sm.value, mem_clock_mhz=mem.value)


def host_prep(src, W, H):
    """detect()'s resize (when the frame is not the camera's size) and cvtColor: (img_rgb, gray)."""
    if cv2 is not None:
        img = src if src.shape[:2] == (H, W) else cv2.resize(src, (W, H), 0, 0, cv2.INTER_LINEAR)
        return img, cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)
    img = src
    if src.shape[:2] != (H, W):
        s = src.astype(np.uint16)
        img = ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    b, g, r = (img[..., k].astype(np.uint32) for k in range(3))
    return img, ((3735 * b + 19235 * g + 9798 * r + (1 << 14)) >> 15).astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(dict(nvml_gpu(), host_prep="cv2 " + cv2.__version__ if cv2 is not None else "numpy")), flush=True)
    for name in ("C2", "C4"):
        seq = flb.synth.make_visual_sequence(name, 2)
        W, H = seq["cam"]["width"], seq["cam"]["height"]
        fr = seq["frames"][1]
        prm = flb.capi.lio_params(dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"]), 3)
        for scale in (1, 2):
            rng = np.random.default_rng(scale)
            base = np.stack([fr["image"], np.roll(fr["image"], 3, 1), 255 - fr["image"]], -1)
            if scale == 2:
                base = np.repeat(np.repeat(base, 2, 0), 2, 1)
            frames = [np.ascontiguousarray(base ^ rng.integers(0, 8, base.shape, dtype=np.uint8)) for _ in range(args.frames)]
            hs = {}
            for arm in ("host", "device"):
                h = hs[arm] = flb.Handle(device=0)
                h.camera_set(seq["cam"])
                h.scan_upload(fr["scan_body"])
                n_pts = h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
            ms = {"host": [], "device": []}
            equal = True
            for k, src in enumerate(frames):
                res = {}
                for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                    h = hs[arm]
                    h.synchronize()
                    t0 = time.perf_counter()
                    if arm == "host":
                        img, gray = host_prep(src, W, H)
                        h.image_upload(gray)
                        rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"], img)
                    else:
                        h.image_upload_bgr(src)
                        rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"])
                    h.synchronize()
                    t1 = time.perf_counter()
                    if k > 1:
                        ms[arm].append(1e3 * (t1 - t0))
                    res[arm] = (h.image_download(bgr=False)[0].tobytes(), rgb.tobytes(), val.tobytes())
                equal = equal and res["host"] == res["device"]
            for h in hs.values():
                h.close()
            for arm in ("host", "device"):
                v = np.array(ms[arm])
                h2d = 4 * W * H if arm == "host" else 3 * scale * scale * W * H
                print(json.dumps({"config": name, "camera": [W, H], "source_scale": scale, "arm": arm, "cloud_points": n_pts,
                                  "h2d_bytes_per_frame": h2d, "steps": len(v), "ms_median": round(float(np.median(v)), 4),
                                  "ms_p10": round(float(np.percentile(v, 10)), 4), "ms_p90": round(float(np.percentile(v, 90)), 4),
                                  "outputs_equal": equal}), flush=True)
            assert equal, f"{name} {scale}x: the two arms differ"
    print(json.dumps(sm_clocks()), flush=True)


if __name__ == "__main__":
    main()
