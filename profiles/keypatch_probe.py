"""display_keypatch's image on the host vs on the device (DESIGN.md section 8): the img_cp a node publishes on img_pub
(src/laserMapping.cpp:1369-1375), LidarSelector::display_keypatch's circles (src/lidar_selection.cpp:985-1005) on the
camera-size colour frame.

Workload: C2's 640 x 512 camera from a 1281 x 1025 bayer_grbg8 message, with 200 patches (a real frame's selection)
and 2000 (C2's), spread over the frame at 5 m.  An uploaded patch list's errors are zero until a VIO pass runs, so
every circle is green on both arms.  The timed step, on the host clock:
  (a) host    what a node does today for img_cp: cv2.cvtColor of the mosaic to BGR (cv_bridge's demosaic),
              cv2.resize(INTER_LINEAR) to the camera's size, then one cv2.circle(c, 6, colour, -1, 8) per patch, on one
              host thread (cv2.setNumThreads(1)); the centres are projected beforehand
  (b) device  flb_keypatch_image into page-locked memory, completed by flb_synchronize (the message was uploaded for
              the VIO update anyway)
The arms alternate step by step in one process after a warm-up, for at least --seconds of timed steps each; their
frames must be byte-identical.  Prints one JSON line per patch count and arm: ms per step (median, p10, p90); the GPU
name, power limit and SM clocks come from NVML in the same run.  Needs a GPU and cv2.
Usage: python profiles/keypatch_probe.py [--seconds 1.5]  (writes nothing)."""
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

W, H = 640, 512
COUNTS = (200, 2000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.5)
    args = ap.parse_args()
    cv2.setNumThreads(1)
    flb = fastlivo_loader.load()
    print(json.dumps(dict(nvml_gpu(), host="cv2 " + cv2.__version__ + ", 1 thread")), flush=True)
    image = flb.synth.make_frame("T0")["image"]
    mosaic = flb.synth.bayer_message(flb.synth.texture_bgr(image, 2 * W + 1, 2 * H + 1), "bayer_grbg8")
    cam = dict(width=W, height=H, fx=0.6 * W, fy=0.6 * W, cx=0.5 * W, cy=0.5 * H, d=[0.0] * 5)
    R, P = np.eye(3), np.zeros(3)
    for n in COUNTS:
        rng = np.random.default_rng(n)
        px = rng.random((n, 2)) * [W + 8, H + 8] - 4
        z = 5.0
        pos = np.stack([(px[:, 0] - cam["cx"]) / cam["fx"] * z, (px[:, 1] - cam["cy"]) / cam["fy"] * z, np.full(n, z)], 1)
        # the device's projection (identity pose, no distortion): x / z, then fx * x + cx; rounded to float, then to int
        pc = np.stack([cam["fx"] * (pos[:, 0] / pos[:, 2]) + cam["cx"], cam["fy"] * (pos[:, 1] / pos[:, 2]) + cam["cy"]], 1)
        centres = [(int(x), int(y)) for x, y in np.rint(pc.astype(np.float32))]
        hd = flb.Handle(device=0)
        hd.camera_set(cam)
        hd.image_upload_msg(mosaic, "bayer_grbg8")
        hd.patches_upload(pos, np.zeros((n, 192), np.float32), np.zeros(n, np.int32))
        out = hd.pinned_like(np.zeros((H, W, 3), np.uint8))

        def host_step():
            img = cv2.resize(cv2.cvtColor(mosaic, cv2.COLOR_BayerGB2BGR), (W, H), 0, 0, cv2.INTER_LINEAR)
            for c in centres:
                cv2.circle(img, c, 6, (0, 255, 0), -1, 8)
            return img

        def device_step():
            hd.keypatch_image(R, P, out=out)
            hd.synchronize()
            return out

        for _ in range(5):
            host_step(), device_step()
        equal = np.array_equal(host_step(), device_step())
        ms = {"host": [], "device": []}
        t_end = {"host": 0.0, "device": 0.0}
        k = 0
        while min(t_end.values()) < args.seconds:
            for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                hd.synchronize()
                t0 = time.perf_counter()
                host_step() if arm == "host" else device_step()
                dt = time.perf_counter() - t0
                ms[arm].append(1e3 * dt)
                t_end[arm] += dt
            k += 1
        hd.close()
        for arm in ("host", "device"):
            v = np.array(ms[arm])
            print(json.dumps({"camera": [W, H], "message": [2 * W + 1, 2 * H + 1], "patches": n, "arm": arm, "steps": len(v),
                              "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                              "ms_p90": round(float(np.percentile(v, 90)), 4), "outputs_equal": bool(equal)}), flush=True)
        assert equal, f"{n} patches: the two arms differ"
    print(json.dumps(sm_clocks()), flush=True)


if __name__ == "__main__":
    main()
