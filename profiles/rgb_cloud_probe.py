"""publish_frame_world_rgb's cloud and the pcd_save_en map: the host route against flb_rgb_cloud (DESIGN.md section 8).

Per world-cloud size (24 k points: C2's scan; 65 k; 130 k: Ouster-64 dense) one C2-camera frame (640 x 512, its image
as the image set's colour frame) and a scan of that many points drawn like C2's (the LiDAR field of view is wider
than the camera's, so only part of the cloud is coloured).  Three handles hold the same world cloud.  Timed on the
host clock, each step ending in a synchronise, the arms alternating their order step by step:
  (a) host    flb_colorize_cloud (rgb + valid read back) + flb_world_cloud_download (xyz) + compaction into 32-byte
              pcl::PointXYZRGB records in numpy (the stand-in for the node's push_back loop)
  (b) device  flb_rgb_cloud + flb_rgb_cloud_download of the records
  (s) save    (b) on a handle with flb_rgb_save_begin open: the per-frame cost of the append is (s) - (b)
After the steps the whole save (steps x records) is read back with flb_rgb_save_download into pageable memory, timed
once: the download rate.  The records of (a) and (b) are asserted byte-identical.  Prints one JSON line per size and
arm (ms per step: median, p10, p90), one per size for the save download (GB/s of 32-byte records); the GPU name, power
limit and maximum SM clock come from NVML in the same run.
Usage: python profiles/rgb_cloud_probe.py [--steps 60]  (needs a GPU; writes nothing)."""
import argparse
import dataclasses
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


def host_route(flb, h):
    """The host route: colour flags and world xyz read back, compacted into records on the host."""
    rgb, val = h.colorize_cloud(None, None)
    xyz = h.world_cloud_download()
    kept = xyz[val]
    out = np.zeros(len(kept), flb.capi.RGB_POINT)
    out["x"], out["y"], out["z"] = kept[:, 0], kept[:, 1], kept[:, 2]
    out["w"] = 1.0
    out["r"], out["g"], out["b"] = rgb[val, 0], rgb[val, 1], rgb[val, 2]
    out["a"] = 255
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    for n_points in (24000, 65000, 130000):
        cfg = dataclasses.replace(flb.synth.CONFIGS["C2"], n_scan=n_points)
        seq = flb.synth.make_visual_sequence(cfg, 1)
        fr = seq["frames"][0]
        prm = flb.capi.lio_params(dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"]), 3)
        bgr = np.ascontiguousarray(np.stack([fr["image"], np.roll(fr["image"], 3, 1), 255 - fr["image"]], -1))
        hs = {}
        for arm in ("host", "device", "save"):
            h = flb.Handle(device=0)
            h.camera_set(seq["cam"])
            h.vmap_reset(seq, grid_size=32, outlier_threshold=1000.0)
            x = flb.capi.State18.make(fr["R"], fr["p"], cov=seq["cov"])
            h.state_upload(x, x.copy())
            h.image_upload_bgr(bgr)
            h.scan_upload(fr["scan_body"])
            assert h.world_cloud(prm, flb.capi.CLOUD_SCAN) == n_points
            hs[arm] = h
        hs["save"].rgb_save_begin(1 << 40)
        ms = {arm: [] for arm in hs}
        ref = None
        for k in range(args.steps + 2):
            order = list(hs) if k % 2 == 0 else list(reversed(list(hs)))
            for arm in order:
                h = hs[arm]
                t0 = time.perf_counter()
                if arm == "host":
                    out = host_route(flb, h)
                else:
                    h.rgb_cloud(None, None)
                    out = h.rgb_cloud_download()
                h.synchronize()
                t1 = time.perf_counter()
                if k >= 2:                                   # two warm-up steps per arm
                    ms[arm].append(1e3 * (t1 - t0))
                if ref is None:
                    ref = out
                assert out.tobytes() == ref.tobytes()
        for arm, v in ms.items():
            v = np.array(v)
            print(json.dumps({"world_points": n_points, "coloured": len(ref), "arm": arm, "steps": len(v),
                              "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                              "ms_p90": round(float(np.percentile(v, 90)), 4)}), flush=True)
        h = hs["save"]
        size = h.rgb_save_size()
        assert size["n"] == (args.steps + 2) * len(ref) and size["dropped"] == 0
        t0 = time.perf_counter()
        whole = h.rgb_save_download()
        t1 = time.perf_counter()
        assert whole[-len(ref):].tobytes() == ref.tobytes()
        print(json.dumps({"world_points": n_points, "save_records": size["n"], "save_device_bytes": size["device_bytes"],
                          "download_ms": round(1e3 * (t1 - t0), 3), "download_gb_s": round(32 * size["n"] / (t1 - t0) / 1e9, 3)}),
              flush=True)
        for h in hs.values():
            h.close()


if __name__ == "__main__":
    main()
