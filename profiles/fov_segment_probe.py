"""lasermap_fov_segment through the host vs on the device (DESIGN.md section 8): the host cube tracker +
flb_map_delete_boxes (a full map rebuild per call) against flb_map_fov_segment (the cube on the device, the points in the
boxes merged out of the live sorted map), each followed by the frame's flb_map_add_scan, because the rebuild's box shrink
moves cost onto the add step.

Maps C2 and C3 (the synthetic room, 240 k / 1 M points).  Configurations:
  shipped  cube_side_length 20, DET_RANGE 300, MOV_THRESHOLD 1.5: three boxes every frame; frame 2 cuts the 20 m cube
           around the start, frame 3 one 140-160 m away, the later boxes lie 290 m or more away and are empty
  slab     cube 100 m, DET_RANGE 30, MOV_THRESHOLD 1.5: the sensor drives along +x at 2 m a frame and a 15 m slab of the
           room is cut every 7-8 frames; the frames in between have no box
Per frame (--frames, the sensor jitters by +-0.5 m about its path), the two arms alternate in one process, one handle each:
  (a) host    oracle tracker step + flb_map_delete_boxes(cub_needrm) when there is a box, then flb_map_add_scan
  (b) device  flb_map_fov_segment, then flb_map_add_scan
Timed on the host clock around the map step (the L2 flush and the scan upload outside it).  Prints one JSON line per
map, configuration and arm: ms per frame (median, p10, p90 over every frame after the first two), launches per frame,
points cut in all, and whether the two maps hold the same point set at the end.  GPU name, power limit and SM clocks come
from NVML in the same run.
Usage: python profiles/fov_segment_probe.py [--frames 40]  (needs a GPU; writes nothing)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fastlivo_loader  # noqa: E402
import fov_oracle  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402

CONFIGS = {"shipped": (fov_oracle.SHIPPED, np.zeros(3)), "slab": ((100.0, 30.0, 1.5), np.array([2.0, 0.0, 0.0]))}


def sm_clock_now():
    nv = C.CDLL("libnvidia-ml.so.1")
    nv.nvmlInit_v2()
    dev = C.c_void_p()
    nv.nvmlDeviceGetHandleByIndex_v2(0, C.byref(dev))
    clk = C.c_uint()
    nv.nvmlDeviceGetClockInfo(dev, 1, C.byref(clk))                 # NVML_CLOCK_SM, current
    nv.nvmlShutdown()
    return clk.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--ds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    clocks = []
    for name in ("C2", "C3"):
        f = flb.synth.make_frame(name)
        lprm = flb.capi.lio_params(f, 3)
        for cfg, (prm, vel) in CONFIGS.items():
            rng = np.random.default_rng(3)
            traj = [np.asarray(f["p_true"], np.float64) + k * vel + rng.uniform(-0.5, 0.5, 3) for k in range(args.frames)]
            hs, ms, launches, cut = {}, {"host": [], "device": []}, {"host": [], "device": []}, {"host": 0, "device": 0}
            for arm in ("host", "device"):
                hs[arm] = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
                hs[arm].map_upload(f["map_xyz"])
                hs[arm].scan_upload(f["scan_body"])
            tracker = fov_oracle.Tracker(*prm)
            for k, p in enumerate(traj):
                for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                    h = hs[arm]
                    flush_buf.fill_(k & 0xFF)
                    torch.cuda.synchronize()
                    h.synchronize()
                    M0, l0 = h.M, h.launch_count()
                    t0 = time.perf_counter()
                    if arm == "host":
                        boxes, _ = tracker.step(p)
                        if len(boxes):
                            h.map_delete_boxes(boxes)
                    else:
                        h.map_fov_segment(*prm, pos=p)
                    Mc = h.M
                    h.map_add_scan(lprm, args.ds, f["R_true"], p)
                    t1 = time.perf_counter()
                    cut[arm] += M0 - Mc
                    if k >= 2:
                        ms[arm].append(1e3 * (t1 - t0))
                        launches[arm].append(h.launch_count() - l0)
            clocks.append(sm_clock_now())
            ma, mb = hs["host"].map_download(), hs["device"].map_download()
            key = lambda m: m[np.lexsort((m[:, 2], m[:, 1], m[:, 0]))].tobytes()   # noqa: E731
            same_set = len(ma) == len(mb) and key(ma) == key(mb)
            for arm in ("host", "device"):
                v = np.array(ms[arm])
                print(json.dumps({"map": name, "config": cfg, "arm": arm, "map_points": len(f["map_xyz"]), "frames": len(v),
                                  "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                                  "ms_p90": round(float(np.percentile(v, 90)), 4),
                                  "launches_per_frame": [int(np.min(launches[arm])), int(np.median(launches[arm])), int(np.max(launches[arm]))],
                                  "points_cut": int(cut[arm]), "map_points_end": int(hs[arm].M), "maps_same_set": same_set}), flush=True)
            for h in hs.values():
                h.close()
    print(json.dumps({"sm_clock_mhz_after_each_case": clocks}), flush=True)


if __name__ == "__main__":
    main()
