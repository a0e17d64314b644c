"""The Velodyne step in front of the undistortion, on the host vs on the device (DESIGN.md section 8), for clouds without
per-point times: velodyne_handler's non-feature branch with the yaw-derived times (reference src/preprocess.cpp:376-428),
the time sort of sync_packages (src/laserMapping.cpp:551) and UndistortPcl's window (src/IMU_Processing.cpp:624-646),
followed by the propagation and undistortion of one scan-end update.

Per case (a VLP-16 spin of 25.2 k records and an HDL-64 spin of 130.2 k from synth.make_velodyne_spin, in two layouts and at
point_filter_num 1 and 4) the timed step, on the host clock and ending in a device synchronise:
  (a) host    the checker's velodyne_handler + std::stable_sort + window (tests/oracle_pre/velo_oracle.cpp and
              pre_oracle.window, one host thread, as the reference runs them; the 16-byte points are widened to the
              reference's 48-byte PointXYZINormal in between) + flb_imu_undistort from those points (out_xyz = NULL)
  (b) device  flb_lidar_upload_velodyne of the raw records (pageable source) + flb_imu_undistort_lidar (out_xyz = NULL)
The arms alternate in one process, one handle each; a 128 MB device fill between steps evicts L2 outside the timed
window; every case is warmed up, then timed for at least --seconds per arm.  The propagated state, the carry and the
point count of the two arms must be byte-identical.  Prints one JSON line per case and arm: ms per step (median, p10,
p90), for (a) also the host-only part, and the bytes the step puts on a copy engine; the GPU name, power limit and SM
clocks come from NVML in the same run.  Kernel-only times (CUDA events) are not taken: the device arm's kernels run
on the copy stream between two blocking reads, so the step time above is what a caller sees.
Usage: python profiles/velodyne_yaw_probe.py [--seconds 1.0]  (needs a GPU; writes nothing)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fastlivo_loader  # noqa: E402
import pre_oracle  # noqa: E402
import velo_oracle  # noqa: E402
from image_prep_probe import sm_clocks  # noqa: E402
from imu_util import product_inputs  # noqa: E402
from lidar_util import scan_end_offset  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402
from velo_util import c_velo_format, spin  # noqa: E402

CASES = [("vlp16_xyzir32_f1", "xyzir32", "vlp16", 1), ("vlp16_packed22_f4", "packed22", "vlp16", 4),
         ("hdl64_xyzirt_f1", "xyzirt", "hdl64", 1), ("hdl64_xyzir32_f4", "xyzir32", "hdl64", 4)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    evict = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    fi = flb.synth.make_imu_frame(seed=52, n_points=0)
    for name, layout, size, pfn in CASES:
        rec, fmt = spin(flb, layout, 1, pfn, size)
        n = len(rec) // fmt["point_step"]
        raw = np.frombuffer(rec, np.uint8)
        cf = c_velo_format(flb, fmt)
        hs = {arm: flb.Handle(device=0) for arm in ("host", "device")}
        ms = {"host": [], "device": []}
        host_only = []
        spent = {"host": 0.0, "device": 0.0}
        k = 0
        taken = {}
        while k < 12 or min(spent.values()) < args.seconds:
            res = {}
            for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                h = hs[arm]
                P, Cc, x = product_inputs(flb, fi)
                h.state_upload(x, x.copy())
                evict.fill_(k & 0xFF)
                torch.cuda.synchronize()
                h.synchronize()
                t0 = time.perf_counter()
                if arm == "host":
                    cloud, _ = velo_oracle.process(fmt, rec)
                    p48 = np.zeros((len(cloud), 12), np.float32)
                    p48[:, [0, 1, 2, 9]] = cloud
                    end, off = scan_end_offset(fi["pcl_beg_time"], p48[-1, 9])
                    win = pre_oracle.window(p48, 0, off)
                    tm = time.perf_counter()
                    h.imu_undistort(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, win, offset_index=9, download=False)
                    taken[arm] = len(win)
                else:
                    _, last, yaw_times = h.lidar_upload_velodyne(cf, raw, n)
                    assert yaw_times
                    end, off = scan_end_offset(fi["pcl_beg_time"], last)
                    taken[arm] = h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, off, True, download=False)[0]
                h.synchronize()
                t1 = time.perf_counter()
                if k >= 4:                                       # the first steps warm every shape up
                    ms[arm].append(1e3 * (t1 - t0))
                    spent[arm] += t1 - t0
                    if arm == "host":
                        host_only.append(1e3 * (tm - t0))
                res[arm] = (taken[arm], bytes(Cc), bytes(h.state_download()[0]))
            assert res["host"] == res["device"], f"{name}: the two arms differ"
            k += 1
        for h in hs.values():
            h.close()
        for arm in ("host", "device"):
            v = np.array(ms[arm])
            row = {"case": name, "arm": arm, "records": n, "point_step": fmt["point_step"], "point_filter_num": pfn,
                   "points_in_update": taken[arm],
                   "h2d_point_bytes_per_frame": 16 * taken[arm] if arm == "host" else fmt["point_step"] * n, "steps": len(v),
                   "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                   "ms_p90": round(float(np.percentile(v, 90)), 4), "outputs_equal": True}
            if arm == "host":
                row["host_only_ms_median"] = round(float(np.median(host_only)), 4)
            print(json.dumps(row), flush=True)
    print(json.dumps(sm_clocks()), flush=True)


if __name__ == "__main__":
    main()
