"""Surface features in front of the undistortion, on the host vs on the device (DESIGN.md section 8), for
feature_extract_enable: 1: the handlers' feature branches with give_feature (reference src/preprocess.cpp:94-135,
:174-227, :299-373, :466-936), the time sort of sync_packages (src/laserMapping.cpp:551) and UndistortPcl's window
(src/IMU_Processing.cpp:624-646), followed by the propagation and undistortion of one scan-end update.

Per case (an Avia message of 24 k records, Ouster-64 and Ouster-128 spins of 1024 columns and an HDL-64 spin of 1800
columns, all from synth.make_feature_scan) the timed step, on the host clock and ending in a device synchronise:
  (a) host    the checker's restatement of the feature branch + std::stable_sort (tests/oracle_pre/feat_oracle.cpp,
              one host thread, g++ -O2 -ffp-contract=off) + the window + flb_imu_undistort from those points
  (b) device  flb_lidar_upload_features / flb_lidar_upload_velodyne_features of the raw records (pageable source) +
              flb_imu_undistort_lidar
Both with out_xyz = NULL.  The arms alternate in one process, one handle each; a 128 MB device fill between steps evicts
L2 outside the timed window; every case is warmed up, then timed for at least --seconds per arm.  The propagated state,
the carry and the point count of the two arms must be byte-identical.  Prints one JSON line per case and arm: ms per
step (median, p10, p90), for (a) also the host-only part, and the point bytes the step puts on a copy engine; the GPU
name, power limit and SM clocks come from NVML in the same run.  Kernel-only times are not taken.
Usage: python profiles/lidar_features_probe.py [--seconds 1.0]  (needs a GPU; writes nothing)."""
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
import feat_oracle  # noqa: E402
import pre_oracle  # noqa: E402
from feat_util import scene  # noqa: E402
from image_prep_probe import sm_clocks  # noqa: E402
from imu_util import product_inputs  # noqa: E402
from lidar_util import c_format, scan_end_offset  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402
from velo_util import c_velo_format  # noqa: E402

CASES = [("avia_f1", "livox", dict(n_cols=4000), 1), ("ouster64_f1", "ouster", dict(n_scans=64, n_cols=1024), 1),
         ("ouster128_f2", "ouster", dict(n_scans=128, n_cols=1024), 2),
         ("hdl64_f1", "velodyne", dict(n_scans=64, n_cols=1800, timed=True, nan_returns=False), 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    evict = torch.empty(128 << 20, dtype=torch.uint8, device="cuda")
    fi = flb.synth.make_imu_frame(seed=53, n_points=0)
    for name, kind, kw, pfn in CASES:
        rec, fmt = scene(kind, point_filter_num=pfn, seed=1, **kw)
        n = len(rec) // fmt["point_step"]
        raw = np.frombuffer(rec, np.uint8)
        if kind == "velodyne":
            cf = c_velo_format(flb, dict(point_step=fmt["point_step"], off_x=0, off_y=4, off_z=8, off_time=fmt["off_time"],
                                         off_ring=fmt["off_line"], n_scans=fmt["n_scans"], point_filter_num=pfn, blind=fmt["blind"]))
            dev_upload = lambda h: h.lidar_upload_velodyne_features(cf, raw, 0.0, n)[:2]  # noqa: E731
        else:
            cf = c_format(flb, fmt)
            dev_upload = lambda h: h.lidar_upload_features(cf, raw, 0.0, n)  # noqa: E731
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
                    cloud = feat_oracle.process(fmt, rec)[0]
                    p48 = np.zeros((len(cloud), 12), np.float32)
                    p48[:, [0, 1, 2, 9]] = cloud
                    end, off = scan_end_offset(fi["pcl_beg_time"], p48[-1, 9])
                    win = pre_oracle.window(p48, 0, off)
                    tm = time.perf_counter()
                    h.imu_undistort(P, Cc, fi["v_imu"], fi["pcl_beg_time"], end, win, offset_index=9, download=False)
                    taken[arm] = len(win)
                else:
                    _, last = dev_upload(h)
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
