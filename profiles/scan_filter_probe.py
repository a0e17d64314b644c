"""The LIO scan from the undistorted cloud through the host vs on the device (DESIGN.md section 8): the per-frame step
undistort -> downSizeFilterSurf -> scan upload, as the host chain against flb_scan_from_undistorted.

Per raw cloud (the C2 and C3 frames' scan_body, 24 k and 100 k points, as the raw points of one IMU frame) and leaf
(0.15: filter_size_surf of config/avia.yaml / mid360.yaml / MARS_LVIG.yaml; 0.5: of NTU_VIRAL.yaml), --frames frames,
each a small rotation of the cloud.  Every frame, untimed: state upload, synchronise.  Then the timed step on the host
clock, ending in a synchronise:
  (a) host    flb_imu_undistort with out_xyz + flb_voxel_grid on a second handle (host in, host out: a stand-in for
              PCL, if anything an optimistic one) + flb_scan_upload
  (b) device  flb_imu_undistort with out_xyz = NULL + flb_scan_from_undistorted
The arms alternate frame by frame in one process, one handle each (same map).  After every frame, untimed, both scan
orders and the posterior and report of a flb_lio_update on the scan must be byte-identical.  Prints one JSON line per
configuration and arm: ms per step (median, p10, p90 over every frame but the first); the GPU name, power limit and
maximum SM clock come from NVML in the same run.
Usage: python profiles/scan_filter_probe.py [--frames 40]  (needs a GPU; writes nothing)."""
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
from imu_util import product_inputs  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    imu = flb.synth.make_imu_frame(seed=5, n_points=0)
    for name in ("C2", "C3"):
        f = flb.synth.make_frame(name)
        prm = flb.capi.lio_params(f, 3)
        for leaf in (0.15, 0.5):
            hs = {arm: flb.Handle(device=0, cell_size=f["cfg"].cell_size) for arm in ("host", "device")}
            for h in hs.values():
                h.map_upload(f["map_xyz"])
            scratch = flb.Handle(device=0)
            ms = {"host": [], "device": []}
            equal, n_down = True, 0
            for k in range(args.frames):
                rng = np.random.default_rng(k)
                body = (f["scan_body"].astype(np.float64) @ flb.synth.exp_so3(rng.normal(0, 0.01, 3)).T).astype(np.float32)
                off = np.sort(rng.uniform(0.0, 100.0, len(body))).astype(np.float32)
                packed = np.concatenate([body, off[:, None]], 1)
                res = {}
                for arm in (("host", "device") if k % 2 == 0 else ("device", "host")):
                    h = hs[arm]
                    P, Cc, x_imu = product_inputs(flb, imu)
                    h.state_upload(x_imu, x_imu.copy())
                    h.synchronize()
                    t0 = time.perf_counter()
                    if arm == "host":
                        und, _ = h.imu_undistort(P, Cc, imu["v_imu"], imu["pcl_beg_time"], imu["pcl_end_time"], packed, offset_index=3)
                        h.scan_upload(scratch.voxel_grid(und, leaf))
                    else:
                        h.imu_undistort(P, Cc, imu["v_imu"], imu["pcl_beg_time"], imu["pcl_end_time"], packed, offset_index=3,
                                        download=False)
                        h.scan_from_undistorted(leaf)
                    h.synchronize()
                    t1 = time.perf_counter()
                    if k > 0:                            # the first frame warms both arms up
                        ms[arm].append(1e3 * (t1 - t0))
                    x = flb.capi.State18.from_frame(f)
                    rep = h.lio_update(prm, x, x.copy())
                    res[arm] = (h.N, h.debug_scan_order().tobytes(), bytes(x), bytes(rep))
                    n_down = h.N
                equal = equal and res["host"] == res["device"]
            for h in list(hs.values()) + [scratch]:
                h.close()
            for arm in ("host", "device"):
                v = np.array(ms[arm])
                print(json.dumps({"config": name, "raw_points": len(f["scan_body"]), "leaf": leaf, "scan_points": n_down, "arm": arm,
                                  "steps": len(v), "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                                  "ms_p90": round(float(np.percentile(v, 90)), 4), "outputs_equal": equal}), flush=True)
            assert equal, f"{name} leaf {leaf}: the two arms differ"


if __name__ == "__main__":
    main()
