"""The LiDAR frame with intensity on the device (DESIGN.md section 8): what carrying intensity costs through the chain,
publish_frame_world's records against the host route, and the per-frame append to pcl_wait_save_lidar.

Per message (an Avia's 24 k records, an OS1-64's 65 536 and a 32-beam Velodyne's 57 600 per spin, all from synth.py with
their intensities set), two handles, the arms alternating their order step by step, each step timed on the host clock
and ending in a device synchronise:
  chain   upload -> flb_imu_undistort_lidar (whole cloud, out_xyz = NULL) -> flb_scan_from_undistorted (leaf 0.5)
          -> flb_world_cloud(FLB_CLOUD_UNDISTORTED): (plain) through flb_lidar_upload*, (intensity) through the
          *_intensity calls.  The world clouds' xyz bytes of the two arms must be identical.
  publish (host) flb_world_cloud_download + a 48-byte PointXYZINormal cloud filled in numpy, without intensities (the
          host has none to give), against (device) flb_world_cloud_points (records with intensities);
          (save) the same on a handle with flb_lidar_save_begin open: the append's cost is (save) - (device).
Prints one JSON line per message and arm (ms per step: median, p10, p90); the GPU name, power limit and maximum SM clock
come from NVML in the same run.
Usage: python profiles/intensity_cloud_probe.py [--steps 60]  (needs a GPU; writes nothing)."""
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
from lidar_util import c_format  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402

OFF = {"livox": 16, "ouster": 16, "velodyne": 12}
CASES = [("avia_24k", "livox", 24000, 1), ("os1_64_65k", "ouster", 65536, 1), ("vlp32_57k", "velodyne", 57600, 1)]


def message(flb, kind, n, pfn):
    rec, fmt = flb.synth.make_lidar_message(kind, 1, n, point_filter_num=pfn)
    dt = {"livox": flb.synth.LIVOX_POINT, "ouster": flb.synth.OUSTER_POINT, "velodyne": flb.synth.VELODYNE_POINT}[kind]
    a = np.frombuffer(rec, dt).copy()
    rng = np.random.default_rng(3)
    if kind == "livox":
        a["reflectivity"] = rng.integers(0, 256, n)
    else:
        a["intensity"] = rng.uniform(0, 255, n).astype(np.float32)
    return np.frombuffer(a.tobytes(), np.uint8), fmt


def stats(v):
    v = np.array(v)
    return dict(steps=len(v), ms_median=round(float(np.median(v)), 4), ms_p10=round(float(np.percentile(v, 10)), 4),
                ms_p90=round(float(np.percentile(v, 90)), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    f = flb.synth.make_frame("T0")
    prm = flb.capi.lio_params(f, 3)
    fi = flb.synth.make_imu_frame(seed=5, n_points=0)
    P, Cc0, x = product_inputs(flb, fi)
    for name, kind, n, pfn in CASES:
        raw, fmt = message(flb, kind, n, pfn)
        cf = c_format(flb, fmt)
        hs = {arm: flb.Handle(device=0) for arm in ("plain", "intensity")}

        def chain(arm):
            h = hs[arm]
            h.state_upload(x, x.copy())
            Cc = type(Cc0).from_buffer_copy(bytes(Cc0))
            if arm == "plain":
                h.lidar_upload(cf, raw)
            else:
                h.lidar_upload_intensity(cf, raw, OFF[kind])
            h.imu_undistort_lidar(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9, True, download=False)
            h.scan_from_undistorted(0.5)
            m = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
            h.synchronize()
            return m

        ms = {arm: [] for arm in hs}
        for k in range(args.steps + 2):
            for arm in (("plain", "intensity") if k % 2 == 0 else ("intensity", "plain")):
                t0 = time.perf_counter()
                m = chain(arm)
                t1 = time.perf_counter()
                if k >= 2:
                    ms[arm].append(1e3 * (t1 - t0))
        assert hs["plain"].world_cloud_download().tobytes() == hs["intensity"].world_cloud_download().tobytes()
        for arm, v in ms.items():
            print(json.dumps(dict(message=name, records=n, world_points=m, step="chain", arm=arm, **stats(v))), flush=True)

        # publish_frame_world: host route vs records on the device, and the save's append
        hp = hs["intensity"]
        hsave = flb.Handle(device=0)
        hs_all = {"host": hp, "device": hp, "save": hsave}
        hsave.state_upload(x, x.copy())
        hsave.lidar_upload_intensity(cf, raw, OFF[kind])
        hsave.imu_undistort_lidar(P, type(Cc0).from_buffer_copy(bytes(Cc0)), fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], 1e9,
                                  True, download=False)
        assert hsave.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"]) == m
        hsave.lidar_save_begin(1 << 40)
        ms = {arm: [] for arm in hs_all}
        for k in range(args.steps + 2):
            order = list(hs_all) if k % 2 == 0 else list(reversed(list(hs_all)))
            for arm in order:
                h = hs_all[arm]
                t0 = time.perf_counter()
                if arm == "host":
                    xyz = h.world_cloud_download()
                    out = np.zeros(len(xyz), flb.capi.XYZINORMAL_POINT)
                    out["x"], out["y"], out["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
                    out["w"] = 1.0
                else:
                    out = h.world_cloud_points()
                h.synchronize()
                t1 = time.perf_counter()
                if k >= 2:
                    ms[arm].append(1e3 * (t1 - t0))
        for arm, v in ms.items():
            print(json.dumps(dict(message=name, world_points=m, step="publish", arm=arm, **stats(v))), flush=True)
        size = hsave.lidar_save_size()
        assert size["n"] == (args.steps + 2) * m and size["dropped"] == 0
        t0 = time.perf_counter()
        whole = hsave.lidar_save_download()
        t1 = time.perf_counter()
        assert whole[-m:].tobytes() == hp.world_cloud_points().tobytes()
        print(json.dumps(dict(message=name, save_records=size["n"], save_device_bytes=size["device_bytes"],
                              download_ms=round(1e3 * (t1 - t0), 3), download_gb_s=round(48 * size["n"] / (t1 - t0) / 1e9, 3))),
              flush=True)
        for h in (hsave, *hs.values()):
            h.close()


if __name__ == "__main__":
    main()
