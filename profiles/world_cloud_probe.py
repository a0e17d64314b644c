"""The frame's world cloud (pcl_wait_pub) through the host vs on the device: the visual-map steps of one LiDAR frame fed
from a host-built cloud against flb_world_cloud and the *_cloud calls (DESIGN.md section 8).

Per configuration (C2, C3) a visual sequence of --frames frames.  Every frame, untimed: image upload, flb_imu_undistort
of the frame's scan (dense_map_en = 1: the source is feats_undistort), state upload of the frame's posterior,
synchronise.  Then the timed step on the host clock, ending in a synchronise:
  (a) host    flb_state_download + RGBpointBodyToWorld of the undistorted cloud in numpy (float64, the reference's
              operation order) + the 0.2 m filter (flb_voxel_grid on a second handle: host in, host out, as PCL's is) +
              flb_vmap_select (enqueue-only) + flb_vmap_grow + flb_colorize
  (b) device  flb_world_cloud at the device state + flb_vmap_select_cloud (enqueue-only) + flb_vmap_grow_cloud +
              flb_colorize_cloud
Both arms take the camera pose from the device state.  The arms alternate frame by frame in one process, one handle
each, for --rounds rounds; their selections, colours and final visual-map dumps must be byte-identical.  Prints one
JSON line per configuration and arm: ms per step (median, p10, p90 over every frame of every round but the first
frame); the GPU name, power limit and maximum SM clock come from NVML in the same run.
Usage: python profiles/world_cloud_probe.py [--rounds 3] [--frames 8]  (needs a GPU; writes nothing)."""
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
from map_add_scan_probe import body_to_world, nvml_gpu  # noqa: E402

LEAF = 0.2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--grid", type=int, default=40)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    for name in ("C2", "C3"):
        seq = flb.synth.make_visual_sequence(name, args.frames)
        f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
        lprm = flb.capi.lio_params(f, 3)
        R_LI, t_LI = np.asarray(seq["R_LI"], np.float64), np.asarray(seq["t_LI"], np.float64)
        imu = flb.synth.make_imu_frame(seed=5, n_points=0)
        ms = {"host": [], "device": []}
        equal = True
        n_pts = 0
        for r in range(args.rounds):
            hs, scratch = {}, flb.Handle(device=0)
            for arm in ("host", "device"):
                h = hs[arm] = flb.Handle(device=0)
                h.camera_set(seq["cam"])
                h.image_upload(seq["frames"][0]["image"])
                h.vmap_reset(seq, grid_size=args.grid, outlier_threshold=300.0)
            for k, fr in enumerate(seq["frames"]):
                rng = np.random.default_rng(100 * r + k)
                bgr = np.ascontiguousarray(np.stack([fr["image"], np.roll(fr["image"], 3, 1), 255 - fr["image"]], -1))
                off = np.sort(rng.uniform(0.0, 100.0, len(fr["scan_body"]))).astype(np.float32)
                packed = np.concatenate([fr["scan_body"], off[:, None]], 1)
                x = flb.capi.State18.make(fr["R"] @ flb.synth.exp_so3(rng.normal(0, 0.002, 3)), fr["p"] + rng.normal(0, 0.01, 3),
                                          cov=seq["cov"])
                res = {}
                for arm in (("host", "device") if (r + k) % 2 == 0 else ("device", "host")):
                    h = hs[arm]
                    h.image_upload(fr["image"])
                    P, Cc, x_imu = product_inputs(flb, imu)
                    h.state_upload(x_imu, x_imu.copy())
                    und, _ = h.imu_undistort(P, Cc, imu["v_imu"], imu["pcl_beg_time"], imu["pcl_end_time"], packed, offset_index=3)
                    h.state_upload(x, x.copy())
                    h.synchronize()
                    t0 = time.perf_counter()
                    if arm == "host":
                        xs, _, _ = h.state_download()
                        pg = body_to_world(xs.R, xs.p, R_LI, t_LI, und)
                        pg_down = scratch.voxel_grid(pg, LEAF)
                        h.vmap_select(None, None, pg_down, blocking=False)
                        h.vmap_grow(None, None, pg, k)
                        rgb, val = h.colorize(None, None, bgr, pg)
                    else:
                        n_pts = h.world_cloud(lprm, flb.capi.CLOUD_UNDISTORTED)
                        h.vmap_select_cloud(None, None, LEAF, blocking=False)
                        h.vmap_grow_cloud(None, None, k)
                        rgb, val = h.colorize_cloud(None, None, bgr)
                    h.synchronize()
                    t1 = time.perf_counter()
                    if r > 0 or k > 0:                   # the first frame of the first round warms both arms up
                        ms[arm].append(1e3 * (t1 - t0))
                    s = h.vmap_selected()
                    res[arm] = (rgb.tobytes(), val.tobytes(), s["index"].tobytes(), s["patch"].tobytes())
                equal = equal and res["host"] == res["device"]
            da, db = hs["host"].vmap_dump(), hs["device"].vmap_dump()
            equal = equal and all(da[key].tobytes() == db[key].tobytes() for key in da)
            for h in list(hs.values()) + [scratch]:
                h.close()
        for arm in ("host", "device"):
            v = np.array(ms[arm])
            print(json.dumps({"config": name, "arm": arm, "cloud_points": n_pts, "grid": args.grid, "steps": len(v),
                              "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                              "ms_p90": round(float(np.percentile(v, 90)), 4), "outputs_equal": equal}), flush=True)
        assert equal, f"{name}: the two arms differ"


if __name__ == "__main__":
    main()
