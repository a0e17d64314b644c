"""Memory of the device visual map on a loitering run, with and without flb_vmap_reclaim.

A few C2-sized frames 0.6 m apart are rendered once and replayed back and forth with increasing frame ids (a robot
working one spot).  Every frame runs the stages of bench.py's full-frame leg (IMU undistortion, LIO update, map
maintenance, selection, VIO update, map growth, new observations, state download); the reclaim cadences are: never,
every frame, every 10 frames.  The scan feeds flb_vmap_grow on every frame, or only on the first N frames (the site
is mapped, later frames only observe it).  Prints, per run, the visual map's device bytes / slots / features against the frame
index, the host ms per frame, and the device time of one reclaim call (CUDA events) against the live points and features.

    python profiles/vmap_memory_probe.py [--frames 2000] [--workload C2] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def run(flb, torch, seq, cfg, frames, cadence, every, mapping_frames):
    from imu_util import product_inputs
    fi = flb.synth.make_imu_frame(seed=41, n_points=cfg.n_scan)
    grid = 12 if cfg.img_w <= 640 else 16
    stream = torch.cuda.Stream()
    h = flb.Handle(device=0, cell_size=cfg.cell_size)
    h.set_stream(stream.cuda_stream)
    fdict = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=cfg)
    lprm = flb.capi.lio_params(fdict, cfg.lio_passes, early_stop=False)
    vprm = flb.capi.vio_params(fdict, cfg.vio_passes, early_stop=False, force_all_passes=True)
    h.map_upload(seq["map_xyz"])
    h.camera_set(seq["cam"])
    h.image_upload(seq["frames"][0]["image"])
    h.vmap_reset(seq, grid_size=grid, outlier_threshold=300.0)
    n = len(seq["frames"])
    rows, host_ms, reclaim_us = [], [], []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for k in range(frames):
        r = k % (2 * (n - 1))
        f = seq["frames"][r if r < n else 2 * (n - 1) - r]
        body = f["scan_body"]
        packed = np.concatenate([body, fi["offset_ms"][:len(body), None]], 1).astype(np.float32)
        x0 = flb.capi.State18.make(f["R_prop"], f["p_prop"], cov=seq["cov"], grav=seq["grav"])
        t0 = time.perf_counter()
        Pg, Cg, _ = product_inputs(flb, fi)
        h.state_upload(x0, x0.copy())
        h.imu_undistort(Pg, Cg, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], packed, offset_index=3)
        h.state_upload(x0, x0.copy())
        h.scan_upload(body)
        h.lio_update_enqueue(lprm)
        h.map_add_points(f["pg"], cfg.pitch)
        h.image_upload(f["image"])
        h.vmap_select(None, None, f["pg_down"], blocking=False)
        h.vmap_grow(None, None, f["pg"] if k < mapping_frames else f["pg"][:0], k)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
        h.vmap_add_observations(None, None, k)
        timed = cadence and (k + 1) % cadence == 0 and (k + 1) % every == 0
        if cadence and (k + 1) % cadence == 0:
            if timed:
                ev0.record(stream)
            h.vmap_reclaim()
            if timed:
                ev1.record(stream)
        h.state_download()
        host_ms.append(1e3 * (time.perf_counter() - t0))
        if timed:
            ev1.synchronize()
            u = h.vmap_usage()
            reclaim_us.append(dict(frame=k, us=1e3 * ev0.elapsed_time(ev1), points=u["points"], features=u["features"]))
        if (k + 1) % every == 0 or k == 0:
            u = h.vmap_usage()
            rows.append(dict(frame=k, **u))
    h.close()
    ms = np.array(host_ms[20:])
    return dict(cadence=cadence or "never", host_ms_per_frame=dict(median=float(np.median(ms)), mean=float(ms.mean()),
                                                                    p99=float(np.percentile(ms, 99))),
                usage=rows, reclaim_device_us=reclaim_us)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--workload", default="C2")
    ap.add_argument("--render", type=int, default=4, help="rendered poses replayed back and forth")
    ap.add_argument("--every", type=int, default=100, help="usage / reclaim timing sample period (frames)")
    ap.add_argument("--mapping-frames", default="all,12",
                    help="frames whose scan feeds flb_vmap_grow (all: every frame; N: the first N, then the site is only observed)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import fastlivo_loader
    flb = fastlivo_loader.load()
    cfg = flb.synth.CONFIGS[args.workload]
    seq = flb.synth.make_visual_sequence(cfg, args.render, step=(0.6, 0.0, 0.0), yaw_step_deg=1.0, with_map=True)
    res = dict(gpu=gpu_info(), workload=args.workload, image=f"{cfg.img_w}x{cfg.img_h}", frames=args.frames, runs=[])
    for mf in args.mapping_frames.split(","):
        mapping = args.frames if mf == "all" else int(mf)
        for cadence in (0, 1, 10):
            d = run(flb, torch, seq, cfg, args.frames, cadence, args.every, mapping)
            d["mapping_frames"] = mf
            res["runs"].append(d)
            last = d["usage"][-1]
            print(f"grow fed for {mf} frames, reclaim cadence {d['cadence']}: host ms/frame median {d['host_ms_per_frame']['median']:.3f} mean {d['host_ms_per_frame']['mean']:.3f}"
                  f"  final: {last['device_bytes'] / 2**20:.1f} MiB, slots in use {last['slots_in_use']} of {last['pool_slots']}, "
                  f"features {last['features']} ({last['dead_features']} dead) of {last['feature_capacity']}, points {last['points']}", flush=True)
            for row in d["usage"]:
                print(f"   frame {row['frame']:5d}: {row['device_bytes'] / 2**20:8.1f} MiB  slots {row['slots_in_use']:5d} / {row['pool_slots']:5d}"
                      f"  free {row['free_slots']:4d}  features {row['features']:7d} dead {row['dead_features']:7d}  points {row['points']:6d}")
            for t in d["reclaim_device_us"]:
                print(f"   reclaim at frame {t['frame']:5d}: {t['us']:7.1f} us  ({t['points']} points, {t['features']} features)")
    print("gpu:", res["gpu"])
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
