"""publish_effect_world's cloud: the earlier host recipe against flb_effect_cloud (DESIGN.md section 8).

Per configuration (C2, C3) a moving trajectory of --frames frames (map_add_scan_probe's), on two handles that run the
same frames.  Every frame, untimed: scan upload and the blocking flb_lio_update from the frame's prior.  Then the timed
step on the host clock, ending in a synchronise:
  (a) recipe  flb_lio_pass (width 6, cached planes) at the posterior + flb_lio_export of sel_idx + the host select of
              the body points + RGBpointBodyToWorld in numpy (float64, the reference's operation order)
  (b) device  flb_effect_cloud at the device state + flb_effect_cloud_download
The arms alternate their order frame by frame in one process, for --rounds rounds.  Untimed, each frame also counts
whether the recipe's point set differs from laserCloudOri of the update's stop pass (the device arm's, read back in
the body frame through an identity pose and extrinsic).  Prints one JSON line per configuration and arm: ms per step
(median, p10, p90 over every frame of every round but the first frame); the GPU name, power limit and maximum SM clock
come from NVML in the same run.
Usage: python profiles/effect_cloud_probe.py [--rounds 3] [--frames 8]  (needs a GPU; writes nothing)."""
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
from map_add_scan_probe import body_to_world, nvml_gpu, trajectory  # noqa: E402


def recipe(flb, h, prm, x, body, R_LI, t_LI):
    """The earlier recipe: one more pass at the posterior, its sel_idx read back, the host select and transform."""
    h.lio_pass(prm, x.R, x.p, False, width=6, export=False)
    sel_idx = np.empty(len(body), np.int32)
    n = C.c_int()
    h._ck(h.L.flb_lio_export(h.h, None, None, None, None, None, None, None, None, sel_idx.ctypes.data_as(C.c_void_p), C.byref(n)))
    sel_idx = sel_idx[:n.value]
    return body_to_world(x.R, x.p, R_LI, t_LI, body[sel_idx]), sel_idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=8)
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    for name in ("C2", "C3"):
        f = flb.synth.make_frame(name)
        prm = flb.capi.lio_params(f, 3)
        ident = flb.capi.lio_params(dict(f, R_LI=np.eye(3), t_LI=np.zeros(3)), 3)
        R_LI, t_LI = np.asarray(f["R_LI"], np.float64), np.asarray(f["t_LI"], np.float64)
        ms = {"recipe": [], "device": []}
        differ, frames_seen, n_rows = 0, 0, []
        for r in range(args.rounds):
            traj = trajectory(flb, f, args.frames, np.random.default_rng(7 + r))
            hs = {arm: flb.Handle(device=0, cell_size=f["cfg"].cell_size) for arm in ms}
            for h in hs.values():
                h.map_upload(f["map_xyz"])
            for k, (body, x0) in enumerate(traj):
                xs = {}
                for arm in ms:
                    h = hs[arm]
                    h.scan_upload(body)
                    xs[arm] = x0.copy()
                    h.lio_update(prm, xs[arm], x0)
                    h.synchronize()
                assert bytes(xs["recipe"]) == bytes(xs["device"])
                out = {}
                for arm in (("recipe", "device") if (r + k) % 2 == 0 else ("device", "recipe")):
                    h = hs[arm]
                    t0 = time.perf_counter()
                    if arm == "recipe":
                        out[arm] = recipe(flb, h, prm, xs[arm], body, R_LI, t_LI)
                    else:
                        h.effect_cloud(prm)
                        out[arm] = h.effect_cloud_download()
                    h.synchronize()
                    t1 = time.perf_counter()
                    if r > 0 or k > 0:                   # the first frame of the first round warms both arms up
                        ms[arm].append(1e3 * (t1 - t0))
                h = hs["device"]
                h.effect_cloud(ident, np.eye(3), np.zeros(3))
                ori_body = h.effect_cloud_download()     # laserCloudOri itself, in the body frame
                differ += int(ori_body.tobytes() != np.ascontiguousarray(body[out["recipe"][1]]).tobytes())
                frames_seen += 1
                n_rows.append(len(ori_body))
            for h in hs.values():
                h.close()
        for arm in ms:
            v = np.array(ms[arm])
            print(json.dumps({"config": name, "arm": arm, "scan_points": len(f["scan_body"]), "rows_median": int(np.median(n_rows)),
                              "steps": len(v), "ms_median": round(float(np.median(v)), 4), "ms_p10": round(float(np.percentile(v, 10)), 4),
                              "ms_p90": round(float(np.percentile(v, 90)), 4), "frames": frames_seen,
                              "recipe_set_differs_frames": differ}), flush=True)


if __name__ == "__main__":
    main()
