"""Dense cell table vs sparse cell index at growing map extent (DESIGN.md section 8).

Maps: the C2 room alone, and the room plus four translated copies +-0.5 km and +-1.5 km away.  Modes: dense (the
automatic choice; the cell is enlarged until the table fits 2^25 cells) and sparse (flb_debug_set_map_index 2, the
configured cell).  Per case, alternating the modes round by round (median of the rounds):
  lio_fps     LIO updates/s, C2 scan placed in the far room, 3 passes, early stop off; host clock around each
              synchronous flb_lio_update, the 256 MiB L2 flush (as bench.py) outside the timed window
  knn_qps     flb_knn queries/s, 200 000 queries near the map surfaces (includes the query / result copies)
  add_ms      flb_map_add_points ms per call over a 20-frame trajectory moving between the rooms (downsample 0.3 m)
  index_mb    device bytes of the cell index
Usage: python profiles/map_extent_probe.py [--rounds 5]  (needs a GPU; writes nothing)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fastlivo_loader  # noqa: E402

DENSE, SPARSE = 1, 2


def extent_map(m, spread):
    if spread == 0:
        return m.astype(np.float32), np.zeros((1, 3), np.float32)
    offs = np.array([[0, 0, 0], [spread, 0, 0], [-spread, spread, 0], [0, -spread, 0], [spread, spread, 0]], np.float32)
    return np.concatenate([m + o for o in offs]).astype(np.float32), offs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    flb = fastlivo_loader.load()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}), flush=True)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    f = flb.synth.make_frame("C2")
    scan_w = ((f["R_true"] @ (f["R_LI"] @ f["scan_body"].T.astype(np.float64) + f["t_LI"][:, None])).T + f["p_true"]).astype(np.float32)
    lprm = flb.capi.lio_params(f, 3, early_stop=False)
    rng = np.random.default_rng(1)
    for spread in (0.0, 500.0, 1500.0):
        m, offs = extent_map(f["map_xyz"], spread)
        far = offs[-1]
        q = (m[rng.integers(0, len(m), 200000)] + rng.normal(0, 0.3, (200000, 3))).astype(np.float32)
        traj = [(scan_w + offs[k % len(offs)] + rng.normal(0, 0.05, scan_w.shape)).astype(np.float32) for k in range(20)]
        modes = [DENSE, SPARSE]
        res = {md: dict(lio=[], knn=[], add=[]) for md in modes}
        info = {}
        for r in range(args.rounds):
            for md in modes:
                h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
                h.debug_set_map_index(md)
                h.map_upload(m)
                h.scan_upload(f["scan_body"])
                info[md] = h.map_grid_info()
                x0 = flb.capi.State18.from_frame(f)
                p = np.array(x0.pos[:]) + far
                x0.pos[:] = list(p)
                for it in range(6):
                    x = x0.copy()
                    flush_buf.fill_(it & 0xff)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    h.lio_update(lprm, x, x.copy())
                    t1 = time.perf_counter()
                    if it >= 1:
                        res[md]["lio"].append(t1 - t0)
                h.knn(q[:1000])
                t0 = time.perf_counter()
                h.knn(q)
                res[md]["knn"].append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                for b in traj:
                    h.map_add_points(b, 0.3)
                res[md]["add"].append((time.perf_counter() - t0) / len(traj))
                h.close()
        for md in modes:
            i = info[md]
            print(json.dumps({"extent_m": 2 * spread, "mode": {DENSE: "dense", SPARSE: "sparse"}[md], "sparse": i["sparse"],
                              "cell_m": round(i["cell_size"], 4), "cells": i["cells"], "index_mb": round(i["index_bytes"] / 2 ** 20, 2),
                              "map_points": len(m), "lio_fps": round(1.0 / float(np.median(res[md]["lio"])), 1),
                              "knn_qps": round(len(q) / float(np.median(res[md]["knn"]))),
                              "add_ms": round(1e3 * float(np.median(res[md]["add"])), 3)}), flush=True)


if __name__ == "__main__":
    main()
