"""Profiling aid: host-clock time of the point uploads (the call and a device synchronise) at 8k-40k points --
flb_scan_upload from pageable and from page-locked memory, flb_map_add_points, flb_map_upload, flb_voxel_grid and
flb_vmap_select -- so a change to the host pack and check shows beside the copy and the kernels behind it.
Prints the median and minimum over 25 calls after 5 warm-up calls, in microseconds."""
import ctypes as C
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import fastlivo_loader

flb = fastlivo_loader.load()
cp = flb.capi
L = cp.lib()
f = flb.synth.make_frame("C2")
mp = np.ascontiguousarray(f["map_xyz"], np.float32)
sc = np.ascontiguousarray(f["scan_body"], np.float32)
seq = flb.synth.make_visual_sequence("T0", 3)
fr0 = seq["frames"][0]
print("device:", torch.cuda.get_device_name(0), "map", len(mp), "scan", len(sc))


def cloud(src, n):
    return np.ascontiguousarray(np.concatenate([src + np.float32(0.01 * r) for r in range(-(-n // len(src)))])[:n])


def timed(h, call, before=None, reps=25, warm=5):
    ts = []
    for i in range(warm + reps):
        if before:
            before()
        L.flb_synchronize(h.h)
        t0 = time.perf_counter()
        rc = call()
        L.flb_synchronize(h.h)
        t1 = time.perf_counter()
        assert rc == 0, L.flb_last_error(h.h).decode()
        if i >= warm:
            ts.append((t1 - t0) * 1e6)
    return "median %8.1f  min %8.1f" % (float(np.median(ts)), float(np.min(ts)))


h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
h.map_upload(mp)
for n in (8000, 16000, 24000, 40000):
    s = cloud(sc, n)
    pin = h.pinned_like(s)
    s4 = np.ascontiguousarray(np.pad(s, ((0, 0), (0, 1))))
    add = cloud(mp, n) + np.float32(0.05)
    big = cloud(mp, n)
    print(f"n {n:6d}  scan_upload pageable  {timed(h, lambda: L.flb_scan_upload(h.h, cp._p(s), n, 3))}")
    print(f"n {n:6d}  scan_upload pinned    {timed(h, lambda: L.flb_scan_upload(h.h, cp._p(pin), n, 3))}")
    print(f"n {n:6d}  scan_upload stride 4  {timed(h, lambda: L.flb_scan_upload(h.h, cp._p(s4), n, 4))}")
    add_points = lambda: L.flb_map_add_points(h.h, cp._p(add), n, 3, C.c_float(0.5))
    print(f"n {n:6d}  map_add_points        {timed(h, add_points, before=lambda: h.map_upload(mp))}")
    print(f"n {n:6d}  map_upload            {timed(h, lambda: L.flb_map_upload(h.h, cp._p(big), n, 3))}")
    out, m = np.zeros((n, 3), np.float32), C.c_int()
    print(f"n {n:6d}  voxel_grid            "
          f"{timed(h, lambda: L.flb_voxel_grid(h.h, cp._p(s), n, 3, C.c_float(0.5), cp._p(out), n, C.byref(m)))}")
    h.map_upload(mp)
h.close()

hv = flb.Handle(device=0)
hv.camera_set(seq["cam"])
hv.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
hv.image_upload(fr0["image"])
R0, P0 = np.ascontiguousarray(fr0["Rcw"], np.float64), np.ascontiguousarray(fr0["Pcw"], np.float64)
for n in (8000, 40000):
    pg = cloud(np.ascontiguousarray(fr0["pg"], np.float32), n)
    ns = C.c_int()
    print(f"n {n:6d}  vmap_select           "
          f"{timed(hv, lambda: L.flb_vmap_select(hv.h, cp._p(R0), cp._p(P0), cp._p(pg), n, 3, C.byref(ns)))}")
hv.close()
