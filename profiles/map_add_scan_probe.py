"""map_incremental through the host vs on the device: flb_map_add_points on a host-transformed scan against
flb_map_add_scan (DESIGN.md section 8).

Per configuration (C2, C3, C4) a 20-frame trajectory: the sensor moves 5 cm and turns 0.3 degrees per frame and sees the
map's surfaces from there.  Every frame: L2 flush (256 MiB, as bench.py), scan upload, state upload, LIO update
(flb_lio_update_enqueue, 3 passes), synchronise; then the timed map step on the host clock:
  (a) host    flb_state_download + pointBodyToWorld in numpy (float64, the reference's operation order) +
              flb_map_add_points
  (b) device  flb_map_add_scan at the device posterior
The two arms alternate in the same process, one handle each, for --rounds rounds; the two maps must stay byte-identical.
Prints one JSON line per configuration and arm: ms per map step (median, p10, p90 over every frame of every round),
flb_launch_count per map step; the GPU name, power limit and maximum SM clock come from NVML in the same run.
Usage: python profiles/map_add_scan_probe.py [--rounds 5] [--ds 0.5]  (needs a GPU; writes nothing)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fastlivo_loader  # noqa: E402


def nvml_gpu():
    """Name, power limits (W) and maximum SM clock (MHz) of GPU 0 through NVML (read only)."""
    nv = C.CDLL("libnvidia-ml.so.1")
    if nv.nvmlInit_v2() != 0:
        raise RuntimeError("nvmlInit failed")
    dev = C.c_void_p()
    nv.nvmlDeviceGetHandleByIndex_v2(0, C.byref(dev))
    name = C.create_string_buffer(96)
    nv.nvmlDeviceGetName(dev, name, 96)
    lim, enf = C.c_uint(), C.c_uint()
    nv.nvmlDeviceGetPowerManagementLimit(dev, C.byref(lim))
    nv.nvmlDeviceGetEnforcedPowerLimit(dev, C.byref(enf))
    sm_max = C.c_uint()
    nv.nvmlDeviceGetMaxClockInfo(dev, 1, C.byref(sm_max))          # NVML_CLOCK_SM
    nv.nvmlShutdown()
    return dict(gpu=name.value.decode(), power_limit_w=lim.value / 1000.0, enforced_power_limit_w=enf.value / 1000.0,
                max_sm_clock_mhz=sm_max.value)


def body_to_world(R, p, R_LI, t_LI, b):
    """pointBodyToWorld (src/laserMapping.cpp:272-286) over numpy columns: double math in the reference's order, float store."""
    b = b.astype(np.float64)
    pI = [R_LI[i, 0] * b[:, 0] + R_LI[i, 1] * b[:, 1] + R_LI[i, 2] * b[:, 2] + t_LI[i] for i in range(3)]
    return np.stack([R[i, 0] * pI[0] + R[i, 1] * pI[1] + R[i, 2] * pI[2] + p[i] for i in range(3)], 1).astype(np.float32)


def trajectory(flb, f, n_frames, rng):
    R_LI, t_LI = f["R_LI"], f["t_LI"]
    world = (f["R_true"] @ (R_LI @ f["scan_body"].T.astype(np.float64) + t_LI[:, None])).T + f["p_true"]
    out = []
    for k in range(n_frames):
        Rk = f["R_true"] @ flb.synth.exp_so3(np.array([0.0, 0.0, np.deg2rad(0.3) * k]))
        pk = f["p_true"] + k * np.array([0.05, 0.0, 0.0])
        body = (R_LI.T @ (Rk.T @ (world - pk).T - t_LI[:, None])).T.astype(np.float32)
        x = flb.capi.State18.make(Rk @ flb.synth.exp_so3(rng.normal(0, 0.004, 3)), pk + rng.normal(0, 0.03, 3), f["vel"], f["bg"],
                                  f["ba"], f["grav"], f["cov"])
        out.append((body, x))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--ds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for name in ("C2", "C3", "C4"):
        f = flb.synth.make_frame(name)
        lprm = flb.capi.lio_params(f, 3)
        R_LI, t_LI = np.asarray(f["R_LI"], np.float64), np.asarray(f["t_LI"], np.float64)
        traj = trajectory(flb, f, args.frames, np.random.default_rng(1))
        ms = {"host": [], "device": []}
        launches = {"host": [], "device": []}
        equal = True
        for r in range(args.rounds):
            hs = {}
            for arm in ("host", "device"):
                hs[arm] = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
                hs[arm].map_upload(f["map_xyz"])
            for k, (body, x) in enumerate(traj):
                arms = ("host", "device") if (r + k) % 2 == 0 else ("device", "host")
                for arm in arms:
                    h = hs[arm]
                    flush_buf.fill_((r + k) & 0xFF)
                    torch.cuda.synchronize()
                    h.scan_upload(body)
                    h.state_upload(x, x.copy())
                    h.lio_update_enqueue(lprm)
                    h.synchronize()
                    l0 = h.launch_count()
                    t0 = time.perf_counter()
                    if arm == "host":
                        xs, _, _ = h.state_download()
                        h.map_add_points(body_to_world(xs.R, xs.p, R_LI, t_LI, body), args.ds)
                    else:
                        h.map_add_scan(lprm, args.ds)
                    t1 = time.perf_counter()
                    if r > 0 or k > 0:                   # the first frame of the first round warms both arms up
                        ms[arm].append(1e3 * (t1 - t0))
                        launches[arm].append(h.launch_count() - l0)
            equal = equal and hs["host"].map_download().tobytes() == hs["device"].map_download().tobytes()
            for h in hs.values():
                h.close()
        for arm in ("host", "device"):
            v = np.array(ms[arm])
            print(json.dumps({"config": name, "arm": arm, "scan_points": len(f["scan_body"]), "map_points": len(f["map_xyz"]),
                              "ds": args.ds, "steps": len(v), "ms_median": round(float(np.median(v)), 4),
                              "ms_p10": round(float(np.percentile(v, 10)), 4), "ms_p90": round(float(np.percentile(v, 90)), 4),
                              "launches_per_step": sorted(set(launches[arm])), "maps_equal": equal}), flush=True)


if __name__ == "__main__":
    main()
