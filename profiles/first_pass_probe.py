"""Profiling aid: the first pass of the LIO and the VIO kernel of a frame, cold (L2 flushed before the frame, as bench.py
does) against warm (the same frame again, nothing in between), for C2, C3 and C4.

Per workload and condition, medians over --frames traced frames of the bench's frame (state reset, LIO update, prior
:= state, VIO update; inputs resident):
  * per-pass trace of both kernels (`%globaltimer`): pass = until the leader has every worker's sums, solve = leader
    reduce + solve + publish; pass 0 of each kernel against its warm twin (the next rematch pass of the LIO, the mean
    of the later VIO passes);
  * the frame's CUDA-event time, and what the two kernels' traces do not cover (launch of each kernel to its first
    stamp, the LIO kernel's last publish to its exit, the gap between the two cooperative launches);
  * the first LIO pass alone (max_iteration 0), per worker block: kernel start -> block wake, pose ready, warps'
    compute done, sums stored; and the leader's first solve.
GPU name, power limit and SM clock from NVML in the same run.  Run from the repository root: python
profiles/first_pass_probe.py [--frames 50]."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import fastlivo_loader  # noqa: E402
import bench  # noqa: E402
from map_add_scan_probe import nvml_gpu  # noqa: E402


def sm_clock_now():
    nv = C.CDLL("libnvidia-ml.so.1")
    nv.nvmlInit_v2()
    dev = C.c_void_p()
    nv.nvmlDeviceGetHandleByIndex_v2(0, C.byref(dev))
    clk = C.c_uint()
    nv.nvmlDeviceGetClockInfo(dev, 1, C.byref(clk))                 # NVML_CLOCK_SM, current
    nv.nvmlShutdown()
    return clk.value


def trace_of(h, which):
    t = h.trace_download(which)[:63]
    t = t[:int(np.argmax(t == 0))] if (t == 0).any() else t
    t = np.concatenate([[0.0], t])
    return np.diff(t[:len(t) - (len(t) - 1) % 2])          # pass0, solve0, pass1, solve1, ...


def frames(rig, h, flush, n, cold):
    """n traced frames; per frame the (LIO, VIO) pass/solve vectors and the frame's event ms."""
    lio, vio, ms = [], [], []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(n):
        h.trace_enable(True)
        if cold:
            flush.zero_()
        e0.record(rig.stream)
        rig.enqueue_frame()
        e1.record(rig.stream)
        rig.barrier()
        lio.append(trace_of(h, 0))
        vio.append(trace_of(h, 1))
        ms.append(e0.elapsed_time(e1))
    h.trace_enable(False)
    return np.median(np.stack(lio), 0), np.median(np.stack(vio), 0), float(np.median(ms))


def first_lio_pass(f, cfg, flush, n, cold):
    """max_iteration 0: exactly one (rematch) pass; per-block stamps of it, medians over n launches (us)."""
    h = fastlivo_loader.load().Handle(cell_size=cfg.cell_size)
    h.load_frame(f)
    flb = fastlivo_loader.load()
    lprm = flb.capi.lio_params(f, 0, early_stop=False)
    x = flb.capi.State18.from_frame(f)
    h.L.flb_debug_block_stamps.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    rows = []
    for it in range(n + 1):
        h.trace_enable(True)
        h.state_upload(x, x.copy())
        h.synchronize()
        if cold:
            flush.zero_()
            torch.cuda.synchronize()
        h.lio_update_enqueue(lprm)
        h.synchronize()
        t = h.trace_download(0)
        buf = np.zeros((1024, 16), np.uint64)
        nb = C.c_int()
        h.L.flb_debug_block_stamps(h.h, buf.ctypes.data_as(C.c_void_p), 1024, C.byref(nb))
        b = buf[:nb.value - 1].astype(np.float64)
        # trace[0] (kernel start, block 0) is not downloaded in absolute time: block 0's wake is the origin
        rel = (b - b[0, 0]) * 1e-3
        w = rel[:, 4:12]
        if it:
            rows.append([np.percentile(rel[:, 0], 90), np.percentile(rel[:, 1], 90), np.percentile(w[w > -1e5], 50),
                         np.percentile(w[w > -1e5], 90), w[w > -1e5].max(), rel[:, 2].max(), t[0], t[1] - t[0]])
    h.close()
    r = np.median(np.array(rows), 0)
    keys = ["wake_p90", "pose_ready_p90", "warp_done_p50", "warp_done_p90", "warp_done_max", "stored_max",
            "all_arrived", "leader_solve"]
    return {k: round(float(v), 2) for k, v in zip(keys, r)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--workloads", default="C2,C3,C4")
    args = ap.parse_args()
    flb = fastlivo_loader.load()
    print(json.dumps(nvml_gpu()), flush=True)
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for name in args.workloads.split(","):
        cfg = flb.synth.CONFIGS[name]
        f = flb.synth.make_frame(cfg)
        h = flb.Handle(cell_size=cfg.cell_size)
        stream = torch.cuda.Stream(dev)
        torch.cuda.set_stream(stream)
        h.set_stream(stream.cuda_stream)
        rig = bench.Rig(flb, torch, cfg, f, h, dev, stream, flush=flush)
        rig.upload()
        for _ in range(10):
            rig.enqueue_frame()
        rig.barrier()
        out = {"workload": name}
        for cond in ("cold", "warm"):
            lio, vio, ms = frames(rig, h, flush, args.frames, cond == "cold")
            lp, ls, vp, vs = lio[0::2], lio[1::2], vio[0::2], vio[1::2]
            span = lio.sum() + vio.sum()
            out[cond] = {
                "frame_us": round(1e3 * ms, 2),
                "lio_pass_us": [round(float(v), 2) for v in lp], "lio_solve_us": [round(float(v), 2) for v in ls],
                "vio_pass_us": [round(float(v), 2) for v in vp], "vio_solve_us": [round(float(v), 2) for v in vs],
                "lio_span_us": round(float(lio.sum()), 2), "vio_span_us": round(float(vio.sum()), 2),
                "outside_traces_us": round(1e3 * ms - float(span), 2),
                "vio_pass0_excess_us": round(float(vp[0] + vs[0] - np.mean(vp[1:] + vs[1:len(vp)])), 2),
                "first_lio_pass": first_lio_pass(f, cfg, flush, max(5, args.frames // 5), cond == "cold"),
            }
            if len(lp) >= 3:      # pass 0 and pass 2 both rematch (kNN) passes
                out[cond]["lio_pass0_excess_us"] = round(float(lp[0] + ls[0] - lp[2] - ls[2]), 2)
        h.close()
        out["sm_clock_mhz_after"] = sm_clock_now()
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
