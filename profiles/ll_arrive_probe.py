"""A/B of the persistent kernels' arrival: worker sums as tagged lines the leader polls (FLB_LL_ARRIVE=1, default)
vs the arrival counter (FLB_LL_ARRIVE=0).  The switch is read once per process, so every measurement is a child
`bench.py --quick` run; the two paths alternate.  Prints device-resident frames/s (L2 flushed) and the per-pass
trace (time until the leader has every worker's sums / leader reduce + solve + publish) for C2, C3 and C4.

    python profiles/ll_arrive_probe.py [--rounds 3] [--steps 1000] [--workloads C2,C3,C4]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(workload, mode, steps):
    env = dict(os.environ, FLB_LL_ARRIVE=mode)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--quick", "--workload", workload,
                        "--steps", str(steps), "--warmup", "20"], env=env, capture_output=True, text=True, check=True)
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--workloads", default="C2,C3,C4")
    args = ap.parse_args()
    for wl in args.workloads.split(","):
        fps = {"0": [], "1": []}
        last = {}
        for _ in range(args.rounds):
            for mode in ("0", "1"):
                d = run(wl, mode, args.steps)
                fps[mode].append(d["value"])
                last[mode] = d["trace"]
        for mode, name in (("0", "counter"), ("1", "lines")):
            v = np.array(fps[mode])
            print("%s %-7s frames/s %s  median %.0f  spread %.1f%%" % (wl, name, " ".join("%.0f" % x for x in v), np.median(v),
                                                                     100 * (v.max() - v.min()) / np.median(v)))
        print("%s lines / counter (medians): %+.2f%%" % (wl, 100 * (np.median(fps["1"]) / np.median(fps["0"]) - 1)))
        for mode, name in (("0", "counter"), ("1", "lines")):
            t = last[mode]
            for k in ("lio", "vio"):
                print("  %-7s %s pass_us %s" % (name, k, t[k]["pass_us"]))
                print("  %-7s %s solve_us %s" % (name, k, t[k]["solve_us"]))


if __name__ == "__main__":
    main()
