"""Writes tests/golden/velodyne_golden.npz: the checker's outputs (tests/oracle_pre/velo_oracle.cpp, the defined yaw) on
small synthetic Velodyne spins without per-point times (16 rings x 60 columns) in every layout, with the spins
themselves, so that the suite can tell a change of the generator from a change of the arithmetic.  No committed spin may
hold a record whose double atan2 lies within a few double ulps of a float rounding midpoint: there another conforming
atan2 could round the yaw the other way.  Run from the repository root: python tests/golden/make_golden_velodyne.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fastlivo_loader  # noqa: E402
import velo_oracle  # noqa: E402
from velo_util import LAYOUTS  # noqa: E402


def main():
    flb = fastlivo_loader.load()
    out = {}
    for layout in LAYOUTS:
        for seed, pfn in ((1, 1), (2, 3)):
            rec, fmt = flb.synth.make_velodyne_spin(layout, seed, point_filter_num=pfn, n_scans=16, n_cols=60)
            assert not velo_oracle.midpoint_flags(fmt, rec).any(), (layout, seed)
            cloud, yaw_times = velo_oracle.process(fmt, rec)
            assert yaw_times and np.isfinite(cloud).all()
            name = f"{layout}-s{seed}-f{pfn}"
            out[name + "__records"] = np.frombuffer(rec, np.uint8)
            out[name + "__cloud"] = cloud
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "velodyne_golden.npz"), **out)


if __name__ == "__main__":
    main()
