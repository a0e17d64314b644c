"""Writes tests/golden/lidar_golden.npz: the checker's outputs (tests/oracle_pre/pre_oracle.cpp) on the synthetic driver
messages of tests/lidar_util.CASES at 1000 records, with the messages themselves, so that the suite can tell a change
of the generator from a change of the arithmetic.  Run from the repository root: python tests/golden/make_golden_lidar.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fastlivo_loader  # noqa: E402
import lidar_util  # noqa: E402
import pre_oracle  # noqa: E402

N = 1000


def main():
    flb = fastlivo_loader.load()
    out = {}
    for c in lidar_util.CASES:
        rec, fmt = lidar_util.message(flb, c, N)
        name = lidar_util.case_id(c)
        out[name + "__records"] = np.frombuffer(rec, np.uint8)
        out[name + "__cloud"] = pre_oracle.process(fmt, rec)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "lidar_golden.npz"), **out)


if __name__ == "__main__":
    main()
