"""Writes tests/golden/lidar_features_golden.npz: the checker's pl_surf and final point types
(tests/oracle_pre/feat_oracle.cpp) on small structured feature scenes of every kind, with the messages and their
formats, so that the suite can tell a change of the generator from a change of the arithmetic.
Run from the repository root: python tests/golden/make_golden_features.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import feat_oracle  # noqa: E402
from feat_util import scene  # noqa: E402

GOLDEN_SCENES = [("livox", dict(seed=21, n_cols=120), 1, 0.0), ("livox", dict(seed=22, n_cols=120), 3, 0.05),
                 ("ouster", dict(seed=21, n_scans=16, n_cols=120), 1, 0.0), ("ouster", dict(seed=22, n_scans=16, n_cols=120), 2, 0.05),
                 ("velodyne", dict(seed=21, n_scans=16, n_cols=120, timed=True, nan_returns=False), 1, 0.0),
                 ("velodyne", dict(seed=22, n_scans=16, n_cols=120, timed=False, nan_returns=False), 4, 0.05)]


def name_of(kind, kw, pf, dis_b):
    return f"{kind}-s{kw['seed']}-f{pf}-b{dis_b}"


def main():
    out = {}
    for kind, kw, pf, dis_b in GOLDEN_SCENES:
        rec, fmt = scene(kind, point_filter_num=pf, **kw)
        cloud, ftypes, _, _ = feat_oracle.process(fmt, rec, dis_b)
        assert len(cloud) > 0 and np.isfinite(cloud).all()
        name = name_of(kind, kw, pf, dis_b)
        out[name + "__records"] = np.frombuffer(rec, np.uint8)
        out[name + "__fmt"] = np.frombuffer(json.dumps(dict(fmt, dis_b=dis_b)).encode(), np.uint8)
        out[name + "__cloud"] = cloud
        out[name + "__ftypes"] = ftypes
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "lidar_features_golden.npz"), **out)


if __name__ == "__main__":
    main()
