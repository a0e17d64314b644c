"""TEST INFRASTRUCTURE -- the feature scenes shared by the CPU and GPU tests of flb_lidar_upload_features."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "fast-livo_b200"))
import synth  # noqa: E402

# (kind, options) of every scene; each runs with point_filter_num 1..4 and dis_b 0 and 0.05
SCENES = [
    ("livox", dict(seed=1)),
    ("livox", dict(seed=2, n_cols=250)),
    ("ouster", dict(seed=1)),
    ("ouster", dict(seed=2, n_scans=32, n_cols=400)),
    ("velodyne", dict(seed=1, timed=True)),
    ("velodyne", dict(seed=2, timed=False)),
    ("velodyne", dict(seed=3, n_scans=32, n_cols=300, timed=False, nan_returns=False)),
    ("velodyne", dict(seed=4, timed=True, nan_returns=False)),
]
FILTERS = (1, 2, 3, 4)
DIS_B = (0.0, 0.05)


def scene(kind, point_filter_num=1, **kw):
    return synth.make_feature_scan(kind, point_filter_num=point_filter_num, **kw)
