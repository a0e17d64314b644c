"""Helpers shared by the LiDAR message tests: the synthetic messages every tier runs, the binding's format struct, and
a scan-end pcl_offset_time that rounds below the last point's time."""
import numpy as np

CASES = [("livox", 1, 1, None), ("livox", 2, 2, None), ("livox", 3, 3, True), ("ouster", 1, 3, None), ("ouster", 2, 1, False),
         ("velodyne", 1, 3, None), ("velodyne", 2, 2, True), ("xt32", 1, 3, None), ("xt32", 2, 1, True)]   # kind, seed, filter, unsorted


def case_id(c):
    return f"{c[0]}-s{c[1]}-f{c[2]}-{'default' if c[3] is None else ('unsorted' if c[3] else 'sorted')}"


def message(flb, case, n):
    kind, seed, pfn, unsorted = case
    return flb.synth.make_lidar_message(kind, seed, n, point_filter_num=pfn, unsorted=unsorted)


def c_format(flb, fmt):
    f = flb.capi.LidarFormat()
    for k, v in fmt.items():
        setattr(f, k, v)
    return f


def scan_end_offset(lidar_beg_time, last_ms):
    """pcl_offset_time of a scan-end update, src/IMU_Processing.cpp:628-632, in the reference's own double arithmetic."""
    pcl_end_time = lidar_beg_time + float(last_ms) / 1000.0
    return pcl_end_time, (pcl_end_time - lidar_beg_time) * 1000.0


def rounding_message(flb, case, n_max, lidar_beg_time=1.7e9):
    """(records, fmt) of at most n_max records whose scan-end pcl_offset_time at lidar_beg_time falls below the last
    point's time.  At 1.7e9 s a double resolves 2.4e-7 s, so lidar_beg_time + curvature / 1000 rounds the offset to that
    grid whatever the start time is; whether it rounds down depends on the last time alone, hence the search over sizes."""
    import pre_oracle
    for n in range(n_max, max(n_max - 400, 1), -1):
        rec, fmt = message(flb, case, n)
        cloud = pre_oracle.process(fmt, rec)
        if len(cloud) > 1 and scan_end_offset(lidar_beg_time, cloud[-1, 3])[1] < float(cloud[-1, 3]):
            return rec, fmt
    raise AssertionError("no rounding case found")
