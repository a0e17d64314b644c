"""Helpers shared by the Velodyne yaw-time tests: the synthetic spins every tier runs and the binding's format struct."""
import numpy as np

LAYOUTS = ["xyzirt", "packed22", "xyzir32"]          # synth.VELODYNE_LAYOUTS: times 0, time at 18, no time field
SIZES = {"vlp16": dict(n_scans=16, n_cols=1800), "hdl64": dict(n_scans=64, n_cols=2100)}     # 25.2 k and 130.2 k records


def spin(flb, layout, seed, pfn, size="vlp16", timed=False):
    return flb.synth.make_velodyne_spin(layout, seed, point_filter_num=pfn, timed=timed, **SIZES[size])


def c_velo_format(flb, fmt):
    f = flb.capi.VelodyneFormat()
    for k, v in fmt.items():
        setattr(f, k, v)
    return f


def lidar_format_of(fmt):
    """The flb_lidar_format of a Velodyne spin with an aligned time field (flb_lidar_upload's FLB_LIDAR_VELODYNE)."""
    return dict(kind=2, point_step=fmt["point_step"], off_x=fmt["off_x"], off_y=fmt["off_y"], off_z=fmt["off_z"],
                off_time=fmt["off_time"], off_tag=0, off_line=0, n_scans=fmt["n_scans"], point_filter_num=fmt["point_filter_num"],
                blind=fmt["blind"])


def assert_time_bound(t, t_atan2f):
    """DESIGN §2: a float ulp of atan2f (at most 2^-22 rad) moves a yaw time by at most 3.8e-6 ms, twice with yaw_fp's,
    and the time's own rounding to float adds up to an ulp of the time on each side: |dt| <= 8e-6 ms + 2 ulp(t).  It holds
    only while no such ulp flips a wrap or a `yaw <= yaw_fp` decision, which the spins the tests run never do."""
    d = np.abs(t.astype(np.float64) - t_atan2f.astype(np.float64))
    assert (d <= 8e-6 + 2 * np.spacing(np.abs(t)).astype(np.float64)).all(), d.max()
