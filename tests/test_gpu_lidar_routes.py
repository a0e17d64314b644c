"""GPU tier: the four LiDAR message uploads pinned to fixed values.  One handle runs a sequence of messages through
flb_lidar_upload, flb_lidar_upload_velodyne, flb_lidar_upload_features and flb_lidar_upload_velodyne_features: every
decode route (the handlers' own times, the Velodyne yaw times, the feature branches), clouds whose times need the
re-sort, the refusals that come back after device work (a bad ring, a kept point that is not finite), empty and fully
filtered messages, and format refusals with one and with two faults.  After every call it records the return code,
the error text, the outputs, the launch count and the current cloud, so a refusal also pins the cloud it left in place.
The other LiDAR tests compare clouds against the checker; this one catches any change to the launches, the messages
and the order in which the checks run."""
import hashlib
import json
import os

import numpy as np
import pytest

from feat_util import scene
from lidar_util import c_format
from velo_util import c_velo_format, spin

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
UNSET = -7                                   # the outputs before the call: a refusal leaves them as they are


def with_field(rec, fmt, n, off, value, dtype, rows):
    """The records with `value` (as dtype) written at byte offset `off` of the given rows."""
    a = np.frombuffer(rec, np.uint8).reshape(n, fmt["point_step"]).copy()
    for r in rows:
        a[r, off:off + np.dtype(dtype).itemsize] = np.frombuffer(np.array(value, dtype).tobytes(), np.uint8)
    return a.tobytes()


def velo_of(fmt):
    """flb_velodyne_format's fields of a make_feature_scan Velodyne message."""
    return dict(point_step=fmt["point_step"], off_x=fmt["off_x"], off_y=fmt["off_y"], off_z=fmt["off_z"],
                off_time=fmt["off_time"], off_ring=fmt["off_line"], n_scans=fmt["n_scans"],
                point_filter_num=fmt["point_filter_num"], blind=fmt["blind"])


def cases(flb):
    """[(label, call, fmt dict, records bytes or None, n_records, dis_b, pinned)] in the order they run."""
    out = []

    def add(label, call, fmt, rec, n=None, dis_b=0.0, pinned=False):
        if n is None:
            n = len(rec) // fmt["point_step"]
        out.append((label, call, fmt, rec, n, dis_b, pinned))

    # flb_lidar_upload: every handler, both filters, the re-sort, and the refusals
    for kind, seed, pfn, unsorted in (("livox", 1, 1, None), ("livox", 2, 2, None), ("ouster", 1, 3, None), ("velodyne", 1, 3, None),
                                      ("xt32", 1, 3, None), ("livox", 3, 3, True), ("velodyne", 2, 2, True), ("xt32", 2, 1, True)):
        rec, fmt = flb.synth.make_lidar_message(kind, seed, 3000, point_filter_num=pfn, unsorted=unsorted)
        add(f"plain-{kind}-s{seed}-f{pfn}-{'unsorted' if unsorted else 'default'}", "plain", fmt, rec, pinned=seed == 2)
    rec, fmt = flb.synth.make_lidar_message("ouster", 4, 3000, point_filter_num=1)
    add("plain-ouster-inf", "plain", fmt, with_field(rec, fmt, 3000, fmt["off_x"], np.inf, np.float32, range(100, 140)))
    add("plain-empty", "plain", fmt, None, 0)
    add("plain-all-in-blind", "plain", dict(fmt, blind=1e4), rec)
    rec, fmt = flb.synth.make_lidar_message("velodyne_notime", 1, 3000)
    add("plain-velodyne-without-times", "plain", fmt, rec)
    rec, fmt = flb.synth.make_lidar_message("livox", 5, 3000, point_filter_num=1)
    add("plain-livox", "plain", fmt, rec)
    for label, bad in (("kind", dict(kind=5)), ("kind+filter", dict(kind=0, point_filter_num=0)), ("nscans", dict(n_scans=0)),
                       ("filter+misaligned", dict(point_filter_num=0, off_x=2)), ("misaligned", dict(off_y=6)),
                       ("time-past-step", dict(off_time=fmt["point_step"] - 2)), ("blind+line", dict(blind=np.nan, off_line=99))):
        add(f"plain-refuse-{label}", "plain", dict(fmt, **bad), rec)
    add("plain-refuse-no-records", "plain", fmt, None, 10)

    # flb_lidar_upload_velodyne: the yaw route in two layouts, the time route, and the refusals
    for layout, seed, pfn, timed in (("xyzirt", 1, 1, False), ("packed22", 2, 2, False), ("xyzir32", 3, 3, False), ("xyzirt", 5, 1, True)):
        rec, fmt = spin(flb, layout, seed, pfn, timed=timed)
        add(f"velo-{layout}-s{seed}-f{pfn}-{'timed' if timed else 'yaw'}", "velo", fmt, rec, pinned=seed == 2)
    rec, fmt = spin(flb, "xyzirt", 7, 1)
    n = len(rec) // fmt["point_step"]
    add("velo-bad-ring", "velo", fmt, with_field(rec, fmt, n, fmt["off_ring"], 16, np.uint16, (5000, 9000)))
    x = np.frombuffer(rec, np.uint8).reshape(n, fmt["point_step"])[:, fmt["off_x"]:fmt["off_x"] + 4].copy().view(np.float32)[:, 0]
    k = next(i for i in range(1000, 2000) if np.isfinite(x[i]))
    add("velo-inf", "velo", fmt, with_field(rec, fmt, n, fmt["off_x"], np.inf, np.float32, (k,)))
    add("velo-empty", "velo", fmt, None, 0)
    add("velo-all-in-blind", "velo", dict(fmt, blind=1e4), rec)
    add("velo-yaw", "velo", fmt, rec)
    for label, bad in (("filter", dict(point_filter_num=0)), ("nscans+x", dict(n_scans=0, off_x=fmt["point_step"])),
                       ("ring", dict(off_ring=fmt["point_step"] - 1)), ("time", dict(off_time=-2)), ("step+blind", dict(point_step=0))):
        add(f"velo-refuse-{label}", "velo", dict(fmt, **bad), rec, n)

    # flb_lidar_upload_features: Livox and Ouster, the committed goldens, and the refusals
    z = np.load(os.path.join(HERE, "golden", "lidar_features_golden.npz"))
    goldens = {}
    for name in sorted({k.split("__")[0] for k in z.files}):
        gf = json.loads(bytes(z[name + "__fmt"]).decode())
        goldens[name] = (gf.pop("dis_b"), gf, z[name + "__records"].tobytes())
    for kind in ("livox", "ouster"):
        rec, fmt = scene(kind, seed=1)
        add(f"feat-{kind}", "feat", fmt, rec, pinned=kind == "ouster")
        for name, (dis_b, gf, grec) in goldens.items():
            if name.startswith(kind):
                add(f"feat-golden-{name}", "feat", gf, grec, dis_b=dis_b)
        add(f"feat-{kind}-empty", "feat", fmt, None, 0)
        add(f"feat-{kind}-all-in-blind", "feat", dict(fmt, blind=1e4), rec)
    rec, fmt = scene("livox", seed=2, n_cols=250)
    n = len(rec) // fmt["point_step"]
    add("feat-livox-inf", "feat", fmt, with_field(rec, fmt, n, fmt["off_x"], np.inf, np.float32, range(600, 640)))
    add("feat-livox", "feat", fmt, rec)
    for label, bad, dis_b in (("dis_b", {}, np.nan), ("dis_b+kind", dict(kind=7), np.inf), ("velodyne", dict(kind=2), 0.0),
                              ("xt32+filter", dict(kind=4, point_filter_num=0), 0.0), ("kind", dict(kind=0), 0.0),
                              ("nscans", dict(n_scans=129), 0.0), ("filter+line", dict(point_filter_num=0, off_line=999), 0.0),
                              ("line", dict(off_line=fmt["point_step"]), 0.0), ("time", dict(off_time=2), 0.0)):
        add(f"feat-refuse-{label}", "feat", dict(fmt, **bad), rec, dis_b=dis_b)

    # flb_lidar_upload_velodyne_features: timed and yaw, the goldens, and the refusals
    for label, kw in (("timed", dict(seed=4, timed=True, nan_returns=False)),
                      ("yaw", dict(seed=3, n_scans=32, n_cols=300, timed=False, nan_returns=False)),
                      ("nan-returns", dict(seed=1, timed=True))):
        rec, fmt = scene("velodyne", **kw)
        add(f"vfeat-{label}", "vfeat", velo_of(fmt), rec, pinned=label == "yaw")
    for name, (dis_b, gf, grec) in goldens.items():
        if name.startswith("velodyne"):
            add(f"vfeat-golden-{name}", "vfeat", velo_of(gf), grec, dis_b=dis_b)
    rec, fmt = scene("velodyne", seed=8, nan_returns=False)
    n = len(rec) // fmt["point_step"]
    vf = velo_of(fmt)
    add("vfeat-inf", "vfeat", vf, with_field(rec, fmt, n, fmt["off_x"], np.inf, np.float32, range(3000, 3040)))
    add("vfeat-empty", "vfeat", vf, None, 0)
    add("vfeat-all-in-blind", "vfeat", dict(vf, blind=1e4), rec)
    add("vfeat", "vfeat", vf, rec)
    for label, bad, dis_b in (("nscans", dict(n_scans=129), 0.0), ("nscans+x", dict(n_scans=129, off_x=-1), 0.0),
                              ("dis_b+filter", dict(point_filter_num=0), np.nan), ("ring", dict(off_ring=fmt["point_step"] - 1), 0.0),
                              ("time", dict(off_time=-3), 0.0)):
        add(f"vfeat-refuse-{label}", "vfeat", dict(vf, **bad), rec, dis_b=dis_b)
    return out


def run_routes(flb):
    """[(label, rc, error text or None, n_points, last_offset_ms bits, yaw_times, launches, cloud size, cloud digest)]."""
    C = flb.capi.C
    L = flb.capi.lib()
    h = flb.Handle(device=0)
    out = []
    for label, call, fmt, rec, n, dis_b, pinned in cases(flb):
        if rec is None:
            ptr = None
        else:
            a = np.frombuffer(rec, np.uint8)
            if pinned:
                a = h.pinned_like(a)
            ptr = a.ctypes.data
        np_out, last, yaw = C.c_int(UNSET), C.c_float(UNSET), C.c_int(UNSET)
        f = (c_format if call in ("plain", "feat") else c_velo_format)(flb, fmt)
        l0 = h.launch_count()
        if call == "plain":
            rc = L.flb_lidar_upload(h.h, C.byref(f), ptr, n, C.byref(np_out), C.byref(last))
        elif call == "velo":
            rc = L.flb_lidar_upload_velodyne(h.h, C.byref(f), ptr, n, C.byref(np_out), C.byref(last), C.byref(yaw))
        elif call == "feat":
            rc = L.flb_lidar_upload_features(h.h, C.byref(f), float(dis_b), ptr, n, C.byref(np_out), C.byref(last))
        else:
            rc = L.flb_lidar_upload_velodyne_features(h.h, C.byref(f), float(dis_b), ptr, n, C.byref(np_out), C.byref(last),
                                                      C.byref(yaw))
        launches = h.launch_count() - l0
        err = L.flb_last_error(h.h).decode() if rc else None
        cloud = h.lidar_download()
        last_bits = int(np.float32(last.value).view(np.uint32))
        out.append((label, rc, err, np_out.value, last_bits, yaw.value, launches, len(cloud),
                    hashlib.sha256(cloud.tobytes()).hexdigest()[:16]))
    h.close()
    return out


EXPECTED = [    # recorded on an NVIDIA H100 80GB HBM3 (700 W power limit); (label, rc, error, n_points, last_offset_ms bits,
                #  yaw_times, launches, cloud size, cloud digest), UNSET where the call left an output alone
    ('plain-livox-s1-f1-default', 0, None, 2280, 1095211425, -7, 6, 2280, '88d79c46e1e09b10'),
    ('plain-livox-s2-f2-default', 0, None, 1186, 1095211425, -7, 6, 1186, 'e861e32857f31e4a'),
    ('plain-ouster-s1-f3-default', 0, None, 939, 1075151479, -7, 7, 939, 'd11a8a289cbcdf51'),
    ('plain-velodyne-s1-f3-default', 0, None, 941, 925741376, -7, 4, 941, '291bc67ea7e6e520'),
    ('plain-xt32-s1-f3-default', 0, None, 931, 1084643824, -7, 4, 931, 'fd91c3a1665b29a9'),
    ('plain-livox-s3-f3-unsorted', 0, None, 778, 1095211425, -7, 9, 778, 'e4ce3075d7727f34'),
    ('plain-velodyne-s2-f2-unsorted', 0, None, 1414, 925746442, -7, 7, 1414, '9d909ab612a7c45f'),
    ('plain-xt32-s2-f1-unsorted', 0, None, 2824, 1051723392, -7, 7, 2824, '2675d7660ac1c6bb'),
    ('plain-ouster-inf', -1, 'flb_lidar_upload: a kept point or time is not finite', -7, 3235905536, -7, 4, 2824, '2675d7660ac1c6bb'),
    ('plain-empty', 0, None, 0, 0, -7, 0, 0, 'e3b0c44298fc1c14'),
    ('plain-all-in-blind', 0, None, 0, 0, -7, 4, 0, 'e3b0c44298fc1c14'),
    ('plain-velodyne-without-times', -1, 'flb_lidar_upload: a Velodyne cloud without per-point times (last time 0): its times come from the yaw angle (src/preprocess.cpp:389-419), which flb_lidar_upload_velodyne derives', -7, 3235905536, -7, 0, 0, 'e3b0c44298fc1c14'),
    ('plain-livox', 0, None, 2284, 1095211425, -7, 6, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-kind', -1, 'flb_lidar_upload: unknown kind 5', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-kind+filter', -1, 'flb_lidar_upload: unknown kind 0', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-nscans', -1, 'flb_lidar_upload: point_filter_num 1, n_scans 0, blind 0.5', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-filter+misaligned', -1, 'flb_lidar_upload: point_filter_num 0, n_scans 6, blind 0.5', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-misaligned', -1, 'flb_lidar_upload: a field does not fit in point_step 20 or is not aligned to its type', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-time-past-step', -1, 'flb_lidar_upload: a field does not fit in point_step 20 or is not aligned to its type', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-blind+line', -1, 'flb_lidar_upload: point_filter_num 1, n_scans 6, blind nan', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('plain-refuse-no-records', -1, 'flb_lidar_upload: bad arguments', -7, 3235905536, -7, 0, 2284, 'a1dfa0dcd61e0d06'),
    ('velo-xyzirt-s1-f1-yaw', 0, None, 23648, 1128755288, 1, 11, 23648, '7fa98c7c1e00aa60'),
    ('velo-packed22-s2-f2-yaw', 0, None, 11850, 1128755714, 1, 11, 11850, 'f2879e717cac3310'),
    ('velo-xyzir32-s3-f3-yaw', 0, None, 7881, 1128754042, 1, 11, 7881, '6211dcc7d6bf2fcc'),
    ('velo-xyzirt-s5-f1-timed', 0, None, 23646, 953200435, 0, 4, 23646, '163b7b631e2f4c40'),
    ('velo-bad-ring', -1, 'flb_lidar_upload_velodyne: record 5000 has ring 16 >= n_scans 16 (the per-ring yaw state has no such ring)', -7, 3235905536, -7, 8, 23646, '163b7b631e2f4c40'),
    ('velo-inf', -1, 'flb_lidar_upload_velodyne: a kept point or time is not finite', -7, 3235905536, -7, 8, 23646, '163b7b631e2f4c40'),
    ('velo-empty', 0, None, 0, 0, 0, 0, 0, 'e3b0c44298fc1c14'),
    ('velo-all-in-blind', 0, None, 0, 0, 1, 8, 0, 'e3b0c44298fc1c14'),
    ('velo-yaw', 0, None, 23671, 1128755673, 1, 11, 23671, 'e6dda7e635b2c3c1'),
    ('velo-refuse-filter', -1, 'flb_lidar_upload_velodyne: point_filter_num 0, n_scans 16, blind 1', -7, 3235905536, -7, 0, 23671, 'e6dda7e635b2c3c1'),
    ('velo-refuse-nscans+x', -1, 'flb_lidar_upload_velodyne: point_filter_num 1, n_scans 0, blind 1', -7, 3235905536, -7, 0, 23671, 'e6dda7e635b2c3c1'),
    ('velo-refuse-ring', -1, 'flb_lidar_upload_velodyne: a field does not fit in point_step 24', -7, 3235905536, -7, 0, 23671, 'e6dda7e635b2c3c1'),
    ('velo-refuse-time', -1, 'flb_lidar_upload_velodyne: a field does not fit in point_step 24', -7, 3235905536, -7, 0, 23671, 'e6dda7e635b2c3c1'),
    ('velo-refuse-step+blind', -1, 'flb_lidar_upload_velodyne: a field does not fit in point_step 0', -7, 3235905536, -7, 0, 23671, 'e6dda7e635b2c3c1'),
    ('feat-livox', 0, None, 432, 1090838682, -7, 46, 432, 'ef03769b7902fe8e'),
    ('feat-golden-livox-s21-f1-b0.0', 0, None, 346, 1075682528, -7, 44, 346, '18e4ba7f1aae3c64'),
    ('feat-golden-livox-s22-f3-b0.05', 0, None, 137, 1075560185, -7, 44, 137, 'fad05561ec160109'),
    ('feat-livox-empty', 0, None, 0, 0, -7, 0, 0, 'e3b0c44298fc1c14'),
    ('feat-livox-all-in-blind', 0, None, 0, 0, -7, 6, 0, 'e3b0c44298fc1c14'),
    ('feat-ouster', 0, None, 12823, 1103576475, -7, 52, 12823, '817b49cadc76ba9e'),
    ('feat-golden-ouster-s21-f1-b0.0', 0, None, 1112, 1094316368, -7, 46, 1112, '92a38bed4fec2d8a'),
    ('feat-golden-ouster-s22-f2-b0.05', 0, None, 577, 1094213968, -7, 46, 577, '24fd964d5fe53e53'),
    ('feat-ouster-empty', 0, None, 0, 0, -7, 0, 0, 'e3b0c44298fc1c14'),
    ('feat-ouster-all-in-blind', 0, None, 0, 0, -7, 6, 0, 'e3b0c44298fc1c14'),
    ('feat-livox-inf', -1, 'flb_lidar_upload_features: a point of pl_surf or its time is not finite', -7, 3235905536, -7, 43, 0, 'e3b0c44298fc1c14'),
    ('feat-livox', 0, None, 448, 1084534288, -7, 46, 448, 'c48280a0a57a3515'),
    ('feat-refuse-dis_b', -1, 'flb_lidar_upload_features: bad arguments', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-dis_b+kind', -1, 'flb_lidar_upload_features: bad arguments', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-velodyne', -1, 'flb_lidar_upload_features: kind 2: a Velodyne cloud goes to flb_lidar_upload_velodyne_features; the XT32 has no feature branch (src/preprocess.cpp:432-464), so flb_lidar_upload serves it', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-xt32+filter', -1, 'flb_lidar_upload_features: kind 4: a Velodyne cloud goes to flb_lidar_upload_velodyne_features; the XT32 has no feature branch (src/preprocess.cpp:432-464), so flb_lidar_upload serves it', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-kind', -1, 'flb_lidar_upload_features: unknown kind 0', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-nscans', -1, 'flb_lidar_upload_features: point_filter_num 1, n_scans 129 (1..128: pl_buff[128]), blind 0.5', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-filter+line', -1, 'flb_lidar_upload_features: point_filter_num 0, n_scans 6 (1..128: pl_buff[128]), blind 0.5', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-line', -1, 'flb_lidar_upload_features: a field does not fit in point_step 20 or is not aligned to its type', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('feat-refuse-time', -1, 'flb_lidar_upload_features: a field does not fit in point_step 20 or is not aligned to its type', -7, 3235905536, -7, 0, 448, 'c48280a0a57a3515'),
    ('vfeat-timed', 0, None, 4550, 936409382, 0, 50, 4550, '0078102151168b0f'),
    ('vfeat-yaw', 0, None, 7413, 1128748786, 1, 54, 7413, 'd0d1ceb99436fe5b'),
    ('vfeat-nan-returns', -1, 'flb_lidar_upload_velodyne_features: a point of pl_surf or its time is not finite', -7, 3235905536, -7, 47, 7413, 'd0d1ceb99436fe5b'),
    ('vfeat-golden-velodyne-s21-f1-b0.0', 0, None, 1086, 920482461, 0, 46, 1086, '6c9d2c970b1a6471'),
    ('vfeat-golden-velodyne-s22-f4-b0.05', 0, None, 302, 1128741951, 1, 48, 302, '26794c2de7bbbef9'),
    ('vfeat-inf', -1, 'flb_lidar_upload_velodyne_features: a point of pl_surf or its time is not finite', -7, 3235905536, -7, 47, 302, '26794c2de7bbbef9'),
    ('vfeat-empty', 0, None, 0, 0, 0, 0, 0, 'e3b0c44298fc1c14'),
    ('vfeat-all-in-blind', 0, None, 0, 0, 0, 47, 0, 'e3b0c44298fc1c14'),
    ('vfeat', 0, None, 4587, 936397981, 0, 50, 4587, 'f71a242452cee50f'),
    ('vfeat-refuse-nscans', -1, 'flb_lidar_upload_velodyne_features: point_filter_num 1, n_scans 129 (1..128: pl_buff[128]), blind 1', -7, 3235905536, -7, 0, 4587, 'f71a242452cee50f'),
    ('vfeat-refuse-nscans+x', -1, 'flb_lidar_upload_velodyne_features: point_filter_num 1, n_scans 129 (1..128: pl_buff[128]), blind 1', -7, 3235905536, -7, 0, 4587, 'f71a242452cee50f'),
    ('vfeat-refuse-dis_b+filter', -1, 'flb_lidar_upload_velodyne_features: bad arguments', -7, 3235905536, -7, 0, 4587, 'f71a242452cee50f'),
    ('vfeat-refuse-ring', -1, 'flb_lidar_upload_velodyne_features: a field does not fit in point_step 24', -7, 3235905536, -7, 0, 4587, 'f71a242452cee50f'),
    ('vfeat-refuse-time', -1, 'flb_lidar_upload_velodyne_features: a field does not fit in point_step 24', -7, 3235905536, -7, 0, 4587, 'f71a242452cee50f'),
]


def test_routes_pinned(flb):
    got = run_routes(flb)
    assert len(got) == len(EXPECTED)
    for g, e in zip(got, EXPECTED):
        assert g == e, g[0]
