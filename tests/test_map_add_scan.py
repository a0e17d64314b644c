"""CPU tier: the per-point rule of flb_map_add_scan (map_scan_point, finite3 and the bounds record's order keys in
flb_device.cuh) compiled for the host (tests/hostemu/map_add_scan.cpp).  From a Morton-ordered scan it must give the
oracle's pointBodyToWorld bit for bit, scattered back to the caller's order, and a bounds / non-finite record equal to
numpy's min / max / isfinite over the same points."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import bits


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def scan_emu(tmp_path_factory):
    """tests/hostemu/map_add_scan.cpp built for the host (into a temporary directory)."""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "map_add_scan.cpp")
    so = str(tmp_path_factory.mktemp("scan_emu") / "libmap_add_scan.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    return C.CDLL(so)


def morton_order(body, cell):
    """A Morton order of the body points (as the scan upload orders them: 2 x the map cell, anchored at the minimum)."""
    q = (np.floor((body - body.min(0)) / (2.0 * cell)).astype(np.int64)) & 0x3FF
    key = np.zeros(len(body), np.int64)
    for b in range(10):
        for k in range(3):
            key |= ((q[:, k] >> b) & 1) << (3 * b + k)
    return np.argsort(key, kind="stable")


def ordered_scan(body, order):
    """The device's ordered scan set: float4 {x, y, z, caller's index as int bits} in `order`."""
    s4 = np.zeros((len(body), 4), np.float32)
    s4[:, :3] = body[order]
    s4[:, 3] = order.astype(np.int32).view(np.float32)
    return s4


def emulate(lib, f, R, p, scan4, n_out):
    R = np.ascontiguousarray(R, np.float64)
    p = np.ascontiguousarray(p, np.float64)
    RLI = np.ascontiguousarray(f["R_LI"], np.float64)
    tLI = np.ascontiguousarray(f["t_LI"], np.float64)
    out = np.full((n_out, 3), np.nan, np.float32)
    rec = np.zeros(8, np.uint32)
    lib.emu_map_scan_world(_p(R), _p(p), _p(RLI), _p(tLI), _p(np.ascontiguousarray(scan4)), len(scan4), _p(out), _p(rec))
    lo = np.empty(3, np.float32)
    hi = np.empty(3, np.float32)
    bad = lib.emu_scan_rec_bounds(_p(rec), _p(lo), _p(hi))
    return out, lo, hi, bad


def oracle_world(po, f, R, p):
    """pointBodyToWorld of the scan as the oracle's LIO pass exports it (the map does not enter the transform)."""
    lio = po.Lio(f["map_xyz"][:64], f["scan_body"])
    return lio.run_pass(po.lio_params(f, 1), np.asarray(R, np.float64), np.asarray(p, np.float64), True)["world"]


def _rot(seed):
    q, _ = np.linalg.qr(np.random.default_rng(seed).normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


POSES = {
    "prop": lambda f: (f["R_prop"], f["p_prop"]),
    "t100m": lambda f: (f["R_prop"], f["p_prop"] + np.array([100.0, -40.0, 3.0])),
    "t1km": lambda f: (f["R_true"], f["p_true"] + np.array([1000.0, 1000.0, -20.0])),
    "rot_t250m": lambda f: (_rot(4), np.array([-250.3, 31.7, 5.1])),
}


@pytest.mark.parametrize("pose", list(POSES))
@pytest.mark.parametrize("name", ["T0", "T1", "C1", "C2"])
def test_scan_world_matches_oracle(scan_emu, po, frames, name, pose):
    f = frames(name)
    body = f["scan_body"]
    R, p = POSES[pose](f)
    want = oracle_world(po, f, R, p)
    order = morton_order(body, f["cfg"].cell_size)
    assert (order != np.arange(len(body))).any()
    got, lo, hi, bad = emulate(scan_emu, f, R, p, ordered_scan(body, order), len(body))
    assert (bits(got) == bits(want)).all()
    assert bad == 0
    assert (bits(lo) == bits(want.min(0))).all() and (bits(hi) == bits(want.max(0))).all()


def test_scan_world_any_order(scan_emu, frames):
    """The scatter makes the result independent of the order the scan set holds."""
    f = frames("T1")
    body = f["scan_body"]
    R, p = POSES["t100m"](f)
    ref = emulate(scan_emu, f, R, p, ordered_scan(body, np.arange(len(body))), len(body))
    for seed in (1, 2):
        perm = np.random.default_rng(seed).permutation(len(body))
        got = emulate(scan_emu, f, R, p, ordered_scan(body, perm), len(body))
        assert (bits(got[0]) == bits(ref[0])).all()
        assert all((bits(a) == bits(b)).all() for a, b in zip(got[1:3], ref[1:3])) and got[3] == ref[3] == 0


def test_bounds_record_matches_numpy(scan_emu, frames):
    """Points of both signs around every axis' zero and far out: the record's bounds are numpy's min / max."""
    f = frames("T0")
    rng = np.random.default_rng(5)
    body = np.concatenate([rng.uniform(-3, 3, (500, 3)), rng.uniform(-2e4, 2e4, (50, 3)),
                           rng.normal(0, 1e-3, (40, 3))]).astype(np.float32)
    fb = dict(f, scan_body=body)
    eye, zero = np.eye(3), np.zeros(3)
    fb["R_LI"], fb["t_LI"] = eye, zero
    order = rng.permutation(len(body))
    got, lo, hi, bad = emulate(scan_emu, fb, eye, zero, ordered_scan(body, order), len(body))
    assert (bits(got) == bits(body)).all() and bad == 0
    assert (bits(lo) == bits(body.min(0))).all() and (bits(hi) == bits(body.max(0))).all()


@pytest.mark.parametrize("case", ["nan_rot", "inf_pos", "overflow"])
def test_non_finite_pose_is_flagged(scan_emu, po, frames, case):
    f = frames("T0")
    R, p = np.array(f["R_prop"], np.float64), np.array(f["p_prop"], np.float64)
    if case == "nan_rot":
        R[1, 2] = np.nan
    elif case == "inf_pos":
        p[0] = np.inf
    else:
        p[2] = 1e39                     # finite in double, beyond float32 once stored
    want = oracle_world(po, f, R, p)
    body = f["scan_body"]
    got, _, _, bad = emulate(scan_emu, f, R, p, ordered_scan(body, morton_order(body, 0.6)), len(body))
    assert (~np.isfinite(want)).any()
    assert bad == 1
    assert (bits(got) == bits(want)).all()


def test_bounds_skip_non_finite_points(scan_emu, frames):
    """Some points not finite: the flag is set and the bounds cover exactly the finite ones."""
    f = frames("T0")
    rng = np.random.default_rng(8)
    body = rng.uniform(-10, 10, (300, 3)).astype(np.float32)
    body[[3, 77, 150], [0, 2, 1]] = [np.inf, -np.inf, np.nan]
    fb = dict(f, R_LI=np.eye(3), t_LI=np.zeros(3))
    got, lo, hi, bad = emulate(scan_emu, fb, np.eye(3), np.zeros(3), ordered_scan(body, rng.permutation(len(body))), len(body))
    ok = np.isfinite(got).all(1)
    assert bad == 1 and ok.sum() == len(body) - 3
    assert (bits(lo) == bits(got[ok].min(0))).all() and (bits(hi) == bits(got[ok].max(0))).all()
