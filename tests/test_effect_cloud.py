"""CPU tier: publish_effect_world's cloud (flb_effect_cloud) from the rules the device applies, compiled for the host
(tests/hostemu/effect_cloud.cpp): the byte each LIO pass leaves per point (bit 0 point_selected_surf, bit 1 "row of the
pass"), the capture of the rows in scan-index order from a Morton-ordered scan, and the RGBpointBodyToWorld transform.
Count and xyz must be byte-identical with the oracle's last-pass laserCloudOri (`Lio.last_ori`) and its
pointBodyToWorld.  The accessor (tests/effect_oracle.py) is checked too: it equals flo_lio_pass's sel_idx for passes the test drives,
and its count equals the update's n_eff_last."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_map_add_scan import morton_order, ordered_scan

import effect_oracle as eo


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "effect_cloud.cpp")
    so = str(tmp_path_factory.mktemp("effect_emu") / "libeffect_cloud.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    return C.CDLL(so)


def effect_emu(lib, out, order, body, R, p, R_LI, t_LI):
    """The device's capture + transform of one pass (out: flo_lio_pass's outputs) over the scan ordered by `order`."""
    sel = np.ascontiguousarray(out["selected"][order], np.uint8)
    pd2 = np.ascontiguousarray(out["pd2"][order], np.float32)
    b = np.zeros(len(order), np.uint8)
    lib.emu_sel_bytes(_p(sel), _p(pd2), len(order), _p(b))
    s4 = np.ascontiguousarray(ordered_scan(body, order))
    body4 = np.zeros((len(order), 4), np.float32)
    world = np.zeros((len(order), 3), np.float32)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    n = lib.emu_effect_cloud(_p(f64(R)), _p(f64(p)), _p(f64(R_LI)), _p(f64(t_LI)), _p(s4), _p(b), len(order), _p(body4), _p(world))
    return n, body4[:n], world[:n], b


def oracle_world(po, f, body, R, p):
    """pointBodyToWorld (double math, float store) of `body` with f's extrinsic, as the oracle's LIO pass exports it."""
    body = np.ascontiguousarray(body, np.float32)
    if len(body) == 0:
        return np.zeros((0, 3), np.float32)
    lio = po.Lio(body[:64].copy(), body)
    return lio.run_pass(po.lio_params(f, 1), np.asarray(R, np.float64), np.asarray(p, np.float64), True)["world"]


def check_pass(lib, po, f, lio, out, order, Rpost, ppost):
    body = np.ascontiguousarray(f["scan_body"], np.float32)
    ori = lio.last_ori()
    assert np.array_equal(ori, out["sel_idx"])                     # the accessor is the pass's laserCloudOri
    n, b4, world, _ = effect_emu(lib, out, order, body, Rpost, ppost, f["R_LI"], f["t_LI"])
    assert n == len(ori) == out["n"]
    assert b4[:, :3].tobytes() == body[ori].tobytes()
    assert b4[:, 3].view(np.int32).tolist() == ori.tolist()
    assert world.tobytes() == np.ascontiguousarray(oracle_world(po, f, body[ori], Rpost, ppost), np.float32).tobytes()
    return n


@pytest.mark.parametrize("name", ["T0", "C2"])
def test_driven_passes_match_oracle(emu, po, frames, name):
    """Three passes the test drives (kNN, then two plane-cache passes at shifted poses): after each, the device rules
    over the Morton-ordered scan give the oracle's laserCloudOri of that pass, at a later (posterior) pose."""
    f = frames(name)
    body = np.ascontiguousarray(f["scan_body"], np.float32)
    order = morton_order(body, f["cfg"].cell_size)
    assert not np.array_equal(order, np.arange(len(order)))        # the scan order differs from the caller's
    lio = eo.Lio(f["map_xyz"], body)
    assert len(lio.last_ori()) == 0                                # no pass yet
    prm = po.lio_params(f, 3)
    R0, p0 = np.asarray(f["R_prop"]), np.asarray(f["p_prop"])
    poses = [(R0, p0, True), (R0, p0 + [0.03, -0.02, 0.01], False), (np.asarray(f["R_true"]), np.asarray(f["p_true"]), False)]
    counts = []
    for R, p, rematch in poses:
        out = lio.run_pass(prm, R, p, rematch)
        counts.append(check_pass(emu, po, f, lio, out, order, f["R_true"], np.asarray(f["p_true"]) + [0.5, -0.25, 0.125]))
    assert min(counts) > len(body) // 4


@pytest.mark.parametrize("name", ["T0", "C2"])
def test_update_last_pass(po, frames, name):
    """After a whole update, the accessor's count is the report's n_eff_last, and a fresh pass overwrites it."""
    f = frames(name)
    lio = eo.Lio(f["map_xyz"], f["scan_body"])
    x = po.state_from_frame(f)
    rep = lio.update(po.lio_params(f, 4), x, x.copy())
    ori = lio.last_ori()
    assert rep.passes >= 2 and len(ori) == rep.n_eff_last > 0
    assert np.all(np.diff(ori) > 0)
    out = lio.run_pass(po.lio_params(f, 4), x.R, x.p, True)
    assert np.array_equal(lio.last_ori(), out["sel_idx"])


def far_scene():
    """A plane x = 397.9 in the world and, with identity extrinsic and pose, body points near it: one at 400 m, 2.1 m
    off the plane (s > 0.9 because |pd2| < sqrt(400) / 9, but |pd2| > 2: selected, not a row), rows at 1.1 m and 0.4 m,
    and a point far from every map point (never selected)."""
    g = np.arange(-2.0, 2.01, 0.3, dtype=np.float32)
    yy, zz = np.meshgrid(g, g)
    plane = np.stack([np.full(yy.size, 397.9, np.float32), yy.ravel(), zz.ravel()], 1)
    scan = np.array([[10.0, 3.0, 1.0], [400.0, 0.02, -0.01], [399.0, 0.05, 0.04], [398.3, -0.11, 0.12], [10.0, 50.0, 1.0]],
                    np.float32)
    f = dict(scan_body=scan, map_xyz=plane, R_LI=np.eye(3), t_LI=np.zeros(3), cfg=type("Cfg", (), {"laser_point_cov": 0.001, "cell_size": 0.6})())
    return f


def test_far_point_is_selected_but_not_a_row(emu, po):
    f = far_scene()
    order = np.array([4, 2, 0, 3, 1])
    lio = eo.Lio(f["map_xyz"], f["scan_body"])
    out = lio.run_pass(po.lio_params(f, 1), np.eye(3), np.zeros(3), True)
    assert out["selected"].tolist() == [0, 1, 1, 1, 0]
    assert abs(out["pd2"][1]) > 2.0 and abs(out["pd2"][2]) <= 2.0
    n = check_pass(emu, po, f, lio, out, order, np.eye(3), np.array([1.0, 2.0, 3.0]))
    assert n == 2 and lio.last_ori().tolist() == [2, 3]
    _, _, _, b = effect_emu(emu, out, order, f["scan_body"], np.eye(3), np.zeros(3), f["R_LI"], f["t_LI"])
    assert b.tolist() == [0, 3, 0, 3, 1]                             # selected without the row bit: the far point


def test_zero_rows(emu, po, frames):
    """A scan far from the whole map: no row, an empty cloud."""
    f = dict(frames("T0"))
    f["scan_body"] = np.ascontiguousarray(f["scan_body"] + np.float32(500.0))
    order = morton_order(f["scan_body"], f["cfg"].cell_size)
    lio = eo.Lio(f["map_xyz"], f["scan_body"])
    out = lio.run_pass(po.lio_params(f, 1), f["R_prop"], f["p_prop"], True)
    assert check_pass(emu, po, f, lio, out, order, f["R_true"], f["p_true"]) == 0


def test_sel_byte_rule(emu):
    """Bit 0 alone for selected points with |pd2| > 2 (NaN included), both bits at |pd2| <= 2, 0 when not selected."""
    pd2 = np.array([0.0, 2.0, -2.0, np.nextafter(np.float32(2.0), np.float32(3.0)), -2.5, np.nan, np.inf, 1.0], np.float32)
    for s in (0, 1):
        sel = np.full(len(pd2), s, np.uint8)
        b = np.zeros(len(pd2), np.uint8)
        emu.emu_sel_bytes(_p(sel), _p(pd2), len(pd2), _p(b))
        assert b.tolist() == ([3, 3, 3, 1, 1, 1, 1, 3] if s else [0] * len(pd2))
