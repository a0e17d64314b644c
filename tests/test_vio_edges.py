"""CPU tier of the VIO patch guard: the oracle's and the host-compiled device math's decisions about which patches a pass
reads, on patches placed exactly at the image edges (tests/vio_edge_util.py), against the guard stated independently
from the reference's read offsets."""
import ctypes as C

import numpy as np
import pytest

import vio_edge_util as U
from conftest import bits

SCENARIOS = [(W, H, cam) for (W, H) in U.SIZES for cam in U.CAMERAS]
IDS = [f"{W}x{H}-{cam}" for (W, H, cam) in SCENARIOS]


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("W,H,cam", SCENARIOS, ids=IDS)
def test_oracle_guard_matches_expected_valid(po, W, H, cam):
    f = U.scenario(W, H, cam, depth_points=True)
    vio = po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])
    for level in (2, 1, 0):
        o = vio.run_pass(po.vio_params(f, 3), f["R_true"], f["p_true"], level)
        skipped = U.skip_set(o["H_sub"], vio.Pn)
        valid = U.expected_valid(f["cam"], f["R_true"], f["p_true"], f["patch_pos"], f["patch_level"], level)[0]
        assert (skipped == ~valid).all(), np.nonzero(skipped != ~valid)[0]
        assert o["skipped"] == skipped.sum()
        assert o["n_meas"] == 64 * valid.sum()
        assert (o["errors"][skipped] == 0).all() and (o["errors"][valid] > 0).all()


@pytest.mark.parametrize("W,H", U.SIZES, ids=[f"{W}x{H}" for W, H in U.SIZES])
def test_fixture_reaches_every_edge(W, H):
    """The fixture keeps exercising the guard: at every scale and on every side, a read patch whose footprint touches the
    image's first or last row or column (where the anchor lattice can reach it) and a skipped one that leaves the
    image by at most one tap step; anchors where the float quotient rounds up, on both sides of the guard; and every depth case."""
    touch, past, rounds = set(), set(), {True: set(), False: set()}
    for cam in U.CAMERAS:
        f = U.scenario(W, H, cam, depth_points=True)
        for level in (2, 1, 0):
            valid, box, scale, pf, pc = U.expected_valid(f["cam"], f["R_true"], f["p_true"], f["patch_pos"], f["patch_level"], level)
            front = np.isfinite(pc).all(1) & (pf[:, 2] > 0) & (np.abs(pc) < 1e6).all(1)
            for i in np.nonzero(front)[0]:
                s = int(scale[i])
                edges = {"left": (box[i, 0], 0), "right": (box[i, 1], W - 1), "top": (box[i, 2], 0), "bottom": (box[i, 3], H - 1)}
                for side, (b, lim) in edges.items():
                    if valid[i] and b == lim:
                        touch.add((s, side))
                    if not valid[i] and 0 < (b - lim if lim else lim - b) <= s:
                        past.add((s, side))
                q = pc[i] / s
                if (np.floor(np.float32(q)) != np.floor(q)).any():
                    rounds[bool(valid[i])].add(s)
            if cam == "k1":
                fold = f["kind"] == "fold"
                assert valid[fold].all() and np.hypot(*(pf[fold, :2] / pf[fold, 2:]).T) > 1.7   # 60 deg out, read inside
    for s in U.SCALES:
        for side, n in (("left", W), ("right", W), ("top", H), ("bottom", H)):
            if side in ("left", "top") or (n - 1) % s == 0:
                assert (s, side) in touch, (s, side)
            assert (s, side) in past, (s, side)
        assert s in rounds[True] and s in rounds[False], s
    pf2 = U.scenario(W, H, "pinhole", depth_points=True)
    kind = pf2["kind"]
    z = U.expected_valid(pf2["cam"], pf2["R_true"], pf2["p_true"], pf2["patch_pos"], pf2["patch_level"], 0)[3][kind == "depth", 2]
    assert (z[0] < 0) and (0 < z[1] < 1e-11) and (-1e-11 < z[2] < 0) and (0 < z[3] < 2e-3) and (0 < z[4] < 2e-7)


@pytest.mark.parametrize("W,H,cam", SCENARIOS, ids=IDS)
def test_hostemu_matches_oracle_on_edges(hostemu, po, W, H, cam):
    """vio_patch_geom and the tap lattice of flb_device.cuh, compiled for the host, at the edges: the same patches read,
    residuals and patch errors bit for bit, Jacobian rows to 1e-12."""
    f = U.scenario(W, H, cam, depth_points=True)
    vio = po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])
    c = f["cam"]
    camv = np.array([c["width"], c["height"], c["fx"], c["fy"], c["cx"], c["cy"], *c["d"]], np.float64)
    Rci, Pci = (np.ascontiguousarray(a) for a in U.extrinsics(f["R_LI"], f["t_LI"], f["Rcl"], f["Pcl"]))
    R = np.ascontiguousarray(f["R_true"], np.float64)
    p = np.ascontiguousarray(f["p_true"], np.float64)
    img = np.ascontiguousarray(f["image"])
    Pn = vio.Pn
    for level in (2, 1, 0):
        o = vio.run_pass(po.vio_params(f, 3), R, p, level)
        z, H_sub = np.empty(Pn * 64), np.empty((Pn * 64, 6))
        err, valid = np.empty(Pn, np.float32), np.empty(Pn, np.uint8)
        hostemu.emu_vio(_p(camv), _p(Rci), _p(Pci), _p(R), _p(p), _p(vio.pos), _p(vio.patch), _p(vio.level), Pn, level,
                        _p(img), _p(z), _p(H_sub), _p(err), _p(valid))
        expect = U.expected_valid(c, R, p, f["patch_pos"], f["patch_level"], level)[0]
        assert (valid.astype(bool) == expect).all(), np.nonzero(valid.astype(bool) != expect)[0]
        assert Pn - valid.sum() == o["skipped"]
        assert (bits(z) == bits(o["z"])).all()
        assert (bits(err) == bits(o["errors"])).all()
        np.testing.assert_allclose(H_sub, o["H_sub"], rtol=1e-12, atol=1e-300)


def test_update_fixture_crosses_the_guard(po):
    """The update scenarios of the GPU tier change their patch sets while they run: at every level the patches read at the
    prior differ from those read at the posterior, and the early-stop updates reject a step (the persistent kernel
    discards a speculated pass there)."""
    rejects = 0
    for W, H, cam in SCENARIOS:
        f = U.scenario(W, H, cam)
        vio = po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])
        x = po.state_from_frame(f)
        rep = vio.update(po.vio_params(f, 4), x, x.copy())
        rejects += rep.rejects
        for level in (2, 1, 0):
            a = U.expected_valid(f["cam"], f["R_prop"], f["p_prop"], f["patch_pos"], f["patch_level"], level)[0]
            b = U.expected_valid(f["cam"], x.R, x.p, f["patch_pos"], f["patch_level"], level)[0]
            assert (a != b).any(), (W, H, cam, level)
        assert np.linalg.norm(x.p - f["p_true"]) < np.linalg.norm(f["p_prop"] - f["p_true"])
    assert rejects >= 1
