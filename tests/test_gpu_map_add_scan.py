"""GPU tier: flb_map_add_scan (map_incremental from the uploaded scan and the device posterior).  Every test compares
handle A, which calls map_add_scan, with handle B, which holds the same map and calls map_add_points on the oracle's
pointBodyToWorld of the same scan at the same pose: the map bytes and order, the grid and everything computed on the
map afterwards must be identical, on each of Add_Points' three internal paths."""
import os

import numpy as np
import pytest

from conftest import bits

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4


def oracle_world(po, f, body, R, p):
    """pointBodyToWorld (double math, float store) of `body` as the oracle's LIO pass exports it."""
    lio = po.Lio(f["map_xyz"][:64], body)
    return lio.run_pass(po.lio_params(f, 1), np.asarray(R, np.float64), np.asarray(p, np.float64), True)["world"]


def pair(flb, f, index_mode=0, scan=True):
    hs = []
    for _ in range(2):
        h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
        if index_mode:
            h.debug_set_map_index(index_mode)
        h.map_upload(f["map_xyz"])
        if scan:
            h.scan_upload(f["scan_body"])
        hs.append(h)
    return hs


def assert_same_map(a, b):
    ma, mb = a.map_download(), b.map_download()
    assert ma.shape == mb.shape and ma.tobytes() == mb.tobytes()
    assert a.map_grid_info() == b.map_grid_info()


def assert_same_after(flb, f, a, b):
    """kNN and a following LIO update on the two maps agree to the bit."""
    rng = np.random.default_rng(2)
    m = a.map_download()
    q = (m[rng.integers(0, len(m), 3000)] + rng.normal(0, 0.2, (3000, 3))).astype(np.float32)
    ia, da = a.knn(q)
    ib, db = b.knn(q)
    assert (ia == ib).all() and (bits(da) == bits(db)).all()
    prm = flb.capi.lio_params(f, 3)
    xa, xb = flb.capi.State18.from_frame(f), flb.capi.State18.from_frame(f)
    ra = a.lio_update(prm, xa, xa.copy())
    rb = b.lio_update(prm, xb, xb.copy())
    assert bytes(xa) == bytes(xb) and bytes(ra) == bytes(rb)


@pytest.mark.parametrize("pose", ["lio_update", "lio_update_enqueue", "explicit"])
@pytest.mark.parametrize("ds", [0.3, 0.5])
@pytest.mark.parametrize("name", ["T0", "T1", "C2"])
def test_map_equals_host_path(flb, po, frames, name, ds, pose):
    f = frames(name)
    a, b = pair(flb, f)
    prm = flb.capi.lio_params(f, 3)
    if pose == "lio_update":
        x = flb.capi.State18.from_frame(f)
        a.lio_update(prm, x, x.copy())
        a.map_add_scan(prm, ds)
        R, p = x.R, x.p
    elif pose == "lio_update_enqueue":
        x = flb.capi.State18.from_frame(f)
        a.state_upload(x, x.copy())
        a.lio_update_enqueue(prm)
        a.map_add_scan(prm, ds)                     # no synchronise in between: stream order
        x, _, _ = a.state_download()
        R, p = x.R, x.p
    else:
        R, p = f["R_true"], f["p_true"]
        a.map_add_scan(prm, ds, R, p)
    b.map_add_points(oracle_world(po, f, f["scan_body"], R, p), ds)
    assert_same_map(a, b)
    assert_same_after(flb, f, a, b)
    a.close()
    b.close()


# (index mode, pose offset from the true pose): dense incremental, full rebuild (the scan leaves the grid box), sparse index
PATHS = {"dense_incremental": (0, (0.0, 0.0, 0.0)), "full_rebuild": (0, (45.0, -30.0, 2.0)),
         "sparse": (2, (0.0, 0.0, 0.0)), "sparse_far": (2, (40.0, 0.0, 0.0)), "sparse_km": (2, (1500.0, -800.0, 10.0))}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("name", ["T1", "C2"])
def test_every_path_and_launch_count(flb, po, frames, name, path):
    mode, off = PATHS[path]
    f = frames(name)
    a, b = pair(flb, f, mode)
    prm = flb.capi.lio_params(f, 3)
    R, p = f["R_true"], f["p_true"] + np.array(off)
    ds = 0.4
    before = a.map_grid_info()
    la = a.launch_count()
    a.map_add_scan(prm, ds, R, p)
    la = a.launch_count() - la
    lb = b.launch_count()
    b.map_add_points(oracle_world(po, f, f["scan_body"], R, p), ds)
    lb = b.launch_count() - lb
    after = a.map_grid_info()
    assert la == lb + 1
    if path == "dense_incremental":
        assert not after["sparse"] and after["cells"] == before["cells"]      # the grid box did not change
    elif path == "full_rebuild":
        assert not after["sparse"] and after["cells"] != before["cells"]      # rebuilt over a larger box
    else:
        assert after["sparse"] == 1
    assert_same_map(a, b)
    assert_same_after(flb, f, a, b)
    a.close()
    b.close()


def test_trajectory_c2(flb, po, frames):
    """20 frames of scan upload -> LIO update -> map_add_scan on a moving C2 trajectory: the map equals the host-path
    handle's after every frame."""
    sy = flb.synth
    f = frames("C2")
    a, b = pair(flb, f, scan=False)
    prm = flb.capi.lio_params(f, 3)
    rng = np.random.default_rng(4)
    R_LI, t_LI = f["R_LI"], f["t_LI"]
    world = (f["R_true"] @ (R_LI @ f["scan_body"].T.astype(np.float64) + t_LI[:, None])).T + f["p_true"]
    for k in range(20):
        # the sensor moves and turns; it sees the same surfaces (a consistent scan of them from the new pose) plus a tenth
        # of points that stay fixed in the body frame (clutter that moves with it, so the map grows)
        Rk = f["R_true"] @ sy.exp_so3(np.array([0.0, 0.0, 0.03 * k]))
        pk = f["p_true"] + k * np.array([0.3, 0.1, 0.01])
        keep = rng.permutation(len(world))[: len(world) - 37 * k]
        body = (R_LI.T @ (Rk.T @ (world[keep] - pk).T - t_LI[:, None])).T.astype(np.float32)
        body[: len(body) // 10] = f["scan_body"][keep[: len(body) // 10]]
        a.scan_upload(body)
        b.scan_upload(body)
        xa = flb.capi.State18.make(Rk @ sy.exp_so3(rng.normal(0, 0.004, 3)), pk + rng.normal(0, 0.03, 3), f["vel"], f["bg"], f["ba"],
                                   f["grav"], f["cov"])
        xb = xa.copy()
        a.lio_update(prm, xa, xa.copy())
        b.lio_update(prm, xb, xb.copy())
        assert bytes(xa) == bytes(xb)
        a.map_add_scan(prm, 0.5)
        b.map_add_points(oracle_world(po, f, body, xb.R, xb.p), 0.5)
        assert_same_map(a, b)
    a.close()
    b.close()


def _frame_arrays(f):
    return (np.ascontiguousarray(f["scan_body"], np.float32), np.ascontiguousarray(f["image"], np.uint8),
            np.ascontiguousarray(f["patch_pos"], np.float64).reshape(-1, 3),
            np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(f["patch_pos"]), 192),
            np.ascontiguousarray(f["patch_level"], np.int32))


def test_frame_api_order(flb, po, frames):
    """After flb_frame_enqueue (LIO + VIO) the NULL pose is the VIO posterior; between separate LIO and VIO updates it
    is the LIO posterior."""
    f = frames("T1")
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 3)
    ds = 0.3
    scan, img, pos, patch, level = _frame_arrays(f)
    # whole frame
    a, b = pair(flb, f, scan=False)
    a.camera_set(f["cam"])
    x0 = flb.capi.State18.from_frame(f)
    fi = a.frame_inputs(scan, x0, x0.copy(), img, pos, patch, level)
    a.frame_enqueue(fi, lprm, vprm)
    a.map_add_scan(lprm, ds)
    xv, _, _ = a.state_download()
    b.map_add_points(oracle_world(po, f, scan, xv.R, xv.p), ds)
    assert_same_map(a, b)
    a.close()
    b.close()
    # separate updates: map_add_scan between them sees the LIO posterior
    a, b = pair(flb, f)
    a.camera_set(f["cam"])
    a.image_upload(img)
    a.patches_upload(pos, patch, level)
    x0 = flb.capi.State18.from_frame(f)
    a.state_upload(x0, x0.copy())
    a.lio_update_enqueue(lprm)
    a.map_add_scan(lprm, ds)
    xl, _, _ = a.state_download()
    a.state_set_prior_enqueue()
    a.vio_update_enqueue(vprm)
    xv2, _, _ = a.state_download()
    assert (xl.vector() != xv2.vector()).any()      # the VIO update moved the state: the two posteriors differ
    b.map_add_points(oracle_world(po, f, scan, xl.R, xl.p), ds)
    assert_same_map(a, b)
    a.close()
    b.close()


def _expect(code, fn):
    with pytest.raises(Exception) as e:
        fn()
    assert getattr(e.value, "code", None) == code, e.value
    return str(e.value)


def test_errors_leave_map_unchanged(flb, po, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    R, p = f["R_true"], f["p_true"]
    # no map
    h = flb.Handle(device=0)
    h.scan_upload(f["scan_body"])
    _expect(ERR_STATE, lambda: h.map_add_scan(prm, 0.3, R, p))
    h.close()

    a = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    a.map_upload(f["map_xyz"])
    b = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    b.map_upload(f["map_xyz"])

    def unchanged_then_valid(code, fn):
        before, info = a.map_download().tobytes(), a.map_grid_info()
        _expect(code, fn)
        assert a.map_download().tobytes() == before and a.map_grid_info() == info
        a.scan_upload(f["scan_body"])
        a.map_add_scan(prm, 0.3, R, p)
        b.map_add_points(oracle_world(po, f, f["scan_body"], R, p), 0.3)
        assert_same_map(a, b)

    unchanged_then_valid(ERR_STATE, lambda: a.map_add_scan(prm, 0.3, R, p))                     # no scan yet
    a.voxel_grid(f["scan_body"], 0.5)                                                           # scan slot used as scratch
    unchanged_then_valid(ERR_STATE, lambda: a.map_add_scan(prm, 0.3, R, p))
    unchanged_then_valid(ERR_STATE, lambda: a.map_add_scan(prm, 0.3))                           # no device state
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(None, 0.3, R, p))
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.3, R, None))
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.3, None, p))
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.0, R, p))
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, -0.5, R, p))
    Rn = np.array(R, np.float64)
    Rn[0, 1] = np.nan
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.3, Rn, p))
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.3, R, p + np.array([4.0e5, 0, 0])))   # > 2^20 voxels of 0.3 m
    # a diverged device state (NULL pose)
    xn = flb.capi.State18.from_frame(f)
    xn.pos[1] = float("nan")
    a.state_upload(xn, xn.copy())
    unchanged_then_valid(ERR_INVALID, lambda: a.map_add_scan(prm, 0.3))
    # and the NULL pose works again once the device state is sane
    xg = flb.capi.State18.from_frame(f, prop=False)
    a.state_upload(xg, xg.copy())
    a.map_add_scan(prm, 0.3)
    b.map_add_points(oracle_world(po, f, f["scan_body"], xg.R, xg.p), 0.3)
    assert_same_map(a, b)
    a.close()
    b.close()


def test_sparse_anchor_limit(flb, po, frames):
    f = frames("T1")
    a, b = pair(flb, f, 2)
    prm = flb.capi.lio_params(f, 3)
    R, p = f["R_true"], f["p_true"]
    before = a.map_download().tobytes()
    # 7e5 m: within 2^20 voxels of 1 m, beyond 2^20 cells of 0.6 m from the anchor
    msg = _expect(ERR_INVALID, lambda: a.map_add_scan(prm, 1.0, R, p + np.array([7.0e5, 0, 0])))
    assert "anchor" in msg
    assert a.map_download().tobytes() == before and a.map_grid_info()["sparse"] == 1
    a.map_add_scan(prm, 1.0, R, p)
    b.map_add_points(oracle_world(po, f, f["scan_body"], R, p), 1.0)
    assert_same_map(a, b)
    a.close()
    b.close()


def test_multi_gpu_refused(flb, frames):
    if not os.environ.get("FLB_TEST_WORLD"):
        pytest.skip("multi-GPU mode: set FLB_TEST_WORLD to run (as test_multirank)")
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    a, _ = pair(flb, f)
    before = a.map_download().tobytes()
    a.p2p_attach(0, 1, [a.p2p_export()])
    _expect(ERR_STATE, lambda: a.map_add_scan(prm, 0.3, f["R_true"], f["p_true"]))
    a.p2p_detach()
    a.comm_init(flb.Handle.comm_unique_id(), 0, 1)
    _expect(ERR_STATE, lambda: a.map_add_scan(prm, 0.3, f["R_true"], f["p_true"]))
    assert a.map_download().tobytes() == before
    a.close()
