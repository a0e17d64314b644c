"""GPU tier: publish_effect_world's cloud on the device (flb_effect_cloud, src/laserMapping.cpp:871-885): laserCloudOri
(:1588-1600) of the last LIO pass, transformed by RGBpointBodyToWorld.

The oracle's side of every check is `Lio.last_ori()` (the scan indices of the rows of the last pass it ran) and the
oracle's pointBodyToWorld of those body points.  Chains run scan upload -> LIO update (blocking, enqueue-only, or
flb_frame_enqueue) -> flb_map_add_scan -> flb_effect_cloud(NULL, NULL) on a moving trajectory, with the oracle on the
device map of the same frame.  The multi-GPU refusal (FLB_ERR_STATE after flb_comm_init / flb_p2p_attach) needs a
second rank and is not exercised on one GPU."""
import ctypes as C

import numpy as np
import pytest

import effect_oracle as eo

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
DS = 0.5


def oracle_world(po, f, body, R, p, R_LI=None, t_LI=None):
    """pointBodyToWorld (double math, float store) of `body`, as the oracle's LIO pass exports it."""
    body = np.ascontiguousarray(body, np.float32)
    if len(body) == 0:
        return np.zeros((0, 3), np.float32)
    g = dict(f, R_LI=f["R_LI"] if R_LI is None else R_LI, t_LI=f["t_LI"] if t_LI is None else t_LI)
    lio = po.Lio(body[:64].copy(), body)
    return np.ascontiguousarray(lio.run_pass(po.lio_params(g, 1), np.asarray(R, np.float64), np.asarray(p, np.float64), True)["world"])


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def ostate(po, x):
    """The oracle's State18 holding the bytes of the binding's (the two share flb_state18's layout)."""
    o = po.State18()
    C.memmove(C.byref(o), C.byref(x), C.sizeof(o))
    return o


def trajectory(flb, f, n, seed=4):
    """n frames of (body scan, prior state) on a moving trajectory over f's surfaces (as test_gpu_map_add_scan's), with a
    tenth of the points fixed in the body frame."""
    sy = flb.synth
    rng = np.random.default_rng(seed)
    R_LI, t_LI = f["R_LI"], f["t_LI"]
    world = (f["R_true"] @ (R_LI @ f["scan_body"].T.astype(np.float64) + t_LI[:, None])).T + f["p_true"]
    out = []
    for k in range(n):
        Rk = f["R_true"] @ sy.exp_so3(np.array([0.0, 0.0, 0.03 * k]))
        pk = f["p_true"] + k * np.array([0.3, 0.1, 0.01])
        keep = rng.permutation(len(world))[: len(world) - len(world) // 60 * k]
        body = (R_LI.T @ (Rk.T @ (world[keep] - pk).T - t_LI[:, None])).T.astype(np.float32)
        body[: len(body) // 10] = f["scan_body"][keep[: len(body) // 10]]
        x = flb.capi.State18.make(Rk @ sy.exp_so3(rng.normal(0, 0.004, 3)), pk + rng.normal(0, 0.03, 3), f["vel"], f["bg"], f["ba"],
                                  f["grav"], f["cov"])
        out.append((np.ascontiguousarray(body), x))
    return out


def run_chain(flb, po, f, route, persistent, n_frames):
    """The chain on one handle; per frame: the effect cloud, the device posterior, the report and the oracle's check."""
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size, persistent=persistent)
    h.map_upload(f["map_xyz"])
    prm = flb.capi.lio_params(f, 3)
    oprm = po.lio_params(f, 3)
    res = []
    for k, (body, x0) in enumerate(trajectory(flb, f, n_frames)):
        dev_map = h.map_download()                            # the map this frame's update searches
        if route == "frame_enqueue":
            pin = h.pinned_like(body)
            fi = h.frame_inputs(pin, x0, x0.copy())
            h.frame_enqueue(fi, prm, None, k & 1)
            x, rep, _ = h.state_download_wait(k & 1)
        else:
            h.scan_upload(body)
            if route == "lio_update":
                x = x0.copy()
                rep = h.lio_update(prm, x, x0)
            else:
                h.state_upload(x0, x0.copy())
                h.lio_update_enqueue(prm)
        h.map_add_scan(prm, DS, x0.R, x0.p)                   # at the prior: both execution modes grow the same map
        n = h.effect_cloud(prm)                               # at the device posterior, in stream order
        got = h.effect_cloud_download()
        if route == "lio_update_enqueue":
            x, rep, _ = h.state_download()
        lio = eo.Lio(dev_map, body)
        xo = ostate(po, x0)
        orep = lio.update(oprm, xo, ostate(po, x0))
        ori = lio.last_ori()
        assert (rep.passes, rep.n_eff_last) == (orep.passes, orep.n_eff_last)
        assert n == len(got) == rep.n_eff_last == len(ori) > len(body) // 8
        assert got.tobytes() == oracle_world(po, f, body[ori], x.R, x.p).tobytes()
        # the oracle's posterior as an explicit pose
        assert h.effect_cloud(prm, xo.R, xo.p) == n
        at_xo = h.effect_cloud_download().tobytes()
        assert at_xo == oracle_world(po, f, body[ori], xo.R, xo.p).tobytes()
        res.append((n, at_xo))
    h.close()
    return res


# C2 runs the blocking route only: the oracle's brute-force kNN dominates its time
@pytest.mark.parametrize("name,route", [("T0", "lio_update"), ("T0", "lio_update_enqueue"), ("T0", "frame_enqueue"),
                                        ("C2", "lio_update")])
def test_chain_matches_oracle_both_modes(flb, po, frames, name, route):
    f = frames(name)
    nf = 4 if name == "T0" else 2
    a = run_chain(flb, po, f, route, 1, nf)
    b = run_chain(flb, po, f, route, 0, nf)
    # persistent == kernel-per-pass, byte for byte, at one pose (the two modes' posteriors differ in the last bits: their
    # reductions are ordered differently)
    assert a == b


def test_ikfom_update(flb, po, frames):
    """flb_lio_update_ikfom's last h_share_model evaluation, with the IKFoM pose and extrinsic given explicitly."""
    f = frames("T0")
    L = po.lib()
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.map_upload(f["map_xyz"])
    h.scan_upload(f["scan_body"])
    xg = flb.capi.StateIkfom()
    C.memmove(C.byref(xg), C.byref(po.state_ikfom_from_frame(f)), C.sizeof(xg))
    prm = flb.capi.IkfomParams()
    prm.laser_point_cov = f["cfg"].laser_point_cov
    prm.max_iteration = 4
    prm.limit[:] = [0.001] * 23
    grep = h.lio_update_ikfom(prm, xg)
    lio = eo.Lio(f["map_xyz"], f["scan_body"])
    xo = po.state_ikfom_from_frame(f)
    orep = lio.update_ikfom(po.ikfom_params(f, 4), xo)
    ori = lio.last_ori()
    assert grep.n_eff_last == orep.n_eff_last == len(ori) > 100

    def R_of(q):
        R = np.zeros(9)
        L.flo_quat_to_R(np.ascontiguousarray(q, np.float64).ctypes.data_as(C.c_void_p), R.ctypes.data_as(C.c_void_p))
        return R.reshape(3, 3)

    R, p = R_of(xg.rot[:]), np.array(xg.pos[:])
    R_LI, t_LI = R_of(xg.offset_R_L_I[:]), np.array(xg.offset_T_L_I[:])
    lprm = flb.capi.lio_params(dict(f, R_LI=R_LI, t_LI=t_LI), 1)
    assert h.effect_cloud(lprm, R, p) == len(ori)
    ref = oracle_world(po, f, f["scan_body"][ori], R, p, R_LI, t_LI)
    assert h.effect_cloud_download().tobytes() == ref.tobytes()
    h.close()


@pytest.mark.parametrize("width", [6, 12])
def test_lio_pass_rows(flb, po, frames, width):
    """flb_lio_pass: the rows of that pass, flb_lio_export's sel_idx, at the oracle's sel_idx too."""
    f = frames("T1")
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.load_frame(f)
    lio = eo.Lio(f["map_xyz"], f["scan_body"])
    prm, oprm = flb.capi.lio_params(f, 3), po.lio_params(f, 3)
    Rq, pq = f["R_true"], np.asarray(f["p_true"]) + [0.2, -0.1, 0.05]
    poses = [(f["R_prop"], f["p_prop"], True),
             (f["R_prop"] @ flb.synth.exp_so3(np.array([0.002, -0.001, 0.003])), f["p_prop"] + [0.01, -0.02, 0.005], False)]
    for R, p, rematch in poses:
        g = h.lio_pass(prm, R, p, rematch, width=width)
        o = lio.run_pass(oprm, R, p, rematch)
        assert np.array_equal(g["sel_idx"], o["sel_idx"]) and np.array_equal(lio.last_ori(), o["sel_idx"])
        assert h.effect_cloud(prm, Rq, pq) == g["n"] == len(g["sel_idx"]) > 100
        assert h.effect_cloud_download().tobytes() == oracle_world(po, f, f["scan_body"][g["sel_idx"]], Rq, pq).tobytes()
    h.close()


def test_far_point_is_not_a_row(flb, po):
    """A point 400 m out, 2.1 m off a plane: s > 0.9 selects it, |pd2| > 2 keeps it out of laserCloudOri."""
    from test_effect_cloud import far_scene
    f = far_scene()
    h = flb.Handle(device=0, cell_size=0.6)
    h.map_upload(f["map_xyz"])
    h.scan_upload(f["scan_body"])
    prm = flb.capi.lio_params(f, 1)
    g = h.lio_pass(prm, np.eye(3), np.zeros(3), True)
    assert g["sel_idx"].tolist() == [2, 3]
    assert h.effect_cloud(prm, np.eye(3), np.array([1.0, 2.0, 3.0])) == 2
    ref = oracle_world(po, f, f["scan_body"][[2, 3]], np.eye(3), np.array([1.0, 2.0, 3.0]))
    assert h.effect_cloud_download().tobytes() == ref.tobytes()
    h.close()


def test_stale_and_lost(flb, po, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    (b0, x0), (b1, x1), (b2, x2) = trajectory(flb, f, 3)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.map_upload(f["map_xyz"])
    h.scan_upload(b0)
    # no pass ever: 0 points, at an explicit pose and at the device state
    assert h.effect_cloud(prm, x0.R, x0.p) == 0 and len(h.effect_cloud_download()) == 0
    expect_error(flb, ERR_STATE, h.effect_cloud, prm)           # no device state yet
    h.state_upload(x0, x0.copy())
    assert h.effect_cloud(prm) == 0
    # frame 0, captured
    x = x0.copy()
    h.lio_update(prm, x, x0)
    lio = eo.Lio(f["map_xyz"], b0)
    xo = ostate(po, x0)
    lio.update(po.lio_params(f, 3), xo, ostate(po, x0))
    ori0 = lio.last_ori()
    assert h.effect_cloud(prm) == len(ori0) > 100
    # a new scan and no pass: the previous rows at the new pose (the reference's stale laserCloudOri)
    h.scan_upload(b1)
    h.state_upload(x1, x1.copy())
    assert h.effect_cloud(prm) == len(ori0)
    assert h.effect_cloud_download().tobytes() == oracle_world(po, f, b0[ori0], x1.R, x1.p).tobytes()
    # a pass, one more scan upload, then the capture: still that pass's rows (the set survives one install)
    x = x1.copy()
    h.lio_update(prm, x, x1)
    lio1 = eo.Lio(f["map_xyz"], b1)
    xo = ostate(po, x1)
    lio1.update(po.lio_params(f, 3), xo, ostate(po, x1))
    ori1 = lio1.last_ori()
    h.scan_upload(b2)
    assert h.effect_cloud(prm, x2.R, x2.p) == len(ori1)
    assert h.effect_cloud_download().tobytes() == oracle_world(po, f, b1[ori1], x2.R, x2.p).tobytes()
    # an uncaptured pass followed by two scan uploads: refused until the next pass
    h.state_upload(x2, x2.copy())
    h.lio_update_enqueue(prm)
    h.scan_upload(b0)
    h.scan_upload(b1)
    expect_error(flb, ERR_STATE, h.effect_cloud, prm, x2.R, x2.p)
    expect_error(flb, ERR_STATE, h.effect_cloud_download)
    expect_error(flb, ERR_STATE, h.effect_cloud, prm, x2.R, x2.p)
    x = x1.copy()
    h.lio_update(prm, x, x1)
    assert h.effect_cloud(prm, x2.R, x2.p) == len(ori1)
    assert h.effect_cloud_download().tobytes() == oracle_world(po, f, b1[ori1], x2.R, x2.p).tobytes()
    # an uncaptured pass followed by flb_voxel_grid (the scan slot as scratch)
    h.lio_update(prm, x1.copy(), x1)
    h.voxel_grid(b0[:100], 0.2)
    expect_error(flb, ERR_STATE, h.effect_cloud, prm, x2.R, x2.p)
    h.close()


def test_bad_arguments(flb, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.load_frame(f)
    x0 = flb.capi.State18.from_frame(f)
    h.lio_update(prm, x0.copy(), x0)
    R, p = f["R_true"], f["p_true"]
    n = h.effect_cloud(prm, R, p)
    assert n > 100
    for bad in (lambda: h.effect_cloud(None, R, p), lambda: h.effect_cloud(prm, R, None), lambda: h.effect_cloud(prm, None, p),
                lambda: h.effect_cloud(prm, R, np.asarray(p) + [1e39, 0.0, 0.0])):
        expect_error(flb, ERR_INVALID, bad)
        expect_error(flb, ERR_STATE, h.effect_cloud_download)      # no effect cloud held after an error
        assert h.effect_cloud(prm, R, p) == n                        # the capture is kept
    out = np.zeros((n, 3), np.float32)
    m = C.c_int()
    L = h.L
    assert L.flb_effect_cloud_download(h.h, out.ctypes.data_as(C.c_void_p), -1, C.byref(m)) == ERR_INVALID
    assert L.flb_effect_cloud_download(h.h, None, 5, C.byref(m)) == ERR_INVALID
    assert L.flb_effect_cloud_download(h.h, out.ctypes.data_as(C.c_void_p), 7, C.byref(m)) == 0 and m.value == n
    assert L.flb_effect_cloud_download(h.h, None, 0, C.byref(m)) == 0 and m.value == n
    h.close()


def test_no_interference(flb, frames):
    """A LIO update after flb_effect_cloud gives the state and report it gives without the call, bit for bit."""
    f = frames("T1")
    prm = flb.capi.lio_params(f, 3)
    traj = trajectory(flb, f, 3)
    out = []
    for call in (False, True):
        h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
        h.map_upload(f["map_xyz"])
        r = []
        for body, x0 in traj:
            h.scan_upload(body)
            x = x0.copy()
            rep = h.lio_update(prm, x, x0)
            if call:
                h.effect_cloud(prm)
                h.effect_cloud_download()
            h.map_add_scan(prm, DS)
            r.append((bytes(x), bytes(rep)))
        out.append(r)
        h.close()
    assert out[0] == out[1]
