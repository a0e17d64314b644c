"""GPU tier of the VIO patch guard: the CUDA update against the oracle on patches placed exactly at the image edges,
behind and at the camera (tests/vio_edge_util.py), in both execution modes; updates whose patch sets change between
passes, a level that loses every patch, batched frames, and the refusal of a camera / image size mismatch on every
path that reads the image."""
import numpy as np
import pytest

import vio_edge_util as U
from conftest import bits
from test_gpu_parity import STATE_RTOL, handle, rel  # noqa: F401  (handle: both execution modes)

pytestmark = pytest.mark.gpu

SCENARIOS = [(W, H, cam) for (W, H) in U.SIZES for cam in U.CAMERAS]
IDS = [f"{W}x{H}-{cam}" for (W, H, cam) in SCENARIOS]
FLB_ERR_STATE = -4


def _ostate(po, f, R=None, p=None):
    return po.State18.make(f["R_prop"] if R is None else R, f["p_prop"] if p is None else p, f["vel"], f["bg"], f["ba"],
                           f["grav"], f["cov"])


def _gstate(flb, f, R=None, p=None):
    return flb.capi.State18.make(f["R_prop"] if R is None else R, f["p_prop"] if p is None else p, f["vel"], f["bg"], f["ba"],
                                 f["grav"], f["cov"])


def _vio(po, f):
    return po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])


@pytest.mark.parametrize("W,H,cam", SCENARIOS, ids=IDS)
def test_vio_pass_parity_at_edges(flb, po, handle, W, H, cam):
    f = U.scenario(W, H, cam, depth_points=True)
    handle.load_frame(f)
    vio = _vio(po, f)
    for level in (2, 1, 0):
        o = vio.run_pass(po.vio_params(f, 3), f["R_true"], f["p_true"], level)
        g = handle.vio_pass(flb.capi.vio_params(f, 3), f["R_true"], f["p_true"], level)
        assert g["n_meas"] == o["n_meas"] and g["skipped"] == o["skipped"]
        skipped = U.skip_set(g["H_sub"], vio.Pn)
        valid = U.expected_valid(f["cam"], f["R_true"], f["p_true"], f["patch_pos"], f["patch_level"], level)[0]
        assert (skipped == ~valid).all(), np.nonzero(skipped != ~valid)[0]
        assert (bits(g["z"]) == bits(o["z"])).all()
        assert (bits(g["errors"]) == bits(o["errors"])).all()
        assert (g["z"].reshape(-1, 64)[skipped] == 0).all() and (g["errors"][skipped] == 0).all()
        np.testing.assert_allclose(g["H_sub"], o["H_sub"], rtol=1e-12, atol=1e-300)
        assert rel(g["HTH6"], o["HTH6"]) < 1e-11 and rel(g["HTz6"], o["HTz6"]) < 1e-10


def _assert_update(grep, orep, xg, xo, handle, vio):
    assert list(grep.passes) == list(orep.passes)
    assert grep.rows_total == orep.rows_total and grep.skipped_last == orep.skipped_last
    assert grep.cov_updated == orep.cov_updated
    np.testing.assert_allclose(list(grep.last_error), list(orep.last_error), rtol=1e-6)     # NaN == NaN
    assert rel(xg.vector(), xo.vector()) < STATE_RTOL
    assert rel(xg.P, xo.P) < 1e-7
    assert (bits(handle.vio_errors()) == bits(vio.errors())).all()


@pytest.mark.parametrize("W,H,cam", SCENARIOS, ids=IDS)
@pytest.mark.parametrize("T,early,force", [(4, True, False), (3, False, True)], ids=["early-stop", "all-passes"])
def test_vio_update_parity_at_edges(flb, po, handle, W, H, cam, T, early, force):
    """Edge patches cross the guard between passes (their skip sets at the prior and the posterior differ); the
    early-stop updates also reject a step, where the persistent kernel discards the pass it published ahead."""
    f = U.scenario(W, H, cam)
    handle.load_frame(f)
    vio = _vio(po, f)
    xo = _ostate(po, f)
    orep = vio.update(po.vio_params(f, T, early_stop=early, force_all_passes=force), xo, xo.copy())
    crossed = [(U.expected_valid(f["cam"], f["R_prop"], f["p_prop"], f["patch_pos"], f["patch_level"], L)[0] !=
                U.expected_valid(f["cam"], xo.R, xo.p, f["patch_pos"], f["patch_level"], L)[0]).any() for L in (2, 1, 0)]
    assert all(crossed)
    gprm = flb.capi.vio_params(f, T, early_stop=early, force_all_passes=force)
    xg = _gstate(flb, f)
    grep = handle.vio_update(gprm, xg, xg.copy())
    _assert_update(grep, orep, xg, xo, handle, vio)
    # the same update enqueued, read back with flb_state_download
    x0 = _gstate(flb, f)
    handle.state_upload(x0, x0.copy())
    handle.vio_update_enqueue(gprm)
    xe, _, erep = handle.state_download()
    _assert_update(erep, orep, xe, xo, handle, vio)


@pytest.fixture(scope="module")
def small():
    """96 x 80 with every patch at search_level 1: level 2 reads 81 rows at scale 8 and never fits, level 1 (41 px) does."""
    return U.scenario(96, 80, "pinhole", search_level=1, n_interior=24)


@pytest.mark.parametrize("early,force", [(True, False), (False, True)], ids=["early-stop", "all-passes"])
def test_level_without_patches(flb, po, handle, small, early, force):
    """n_meas = 0 on level 2: error = 0/0 = NaN; with early stop the pass is rejected and the level ends, with
    force_all_passes the NaN pass is accepted.  Levels 1 and 0 then run normally."""
    f = small
    for L, n in ((2, 0), (1, 24), (0, 24)):
        assert U.expected_valid(f["cam"], f["R_prop"], f["p_prop"], f["patch_pos"], f["patch_level"], L)[0].sum() == n
    handle.load_frame(f)
    vio = _vio(po, f)
    T = 3
    oprm, gprm = po.vio_params(f, T, early_stop=early, force_all_passes=force), \
        flb.capi.vio_params(f, T, early_stop=early, force_all_passes=force)
    xo, xg = _ostate(po, f), _gstate(flb, f)
    orep = vio.update(oprm, xo, xo.copy())
    grep = handle.vio_update(gprm, xg, xg.copy())
    assert np.isnan(orep.last_error[2]) == force and orep.cov_updated == 1
    _assert_update(grep, orep, xg, xo, handle, vio)
    # level by level (LidarSelector::UpdateState alone), the state after each level
    xo, xg = _ostate(po, f), _gstate(flb, f)
    xpo, xpg = xo.copy(), xg.copy()
    Go = np.zeros((18, 18))
    for level in (2, 1, 0):
        now_o, Go, ro = vio.update_level(oprm, level, 1e10, xo, xpo, Go)
        now_g, _, rg = handle.vio_update_level(gprm, level, 1e10, xg, xpg)
        assert list(rg.passes) == list(ro.passes)
        np.testing.assert_allclose(now_g, now_o, rtol=1e-6)
        assert rel(xg.vector(), xo.vector()) < STATE_RTOL
        assert (bits(handle.vio_errors()) == bits(vio.errors())).all()


def test_every_patch_behind_the_camera(flb, po, handle, small):
    """The camera turned 180 degrees: every patch is behind it at every level; every level's first pass has no
    measurement and is rejected, and the state and covariance come back bit for bit."""
    f = small
    R = f["R_prop"] @ flb.synth.exp_so3(np.array([0.0, 0.0, np.pi]))
    for L in (2, 1, 0):
        assert not U.expected_valid(f["cam"], R, f["p_prop"], f["patch_pos"], f["patch_level"], L)[0].any()
    handle.load_frame(f)
    vio = _vio(po, f)
    xo = _ostate(po, f, R=R)
    orep = vio.update(po.vio_params(f, 3), xo, xo.copy())
    x0 = _gstate(flb, f, R=R)
    xg = x0.copy()
    grep = handle.vio_update(flb.capi.vio_params(f, 3), xg, x0.copy())
    assert list(orep.passes) == list(grep.passes) == [1, 1, 1]
    assert orep.cov_updated == grep.cov_updated == 0
    assert (xg.vector() == x0.vector()).all() and (xg.P == x0.P).all()
    assert (xo.vector() == x0.vector()).all() and (xo.P == x0.P).all()


def test_batched_frames_at_edges(flb, po):
    """Three frames whose priors put different edge patches across the guard, batched: each equals the same frame alone
    on the kernel-per-pass handle bit for bit; one also equals the oracle."""
    f = U.scenario(321, 257, "radtan")
    rng = np.random.default_rng(23)
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 4)
    perm = rng.permutation(len(f["scan_body"]))
    fr = []
    for b in range(3):
        idx = np.sort(perm[b::3])                 # disjoint thirds of the scan: three different LIO posteriors
        R = f["R_prop"] @ flb.synth.exp_so3(rng.normal(0, 0.003, 3))
        p = f["p_prop"] + rng.normal(0, 0.01, 3)
        fr.append((np.ascontiguousarray(f["scan_body"][idx]), R, p))
    # the VIO prior of each frame is its LIO posterior: the patches read there differ from frame to frame
    lio_post, skips = [], []
    for scan, R, p in fr:
        xo = _ostate(po, f, R, p)
        po.Lio(f["map_xyz"], scan).update(po.lio_params(f, 3), xo, xo.copy())
        lio_post.append(xo)
        skips.append(np.concatenate([~U.expected_valid(f["cam"], xo.R, xo.p, f["patch_pos"], f["patch_level"], L)[0]
                                     for L in (2, 1, 0)]))
    assert (skips[0] != skips[1]).any() and (skips[1] != skips[2]).any() and (skips[0] != skips[2]).any()
    single = []
    h1 = flb.Handle(device=0, persistent=0)
    h1.load_frame(f)
    for scan, R, p in fr:
        x = _gstate(flb, f, R, p)
        h1.scan_upload(scan)
        h1.state_upload(x, x.copy())
        h1.lio_update_enqueue(lprm)
        h1.state_set_prior_enqueue()
        h1.vio_update_enqueue(vprm)
        single.append(h1.state_download())
    h1.close()
    hb = flb.Handle(device=0)
    hb.load_frame(f)
    hb.batch_begin(3, max(len(s) for s, _, _ in fr))
    for b, (scan, R, p) in enumerate(fr):
        x = _gstate(flb, f, R, p)
        hb.batch_set_frame(b, scan, x, x.copy())
    hb.batch_update_enqueue(lprm, vprm)
    for b in range(3):
        xb, lb, vb = hb.batch_state_download(b)
        xs, ls, vs = single[b]
        assert (lb.passes, lb.rows_total) == (ls.passes, ls.rows_total)
        assert list(vb.passes) == list(vs.passes) and vb.rows_total == vs.rows_total and vb.cov_updated == vs.cov_updated
        assert list(vb.last_error) == list(vs.last_error) and vb.skipped_last == vs.skipped_last
        assert (xb.vector() == xs.vector()).all() and (np.array(xb.cov[:]) == np.array(xs.cov[:])).all()
    hb.close()
    xo = lio_post[1]
    rep = _vio(po, f).update(po.vio_params(f, 4), xo, xo.copy())
    assert list(single[1][2].passes) == list(rep.passes) and single[1][2].rows_total == rep.rows_total
    assert rel(single[1][0].vector(), xo.vector()) < STATE_RTOL


def test_camera_image_size_mismatch_refused(flb, po, frames):
    """A 640 x 512 camera over a 320 x 256 image: every call that reads the image refuses with FLB_ERR_STATE before it
    stages or launches anything, and the handle then runs a correctly sized update as before."""
    f = frames("T0")
    h = flb.Handle(device=0)
    h.load_frame(f)
    big = dict(f["cam"], width=640, height=512)
    h.camera_set(big)
    prm, lprm = flb.capi.vio_params(f, 3), flb.capi.lio_params(f, 3)
    x = flb.capi.State18.from_frame(f)
    Rcw, Pcw = np.eye(3), np.zeros(3)
    pts = f["map_xyz"][:64]
    calls = {
        "flb_vio_pass": lambda: h.vio_pass(prm, f["R_prop"], f["p_prop"], 0),
        "flb_vio_update": lambda: h.vio_update(prm, x.copy(), x.copy()),
        "flb_vio_update_level": lambda: h.vio_update_level(prm, 2, 1e10, x.copy(), x.copy()),
        "flb_vio_update_enqueue": lambda: (h.state_upload(x, x.copy()), h.vio_update_enqueue(prm)),
        "flb_frame_enqueue": lambda: h.frame_enqueue(h.frame_inputs(np.ascontiguousarray(f["scan_body"]), x.copy(), x.copy()), lprm, prm),
        "flb_batch_update_enqueue": lambda: (h.batch_begin(1, len(f["scan_body"])),
                                             h.batch_set_frame(0, f["scan_body"], x.copy(), x.copy()),
                                             h.batch_update_enqueue(lprm, prm)),
        "flb_visual_candidates": lambda: h.visual_candidates(Rcw, Pcw, pts, 40, 40, np.zeros((320 // 40) * (256 // 40), np.float32)),
        "flb_vmap_select": lambda: (h.vmap_reset(f), h.vmap_select(Rcw, Pcw, pts)),
    }
    for name, call in calls.items():
        with pytest.raises(flb.FlbError) as e:
            call()
        assert e.value.code == FLB_ERR_STATE, name
        assert "size mismatch" in str(e.value), name
    h.camera_set(f["cam"])
    h.patches_upload(f["patch_pos"], f["patch_ref"], f["patch_level"])   # flb_vmap_reset gave the patch list to the map
    vio = _vio(po, f)
    xo = po.state_from_frame(f)
    orep = vio.update(po.vio_params(f, 3), xo, xo.copy())
    xg = flb.capi.State18.from_frame(f)
    grep = h.vio_update(prm, xg, xg.copy())
    _assert_update(grep, orep, xg, xo, h, vio)
    h.close()
