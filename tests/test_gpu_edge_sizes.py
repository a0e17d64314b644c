"""GPU tier: degenerate sizes of the persistent update kernels (worker blocks + one leader block, chunked
points, warp-per-patch): one point, one patch, fewer points than a warp, counts around the chunk / block
boundaries, zero iterations -- both execution modes against the oracle."""
import numpy as np
import pytest

from test_gpu_parity import STATE_RTOL, _gstate, _ostate, rel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=[1, 0], ids=["persistent", "kernel-per-pass"])
def handle(flb, request):
    h = flb.Handle(device=0, persistent=request.param)
    yield h
    h.close()


@pytest.mark.parametrize("n", [1, 2, 5, 31, 32, 33, 64, 131, 132, 133, 147, 148, 149, 1047, 1048, 1049, 1175, 1176, 1177, 1185])
def test_lio_update_small_scans(flb, po, frames, handle, n):
    f = dict(frames("T1"))
    rng = np.random.default_rng(n)
    keep = np.sort(rng.choice(len(f["scan_body"]), n, replace=False))
    f["scan_body"] = np.ascontiguousarray(f["scan_body"][keep])
    handle.map_upload(f["map_xyz"])
    for T in (0, 1, 4):
        handle.scan_upload(f["scan_body"])
        lio = po.Lio(f["map_xyz"], f["scan_body"])
        xo, xpo = _ostate(po, f), _ostate(po, f)
        orep = lio.update(po.lio_params(f, T), xo, xpo)
        xg, xpg = _gstate(flb, f), _gstate(flb, f)
        grep = handle.lio_update(flb.capi.lio_params(f, T), xg, xpg)
        assert (grep.passes, grep.knn_passes, grep.n_eff_last, grep.rows_total) == (orep.passes, orep.knn_passes, orep.n_eff_last, orep.rows_total)
        if orep.n_eff_last > 0:
            assert rel(xg.vector(), xo.vector()) < STATE_RTOL
            assert rel(xg.P, xo.P) < 1e-7


@pytest.mark.parametrize("pn", [1, 2, 3, 15, 16, 17, 33, 150])
def test_vio_update_few_patches(flb, po, frames, handle, pn):
    f = frames("T1")
    rng = np.random.default_rng(100 + pn)
    keep = np.sort(rng.choice(len(f["patch_pos"]), pn, replace=False))
    ppos, pref, plev = f["patch_pos"][keep], f["patch_ref"][keep], f["patch_level"][keep]
    handle.camera_set(f["cam"])
    handle.image_upload(f["image"])
    handle.patches_upload(ppos, pref, plev)
    vio = po.Vio(f["image"], ppos, pref, plev, f["cam"])
    for T, force in ((1, False), (3, True), (4, False)):
        xo, xpo = _ostate(po, f), _ostate(po, f)
        orep = vio.update(po.vio_params(f, T, force_all_passes=force), xo, xpo)
        xg, xpg = _gstate(flb, f), _gstate(flb, f)
        grep = handle.vio_update(flb.capi.vio_params(f, T, force_all_passes=force), xg, xpg)
        assert list(grep.passes) == list(orep.passes)
        assert grep.rows_total == orep.rows_total and grep.cov_updated == orep.cov_updated
        np.testing.assert_allclose(list(grep.last_error), list(orep.last_error), rtol=1e-6)
        assert rel(xg.vector(), xo.vector()) < STATE_RTOL
        assert rel(xg.P, xo.P) < 1e-7


@pytest.mark.parametrize("n,pos", [(1, 0), (7, 6), (8, 3), (9, 8), (1000, 0), (1000, 999), (1000, 503)])
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_scan_upload_rejects_non_finite(flb, n, pos, bad):
    """The vectorised bounds / finiteness pass of flb_scan_upload (24 floats at a time + scalar tail)."""
    h = flb.Handle(device=0)
    pts = np.random.default_rng(n).uniform(-5, 5, (n, 3)).astype(np.float32)
    h.scan_upload(pts)                                   # clean input is accepted
    for axis in range(3):
        q = pts.copy()
        q[pos, axis] = bad
        with pytest.raises(flb.capi.FlbError):
            h.scan_upload(q)
    h.close()


def test_packet_flag_wraparound(flb, po, frames):
    """The pose-packet flag base advances by 4096 per persistent launch; before it overflows 32 bits the library
    re-bases it and clears the packet.  Run updates across that point: every one must still match the oracle."""
    import ctypes as C
    f = frames("T1")
    h = flb.Handle(device=0, persistent=1)
    h.load_frame(f)
    lio = po.Lio(f["map_xyz"], f["scan_body"])
    xo, xpo = _ostate(po, f), _ostate(po, f)
    lio.update(po.lio_params(f, 4), xo, xpo)
    vio = po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])
    xv, xpv = _ostate(po, f), _ostate(po, f)
    vio.update(po.vio_params(f, 3), xv, xpv)
    fn = h.L.flb_debug_set_packet_epoch
    fn.argtypes = [C.c_void_p, C.c_uint]
    h._ck(fn(h.h, 0xFFFF0000 - 3 * 4096))
    for it in range(8):                                   # launches 4 and 5 straddle the re-base
        xg, xpg = _gstate(flb, f), _gstate(flb, f)
        h.lio_update(flb.capi.lio_params(f, 4), xg, xpg)
        assert rel(xg.vector(), xo.vector()) < STATE_RTOL, it
        xg, xpg = _gstate(flb, f), _gstate(flb, f)
        h.vio_update(flb.capi.vio_params(f, 3), xg, xpg)
        assert rel(xg.vector(), xv.vector()) < STATE_RTOL, it
    h.close()


def test_deferred_state_moves(flb, frames):
    """flb_state_reset_enqueue / flb_state_set_prior_enqueue are carried out by the next persistent kernel (no separate
    device copy); every other consumer sees them as if they had been plain copies."""
    f = frames("T1")
    h = flb.Handle(device=0)
    h.load_frame(f)
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 3)
    x0 = flb.capi.State18.from_frame(f)
    h.state_upload(x0, x0.copy())
    h.lio_update_enqueue(lprm)
    h.state_set_prior_enqueue()
    h.vio_update_enqueue(vprm)
    x1, _, _ = h.state_download()
    # reset consumed by the LIO kernel, prior by the VIO kernel: the same frame again, bit for bit
    h.state_reset_enqueue()
    h.lio_update_enqueue(lprm)
    h.state_set_prior_enqueue()
    h.vio_update_enqueue(vprm)
    x2, _, _ = h.state_download()
    assert (x2.vector() == x1.vector()).all() and (np.array(x2.cov[:]) == np.array(x1.cov[:])).all()
    # a reset nobody consumes is flushed by the download
    h.state_reset_enqueue()
    x3, _, _ = h.state_download()
    assert (x3.vector() == x0.vector()).all() and (np.array(x3.cov[:]) == np.array(x0.cov[:])).all()
    # reset followed directly by the VIO update (no LIO kernel to consume it): flushed as a copy first
    h.state_reset_enqueue()
    h.state_set_prior_enqueue()
    h.vio_update_enqueue(vprm)
    xa, _, _ = h.state_download()
    xb = x0.copy()
    h.vio_update(vprm, xb, x0)
    assert (xa.vector() == xb.vector()).all()
    h.close()


def test_frame_enqueue_equals_separate_calls(flb, frames):
    """flb_frame_enqueue (one call per frame, pipelined read-back) == the separate upload / update / download calls;
    page-locked caller buffers are read in place."""
    f = frames("T1")
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 3)
    x0 = flb.capi.State18.from_frame(f)
    h = flb.Handle(device=0)
    h.load_frame(f)
    h.state_upload(x0, x0.copy())
    h.lio_update_enqueue(lprm)
    h.state_set_prior_enqueue()
    h.vio_update_enqueue(vprm)
    xs, ls, vs = h.state_download()
    h.close()
    h = flb.Handle(device=0)
    h.map_upload(f["map_xyz"])
    h.camera_set(f["cam"])
    scan = h.pinned_like(np.ascontiguousarray(f["scan_body"], np.float32))
    img = h.pinned_like(f["image"])
    pos = h.pinned_like(np.ascontiguousarray(f["patch_pos"], np.float64))
    ref = h.pinned_like(np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(pos), 192))
    lev = h.pinned_like(np.ascontiguousarray(f["patch_level"], np.int32))
    fi = h.frame_inputs(scan, x0, x0.copy(), img, pos, ref, lev)
    for k in range(3):                                   # three frames in flight over two result slots
        h.frame_enqueue(fi, lprm, vprm, k & 1)
        if k:
            xk, lk, vk = h.state_download_wait((k - 1) & 1)
            assert (xk.vector() == xs.vector()).all() and (np.array(xk.cov[:]) == np.array(xs.cov[:])).all()
            assert lk.rows_total == ls.rows_total and list(vk.passes) == list(vs.passes)
    xk, _, _ = h.state_download_wait(0)
    assert (xk.vector() == xs.vector()).all()
    # LIO only
    h.frame_enqueue(fi, lprm, None, 1)
    xl, ll, _ = h.state_download_wait(1)
    x1 = x0.copy()
    h.lio_update(lprm, x1, x0)
    assert (xl.vector() == x1.vector()).all() and ll.rows_total == ls.rows_total
    h.close()


def test_pipelined_frames_with_distinct_inputs(flb, frames):
    """Every input of a frame (scan, image, patch list, state) has two device sets and is uploaded on its own stream while
    the previous frame's updates still run.  Six frames whose inputs ALL differ, three in flight over two result slots,
    page-locked buffers read in place: each frame's result must be bit-identical to the same frame run alone with
    blocking calls -- a set switched too early / too late, or a copy overtaking a reader, shows up as a mismatch."""
    f = frames("T1")
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 3)
    rng = np.random.default_rng(77)
    n_frames = 6
    base_scan = np.ascontiguousarray(f["scan_body"], np.float32)
    base_pos = np.ascontiguousarray(f["patch_pos"], np.float64)
    base_ref = np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(base_pos), 192)
    base_lev = np.ascontiguousarray(f["patch_level"], np.int32)
    inputs = []
    for k in range(n_frames):
        n_k = len(base_scan) - 37 * k                                   # sizes differ too (k = 0: the full scan)
        p_k = len(base_pos) - 5 * k
        scan = base_scan[:n_k] + rng.normal(0, 0.004 * k, (n_k, 3)).astype(np.float32)
        img = np.clip(f["image"].astype(np.int32) + rng.integers(-3 * k, 3 * k + 1, f["image"].shape), 0, 255).astype(np.uint8)
        pos = base_pos[:p_k] + rng.normal(0, 0.002 * k, (p_k, 3))
        ref = base_ref[:p_k] + rng.normal(0, 0.5 * k, (p_k, 192)).astype(np.float32)
        x0 = flb.capi.State18.from_frame(f)
        x0.pos[0] += 0.003 * k
        x0.pos[1] -= 0.002 * k
        inputs.append((scan, img, pos, ref, base_lev[:p_k].copy(), x0))
    # (a) one frame at a time, blocking
    h = flb.Handle(device=0)
    h.map_upload(f["map_xyz"])
    h.camera_set(f["cam"])
    serial = []
    for scan, img, pos, ref, lev, x0 in inputs:
        h.scan_upload(scan)
        h.image_upload(img)
        h.patches_upload(pos, ref, lev)
        h.state_upload(x0, x0.copy())
        h.lio_update_enqueue(lprm)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
        serial.append(h.state_download())
    h.close()
    assert len({tuple(x.vector()) for x, _, _ in serial}) == n_frames     # the frames really differ
    # (b) pipelined through the one-call frame API, caller buffers page-locked (one set per frame: they stay untouched
    # until that frame's result has been collected)
    h = flb.Handle(device=0)
    h.map_upload(f["map_xyz"])
    h.camera_set(f["cam"])
    keep = []
    fis = []
    for scan, img, pos, ref, lev, x0 in inputs:
        bufs = [h.pinned_like(a) for a in (scan, img, pos, ref, lev)]
        keep.append(bufs)
        fis.append(h.frame_inputs(bufs[0], x0, x0.copy(), bufs[1], bufs[2], bufs[3], bufs[4]))

    def check(k, got):
        xk, lk, vk = got
        xs, ls, vs = serial[k]
        assert (xk.vector() == xs.vector()).all() and (np.array(xk.cov[:]) == np.array(xs.cov[:])).all(), f"frame {k}"
        assert lk.rows_total == ls.rows_total and vk.rows_total == vs.rows_total and list(vk.passes) == list(vs.passes)
    for k in range(n_frames):
        h.frame_enqueue(fis[k], lprm, vprm, k & 1)
        if k:
            check(k - 1, h.state_download_wait((k - 1) & 1))
    check(n_frames - 1, h.state_download_wait((n_frames - 1) & 1))
    # (c) the same through the separate enqueue calls with PAGEABLE buffers (staging path), two frames in flight
    for k in range(n_frames):
        scan, img, pos, ref, lev, x0 = inputs[k]
        h.scan_upload(scan)
        h.state_upload(x0, x0.copy())
        h.lio_update_enqueue(lprm)
        h.image_upload(img)
        h.patches_upload(pos, ref, lev)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
        h.state_download_enqueue(k & 1)
        if k:
            check(k - 1, h.state_download_wait((k - 1) & 1))
    check(n_frames - 1, h.state_download_wait((n_frames - 1) & 1))
    h.close()
