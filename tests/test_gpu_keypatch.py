"""GPU tier: flb_keypatch_image, LidarSelector::display_keypatch's circles (src/lidar_selection.cpp:985-1005) drawn on the
device into a copy of the current colour frame.

- Multi-frame C2 sequences (640 x 512 camera) in both execution modes, each frame taken with flb_image_upload_msg (a
  2W+1 x 2H+1 Bayer mosaic, a 1x bgr8 frame, a 2W x 2H+1 mono8 frame) and run through world cloud -> select -> grow ->
  VIO update -> add_observations.  The frame equals the numpy restatement of tests/test_keypatch.py byte for byte, from
  flb_image_download's colour frame, flb_vmap_selected's positions, flb_vio_errors and the downloaded state projected
  through the oracle's world2cam; before the VIO update it carries the selection's errors; explicit poses shifted so
  that circles cross and leave every border agree too.
- A patch list from flb_patches_upload; page-locked (enqueue-only) and pageable outputs; the colour frame and
  flb_colorize_cloud's output unchanged by the call; a zero-patch list; the documented errors, with nothing written.
The multi-GPU refusal needs flb_comm_init / flb_p2p_attach and is not exercised on one GPU."""
import numpy as np
import pytest

import vio_edge_util as U
from test_keypatch import np_keypatch

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
LEAF = 0.2


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def centres(po, cam, Rcw, Pcw, pos):
    """cv::Point2f(new_frame_->w2c(pos_i)): Rcw * pos + Pcw in the device's operation order, the oracle's world2cam, float."""
    pf = U._mv(np.asarray(Rcw, np.float64), np.asarray(pos, np.float64).reshape(-1, 3)) + np.asarray(Pcw, np.float64)
    pc = np.array([po.world2cam(cam, p) for p in pf]).reshape(-1, 2)
    return pc.astype(np.float32)


def pose_of_state(seq, x):
    Rci, Pci = U.extrinsics(seq["R_LI"], seq["t_LI"], seq["Rcl"], seq["Pcl"])
    Rcw = U._mm(Rci, np.asarray(x.R, np.float64).T.copy())
    return Rcw, -U._mv(Rcw, np.asarray(x.p, np.float64)) + Pci


def message(flb, img, W, H, k):
    """Frame k of a sequence as the driver might deliver it: (pixels, encoding)."""
    s = flb.synth
    if k % 3 == 0:
        return s.bayer_message(s.texture_bgr(img, 2 * W + 1, 2 * H + 1), "bayer_grbg8"), "bayer_grbg8"
    if k % 3 == 1:
        return s.texture_bgr(img, W, H), "bgr8"
    return s.mono_message(s.texture_bgr(img, 2 * W, 2 * H + 1)), "mono8"


def shifted_poses(cam, Rcw, Pcw, pc_depth):
    """Poses moved sideways by a third of the frame, and by more, so that circles cross and leave every border."""
    z = float(np.median(pc_depth))
    out = []
    for fx, fy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1.4, 1.4), (-1.4, -1.4)):
        t = np.array([fx * z * cam["width"] / (3 * cam["fx"]), fy * z * cam["height"] / (3 * cam["fy"]), 0.0])
        out.append((Rcw, np.asarray(Pcw, np.float64) + t))
    return out


@pytest.mark.parametrize("persistent", [1, 0])
def test_sequence_equals_restatement(flb, po, persistent):
    seq = flb.synth.make_visual_sequence("C2", 4)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 4)
    cam = seq["cam"]
    W, H = cam["width"], cam["height"]
    h = flb.Handle(device=0, persistent=persistent)
    h.camera_set(cam)
    h.image_upload(seq["frames"][0]["image"])
    h.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
    pinned = h.pinned_like(np.zeros((H, W, 3), np.uint8))
    drawn = clipped = 0
    for k, fr in enumerate(seq["frames"]):
        msg, enc = message(flb, fr["image"], W, H, k)
        h.image_upload_msg(msg, enc)
        h.scan_upload(fr["scan_body"])
        h.world_cloud(lprm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
        h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF)
        s = h.vmap_selected()
        _, img = h.image_download()
        # before any VIO pass on this list: the selection's errors (:576)
        out, n = h.keypatch_image(fr["Rcw"], fr["Pcw"])
        assert n == len(s["pos"])
        assert np.array_equal(out, np_keypatch(img, centres(po, cam, fr["Rcw"], fr["Pcw"], s["pos"]), s["error"]))
        h.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], k)
        x0 = flb.capi.State18.make(fr["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr["p"] + [0.02, -0.015, 0.01],
                                   cov=seq["cov"])
        h.state_upload(x0, x0.copy())
        h.vio_update_enqueue(vprm)
        h.vmap_add_observations(None, None, k)
        rgb0, val0 = h.colorize_cloud(fr["Rcw"], fr["Pcw"], None)
        out, n = h.keypatch_image(out=pinned)                      # enqueue-only; the pose of ComputeJ from the state
        h.synchronize()
        got = pinned.copy()
        x, _, _ = h.state_download()
        errs = h.vio_errors()
        Rcw, Pcw = pose_of_state(seq, x)
        pc = centres(po, cam, Rcw, Pcw, s["pos"])
        want = np_keypatch(img, pc, errs)
        assert n == len(s["pos"]) and np.array_equal(got, want)
        assert np.array_equal(h.keypatch_image()[0], want)         # pageable: blocking, the same bytes
        drawn += int((got != img).any(2).sum())
        # the colour frame and the colouring read the undrawn img_rgb
        assert np.array_equal(h.image_download()[1], img)
        rgb1, val1 = h.colorize_cloud(fr["Rcw"], fr["Pcw"], None)
        assert np.array_equal(rgb0, rgb1) and np.array_equal(val0, val1)
        pf = U._mv(Rcw, s["pos"]) + Pcw
        for R2, P2 in shifted_poses(cam, Rcw, Pcw, pf[:, 2]) if len(pf) else ():
            pc2 = centres(po, cam, R2, P2, s["pos"])
            out2, _ = h.keypatch_image(R2, P2)
            assert np.array_equal(out2, np_keypatch(img, pc2, errs))
            inside = (pc2 >= -6).all(1) & (pc2[:, 0] <= W + 5) & (pc2[:, 1] <= H + 5)
            edge = inside & ((pc2 < 6).any(1) | (pc2[:, 0] > W - 7) | (pc2[:, 1] > H - 7))
            clipped += int(edge.sum())
    assert drawn > 1000 and clipped > 20
    h.close()


def test_patch_list_upload(flb, po, frames):
    f = frames("T1")
    vprm = flb.capi.vio_params(f, 3)
    pos = np.ascontiguousarray(f["patch_pos"], np.float64)
    ref = np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(pos), 192)
    lev = np.ascontiguousarray(f["patch_level"], np.int32)
    cam = f["cam"]
    W, H = cam["width"], cam["height"]
    h = flb.Handle(device=0)
    h.camera_set(cam)
    h.image_upload_msg(flb.synth.texture_bgr(f["image"], 2 * W, 2 * H), "bgr8")
    _, img = h.image_download()
    h.patches_upload(pos, ref, lev)
    Rci, Pci = U.extrinsics(f["R_LI"], f["t_LI"], f["Rcl"], f["Pcl"])
    x0 = flb.capi.State18.from_frame(f)
    Rcw = U._mm(Rci, np.asarray(x0.R).T.copy())
    Pcw = -U._mv(Rcw, np.asarray(x0.p)) + Pci
    out, n = h.keypatch_image(Rcw, Pcw)                            # no pass yet: the uploaded list's errors are zero
    assert n == len(pos)
    assert np.array_equal(out, np_keypatch(img, centres(po, cam, Rcw, Pcw, pos), np.zeros(len(pos), np.float32)))
    x = x0.copy()
    h.vio_update(vprm, x, x0.copy())
    errs = h.vio_errors()
    Rcw = U._mm(Rci, np.asarray(x.R).T.copy())
    Pcw = -U._mv(Rcw, np.asarray(x.p)) + Pci
    out, n = h.keypatch_image(Rcw, Pcw)
    assert np.array_equal(out, np_keypatch(img, centres(po, cam, Rcw, Pcw, pos), errs))
    assert (out != img).any()
    h.patches_upload(pos[:0], ref[:0], lev[:0])                    # zero patches: the frame unchanged, count 0
    out, n = h.keypatch_image(Rcw, Pcw)
    assert n == 0 and np.array_equal(out, img)
    h.close()


def test_errors_write_nothing(flb, frames):
    f = frames("T1")
    pos = np.ascontiguousarray(f["patch_pos"], np.float64)
    ref = np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(pos), 192)
    lev = np.ascontiguousarray(f["patch_level"], np.int32)
    cam = f["cam"]
    W, H = cam["width"], cam["height"]
    R, P = np.eye(3), np.zeros(3)
    h = flb.Handle(device=0)
    raw = h.L.flb_keypatch_image
    out = np.full((H, W, 3), 77, np.uint8)

    def unchanged():
        assert (out == 77).all()
    expect_error(flb, ERR_STATE, h.keypatch_image, R, P, out=out)                 # no camera
    unchanged()
    h.camera_set(cam)
    expect_error(flb, ERR_STATE, h.keypatch_image, R, P, out=out)                 # no image
    h.image_upload(f["image"])
    h.patches_upload(pos, ref, lev)
    expect_error(flb, ERR_STATE, h.keypatch_image, R, P, out=out)                 # gray only
    unchanged()
    h.close()
    h = flb.Handle(device=0)
    raw = h.L.flb_keypatch_image
    h.camera_set(cam)
    h.image_upload_msg(flb.synth.texture_bgr(f["image"], W, H), "bgr8")
    expect_error(flb, ERR_STATE, h.keypatch_image, R, P, out=out)                 # no patch list
    h.patches_upload(pos, ref, lev)
    expect_error(flb, ERR_STATE, h.keypatch_image, out=out)                       # no pose, no extrinsics / state
    unchanged()
    r9, p3 = np.ascontiguousarray(R), np.ascontiguousarray(P)
    for bad in (lambda: h._ck(raw(h.h, r9.ctypes.data, p3.ctypes.data, None, 3 * W, None)),
                lambda: h._ck(raw(h.h, r9.ctypes.data, p3.ctypes.data, out.ctypes.data, 3 * W - 1, None)),
                lambda: h._ck(raw(h.h, r9.ctypes.data, None, out.ctypes.data, 3 * W, None)),
                lambda: h._ck(raw(h.h, None, p3.ctypes.data, out.ctypes.data, 3 * W, None))):
        expect_error(flb, ERR_INVALID, bad)
        unchanged()
    got, n = h.keypatch_image(R, P, out=out)                                      # and then it works
    assert n == len(pos) and got is out
    h.close()
