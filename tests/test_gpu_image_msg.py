"""GPU tier: the camera message taken in the driver's encoding (flb_image_upload_msg: cv_bridge's conversion to bgr8,
then LidarSelector::detect's resize + cvtColor, src/lidar_selection.cpp:1029-1037, on the device).

- Every case of tests/golden/image_msg_golden.npz gives cv2's colour frame and gray image byte for byte, from pageable
  and page-locked sources, for FLB_GRAY_CV4 and, where the rule takes it, FLB_GRAY_CV3.
- FLB_ENC_BGR8 equals flb_image_upload_bgr byte for byte.
- A C2-sized sequence (select_cloud -> grow_cloud -> VIO update -> colorize_cloud with bgr NULL) after a Bayer upload
  with odd sides equals the same sequence after flb_image_upload_bgr of the converted, resized frame, bit for bit.
- Every error leaves the previous image set current; uploads around a running VIO update do not disturb it."""
import numpy as np
import pytest

from test_image_msg import golden, golden_names, is_linear, np_demosaic, np_resize_linear
from test_image_prep import cv3_rule

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
CV4, CV3 = 0, 1
LEAF = 0.2


def camera(W, H):
    return dict(width=W, height=H, fx=0.6 * W, fy=0.6 * W, cx=0.5 * W, cy=0.5 * H, d=[0.0] * 5)


def message_view(rows, w, h, bpp):
    """The message held in `rows` (h x step bytes, pixels first) as a (h, w, bpp) view with the rows' step."""
    return np.lib.stride_tricks.as_strided(rows, (h, w, bpp), (rows.strides[0], bpp, 1))


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


# ------------------------------------------------------------------------------------------------ the image set itself
@pytest.mark.parametrize("source", ["pageable", "pinned"])
@pytest.mark.parametrize("name", golden_names())
def test_golden(flb, name, source):
    rows, (w, h, W, H, enc, bpp), bgr, gray = golden(name)
    hd = flb.Handle(device=0)
    hd.camera_set(camera(W, H))
    if source == "pinned":
        rows = hd.pinned_like(rows)
    rules = [CV4] if is_linear(w, h, W, H) else [CV4, CV3]
    for rule in rules:
        hd.image_upload_msg(message_view(rows, w, h, bpp), enc, rule)
        hd.synchronize()
        g, c = hd.image_download()
        assert np.array_equal(c, bgr)
        assert np.array_equal(g, gray if rule == CV4 else cv3_rule(bgr))
    hd.close()


@pytest.mark.parametrize("scale", [1, 2])
def test_bgr8_equals_upload_bgr(flb, scale):
    seq = flb.synth.make_visual_sequence("T0", 1)
    cam = seq["cam"]
    src = flb.synth.texture_bgr(seq["frames"][0]["image"], scale * cam["width"], scale * cam["height"])
    src = src ^ np.random.default_rng(scale).integers(0, 8, src.shape, dtype=np.uint8)
    out = []
    for path in ("msg", "bgr"):
        hd = flb.Handle(device=0)
        hd.camera_set(cam)
        for rule in (CV4, CV3):
            if path == "msg":
                hd.image_upload_msg(src, "bgr8", rule)
            else:
                hd.image_upload_bgr(src, rule)
            out.append(hd.image_download())
        hd.close()
    for (ga, ca), (gb, cb) in zip(out[:2], out[2:]):
        assert ga.tobytes() == gb.tobytes() and ca.tobytes() == cb.tobytes()


# ------------------------------------------------------------------------------------------------ readers of the image
def test_c2_bayer_sequence_equals_bgr_upload(flb):
    """detect() per frame on the C2 camera (640 x 512) from a 1281 x 1025 bayer_grbg8 message: A takes the message,
    B flb_image_upload_bgr of its demosaiced, linearly resized frame (the numpy statements the CPU tier checks against
    cv2).  Selection, growth, state, errors, map values and colours bit-identical."""
    seq = flb.synth.make_visual_sequence("C2", 3)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 4)
    cam = seq["cam"]
    W, H = cam["width"], cam["height"]
    grid = 16
    L = (W // grid) * (H // grid)
    hs = [flb.Handle(device=0) for _ in range(2)]
    for h in hs:
        h.camera_set(cam)
        h.image_upload(seq["frames"][0]["image"])
        h.vmap_reset(seq, grid_size=grid, outlier_threshold=300.0)
    out = [[], []]
    for k, fr in enumerate(seq["frames"]):
        mosaic = flb.synth.bayer_message(flb.synth.texture_bgr(fr["image"], 2 * W + 1, 2 * H + 1), "bayer_grbg8")
        bgr = np_resize_linear(np_demosaic(mosaic, 8), W, H)
        x0 = flb.capi.State18.make(fr["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr["p"] + [0.02, -0.015, 0.01],
                                   cov=seq["cov"])
        for i, h in enumerate(hs):
            if i == 0:
                h.image_upload_msg(mosaic, "bayer_grbg8")
            else:
                h.image_upload_bgr(bgr)
            h.scan_upload(fr["scan_body"])
            h.world_cloud(lprm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
            h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF)
            s = h.vmap_selected()
            h.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], k)
            g = h.vmap_counts()["last_added"]
            mv = h.vmap_map_value(L)
            h.state_upload(x0, x0.copy())
            if k > 0:
                h.vio_update_enqueue(vprm)
            x, _, vrep = h.state_download()
            errs = h.vio_errors() if k > 0 else np.zeros(0, np.float32)
            rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"], None)
            img = h.image_download()
            out[i].append((s, g, mv.tobytes(), bytes(x), bytes(vrep), errs.tobytes(), rgb.tobytes(), val.tobytes(),
                           img[0].tobytes(), img[1].tobytes()))
    for fa, fb in zip(*out):
        for key in fa[0]:
            assert fa[0][key].tobytes() == fb[0][key].tobytes(), key
        assert fa[1:] == fb[1:]
    assert min(len(fa[0]["index"]) for fa in out[0][1:]) > 10 and sum(fa[1] for fa in out[0]) > 0
    assert sum(np.frombuffer(fa[7], np.uint8).sum() for fa in out[0]) > 100
    da, db = hs[0].vmap_dump(), hs[1].vmap_dump()
    for key in da:
        assert da[key].tobytes() == db[key].tobytes(), key
    for h in hs:
        h.close()


def test_uploads_around_a_running_update(flb, frames):
    """A message upload enqueued while the VIO update runs, and another after it, leave that update's result equal to
    the same update with no upload in flight; each upload then becomes the current image."""
    f = frames("T1")
    vprm = flb.capi.vio_params(f, 3)
    pos = np.ascontiguousarray(f["patch_pos"], np.float64)
    ref = np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(pos), 192)
    lev = np.ascontiguousarray(f["patch_level"], np.int32)
    cam = f["cam"]
    W, H = cam["width"], cam["height"]
    others = [flb.synth.bayer_message(flb.synth.texture_bgr(255 - f["image"], 2 * W + 1, 2 * H), "bayer_rggb8"),
              flb.synth.mono_message(flb.synth.texture_bgr(np.roll(f["image"], 9, 0), 2 * W, 2 * H + 1))]
    results = []
    for in_flight in (False, True):
        h = flb.Handle(device=0)
        h.camera_set(cam)
        h.image_upload(f["image"])
        h.patches_upload(pos, ref, lev)
        x0 = flb.capi.State18.from_frame(f)
        h.state_upload(x0, x0.copy())
        h.vio_update_enqueue(vprm)
        if in_flight:
            pinned = h.pinned_like(others[0])
            h.image_upload_msg(pinned, "bayer_rggb8")
        results.append(h.state_download())
        if in_flight:
            h.image_upload_msg(others[1], "mono8")
            g, c = h.image_download()
            assert (c[..., 0] == c[..., 1]).all() and (c[..., 1] == c[..., 2]).all() and (g == c[..., 0]).all()
        h.close()
    (xa, _, va), (xb, _, vb) = results
    assert (xa.vector() == xb.vector()).all() and (np.array(xa.cov[:]) == np.array(xb.cov[:])).all()
    assert va.rows_total == vb.rows_total and list(va.passes) == list(vb.passes)


# ------------------------------------------------------------------------------------------------ errors
def test_errors_keep_the_previous_image(flb):
    rows, (w, h_, W, H, enc, bpp), bgr, gray = golden("bayer_rggb8__oddwh")
    src = message_view(rows, w, h_, bpp)
    hd = flb.Handle(device=0)
    raw = hd.L.flb_image_upload_msg
    expect_error(flb, ERR_STATE, hd.image_upload_msg, src, enc)                           # no camera
    hd.camera_set(camera(W, H))
    hd.image_upload_msg(src, enc)

    def unchanged():
        g, c = hd.image_download()
        assert np.array_equal(g, gray) and np.array_equal(c, bgr)
    unchanged()
    a = np.ascontiguousarray(src[..., 0])
    rgb = np.zeros((H, W, 3), np.uint8)
    for bad in (lambda: hd.image_upload_msg(a[:, :-2], enc),                          # 2W - 1 wide
                lambda: hd.image_upload_msg(a[:-2], enc),                             # 2H - 1 high
                lambda: hd.image_upload_msg(np.zeros((H + 1, W), np.uint8), enc),
                lambda: hd.image_upload_msg(np.zeros((4 * H, 4 * W), np.uint8), enc),
                lambda: hd.image_upload_msg(a, enc, CV3),                             # odd sides: no OpenCV 3 rule
                lambda: hd.image_upload_msg(a, enc, 2),
                lambda: hd.image_upload_msg(a, 9), lambda: hd.image_upload_msg(a, -1),
                lambda: hd._ck(raw(hd.h, rgb.ctypes.data, W, H, 3 * W - 1, 1, CV4)),   # step below the row
                lambda: hd._ck(raw(hd.h, a.ctypes.data, w, h_, w - 1, enc, CV4)),
                lambda: hd._ck(raw(hd.h, None, w, h_, w, enc, CV4))):
        expect_error(flb, ERR_INVALID, bad)
        unchanged()
    hd.close()
