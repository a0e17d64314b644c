"""GPU tier: the camera frame prepared on the device (flb_image_upload_bgr: LidarSelector::detect's resize + cvtColor,
src/lidar_selection.cpp:1029-1037) and the colouring that reads its colour frame (flb_colorize / flb_colorize_cloud
with bgr == NULL).

- The image set equals cv2's outputs recorded in tests/golden/image_golden.npz, at 1x and 2x, for both gray rules,
  from pageable, strided and page-locked sources; a 4096 x 4096 frame of every colour gives the integer rules' gray.
- Everything that reads the image (VIO update, visual map, keyframes) is bit-identical to flb_image_upload of the
  same gray image, over multi-frame sequences, and the NULL colouring equals the host-BGR colouring.
- Frames with distinct inputs uploaded while the previous update runs equal the same frames run one at a time.
- Every error leaves the previous image set current."""
import ctypes as C

import numpy as np
import pytest

from test_image_prep import GOLDEN, cv3_rule, cv4_rule, every_colour

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
CV4, CV3 = 0, 1
LEAF = 0.2


def rule_gray(bgr, rule):
    return cv4_rule(bgr) if rule == CV4 else cv3_rule(bgr)


def halve(a):
    """OpenCV's resize(0.5, INTER_LINEAR) of an even-sized frame: the rounded mean of each 2x2 block, per channel."""
    s = a.astype(np.uint16)
    return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)


def camera(W, H):
    return dict(width=W, height=H, fx=0.6 * W, fy=0.6 * W, cx=0.5 * W, cy=0.5 * H, d=[0.0] * 5)


def strided_view(rows, w, h):
    """The (h, w, 3) frame held in `rows` (h x stride bytes, pixels first) as a view with the rows' stride."""
    return np.lib.stride_tricks.as_strided(rows, (h, w, 3), (rows.strides[0], 3, 1))


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def golden(name):
    g = np.load(GOLDEN)
    w, h, W, H = (int(v) for v in g[f"{name}__size"])
    return g[f"{name}__rows"], (w, h, W, H), g[f"{name}__bgr"], g[f"{name}__gray"]


# ------------------------------------------------------------------------------------------------ the image set itself
@pytest.mark.parametrize("source", ["pageable", "pinned"])
@pytest.mark.parametrize("rule", [CV4, CV3])
@pytest.mark.parametrize("name", [str(n) for n in np.load(GOLDEN)["names"]])
def test_golden(flb, name, rule, source):
    rows, (w, h, W, H), bgr, gray = golden(name)
    hd = flb.Handle(device=0)
    hd.camera_set(camera(W, H))
    if source == "pinned":
        rows = hd.pinned_like(rows)
    hd.image_upload_bgr(strided_view(rows, w, h), rule)
    hd.synchronize()
    g, c = hd.image_download()
    assert np.array_equal(c, bgr)
    assert np.array_equal(g, gray if rule == CV4 else cv3_rule(bgr))
    hd.close()


@pytest.mark.parametrize("rule", [CV4, CV3])
def test_every_colour(flb, rule):
    img = every_colour()
    hd = flb.Handle(device=0)
    hd.camera_set(camera(4096, 4096))
    hd.image_upload_bgr(img, rule)
    g, c = hd.image_download()
    assert np.array_equal(c, img) and np.array_equal(g, rule_gray(img, rule))
    hd.close()


# ------------------------------------------------------------------------------------------------ readers of the image
def frame_bgr(img, k, scale):
    """A BGR camera frame at `scale` x the camera size whose channels follow the sequence's gray image."""
    rng = np.random.default_rng(100 + k)
    bgr = np.stack([img, np.roll(img, 3, 1), 255 - img], -1)
    if scale == 2:
        bgr = np.repeat(np.repeat(bgr, 2, 0), 2, 1)
    return np.ascontiguousarray(bgr ^ rng.integers(0, 16, bgr.shape, dtype=np.uint8))


@pytest.mark.parametrize("rule", [CV4, CV3])
@pytest.mark.parametrize("scale", [1, 2])
def test_visual_sequence_equals_gray_upload(flb, scale, rule):
    """detect() per frame (select -> grow -> VIO update -> add_observations -> colorize) on A from flb_image_upload_bgr
    and on B from flb_image_upload of the same gray image: every output bit-identical."""
    seq = flb.synth.make_visual_sequence("T0", 4)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
    vprm = flb.capi.vio_params(f, 4)
    grid = 16
    L = (seq["cam"]["width"] // grid) * (seq["cam"]["height"] // grid)
    a, b, scratch = flb.Handle(device=0), flb.Handle(device=0), flb.Handle(device=0)
    for h in (a, b):
        h.camera_set(seq["cam"])
        h.image_upload(seq["frames"][0]["image"])
        h.vmap_reset(seq, grid_size=grid, outlier_threshold=300.0)
    out = [[], []]
    for k, fr in enumerate(seq["frames"]):
        src = frame_bgr(fr["image"], k, scale)
        bgr = halve(src) if scale == 2 else src
        gray = rule_gray(bgr, rule)
        pg_down = scratch.voxel_grid(fr["pg"], LEAF)
        x0 = flb.capi.State18.make(fr["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr["p"] + [0.02, -0.015, 0.01],
                                   cov=seq["cov"])
        for i, h in enumerate((a, b)):
            if i == 0:
                h.image_upload_bgr(src, rule)
            else:
                h.image_upload(gray)
            h.vmap_select(fr["Rcw"], fr["Pcw"], pg_down)
            s = h.vmap_selected()
            h.vmap_grow(fr["Rcw"], fr["Pcw"], fr["pg"], k)
            g = h.vmap_counts()["last_added"]
            mv = h.vmap_map_value(L)
            h.state_upload(x0, x0.copy())
            if k > 0:
                h.vio_update_enqueue(vprm)
            h.vmap_add_observations(None, None, k)
            x, _, vrep = h.state_download()
            errs = h.vio_errors() if k > 0 else np.zeros(0, np.float32)
            rgb, val = h.colorize(fr["Rcw"], fr["Pcw"], None if i == 0 else bgr, fr["pg"])
            out[i].append((s, g, mv.tobytes(), bytes(x), bytes(vrep), errs.tobytes(), rgb.tobytes(), val.tobytes()))
    for fa, fb in zip(*out):
        for key in fa[0]:
            assert fa[0][key].tobytes() == fb[0][key].tobytes(), key
        assert fa[1:] == fb[1:]
    assert min(len(fa[0]["index"]) for fa in out[0][1:]) > 10 and sum(fa[1] for fa in out[0]) > 0
    da, db = a.vmap_dump(), b.vmap_dump()
    for key in da:
        assert da[key].tobytes() == db[key].tobytes(), key
    n_img = a.vmap_counts()["images"]
    assert n_img == b.vmap_counts()["images"] > 1
    for slot in range(n_img):
        assert a.vmap_keyframe(slot).tobytes() == b.vmap_keyframe(slot).tobytes()
    for h in (a, b, scratch):
        h.close()


@pytest.mark.parametrize("scale", [1, 2])
def test_colorize_null_equals_host_bgr(flb, scale):
    seq = flb.synth.make_visual_sequence("T0", 2)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    fr = seq["frames"][1]
    h = flb.Handle(device=0)
    h.camera_set(seq["cam"])
    h.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
    h.scan_upload(fr["scan_body"])
    h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
    src = frame_bgr(fr["image"], 1, scale)
    bgr = halve(src) if scale == 2 else src
    h.image_upload_bgr(src)
    for R, P in ((fr["Rcw"], fr["Pcw"]), (None, None)):
        if R is None:
            h.state_upload(flb.capi.State18.make(fr["R"], fr["p"], cov=seq["cov"]), flb.capi.State18.make(fr["R"], fr["p"], cov=seq["cov"]))
        dev = h.colorize_cloud(R, P)
        host = h.colorize_cloud(R, P, bgr)
        assert dev[0].tobytes() == host[0].tobytes() and (dev[1] == host[1]).all() and dev[1].sum() > 100
        dev = h.colorize(R, P, None, fr["pg"])
        host = h.colorize(R, P, bgr, fr["pg"])
        assert dev[0].tobytes() == host[0].tobytes() and (dev[1] == host[1]).all() and dev[1].sum() > 100
    h.close()


# ------------------------------------------------------------------------------------------------ pipelining
def test_pipelined_frames_with_distinct_inputs(flb, frames):
    """Six frames whose inputs all differ.  (a) one at a time through flb_image_upload of the numpy gray, blocking;
    (b) flb_image_upload_bgr of a page-locked 2x frame, then flb_frame_enqueue with gray == NULL, three frames in flight
    over two result slots; (c) the separate enqueue calls with pageable 1x frames.  Every frame bit-identical to (a)."""
    f = frames("T1")
    lprm, vprm = flb.capi.lio_params(f, 3), flb.capi.vio_params(f, 3)
    rng = np.random.default_rng(78)
    n_frames = 6
    base_scan = np.ascontiguousarray(f["scan_body"], np.float32)
    pos = np.ascontiguousarray(f["patch_pos"], np.float64)
    ref = np.ascontiguousarray(f["patch_ref"], np.float32).reshape(len(pos), 192)
    lev = np.ascontiguousarray(f["patch_level"], np.int32)
    inputs = []
    for k in range(n_frames):
        scan = base_scan + rng.normal(0, 0.004 * k, base_scan.shape).astype(np.float32)
        src = frame_bgr(np.clip(f["image"].astype(np.int32) + rng.integers(-3 * k, 3 * k + 1, f["image"].shape), 0, 255).astype(np.uint8),
                        k, 2)
        x0 = flb.capi.State18.from_frame(f)
        x0.pos[0] += 0.003 * k
        inputs.append((scan, src, x0))

    def fresh():
        h = flb.Handle(device=0)
        h.map_upload(f["map_xyz"])
        h.camera_set(f["cam"])
        return h
    h = fresh()
    serial = []
    for scan, src, x0 in inputs:
        h.scan_upload(scan)
        h.image_upload(cv4_rule(halve(src)))
        h.patches_upload(pos, ref, lev)
        h.state_upload(x0, x0.copy())
        h.lio_update_enqueue(lprm)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
        serial.append(h.state_download())
    h.close()
    assert len({tuple(x.vector()) for x, _, _ in serial}) == n_frames

    def check(k, got):
        xk, lk, vk = got
        xs, ls, vs = serial[k]
        assert (xk.vector() == xs.vector()).all() and (np.array(xk.cov[:]) == np.array(xs.cov[:])).all(), f"frame {k}"
        assert lk.rows_total == ls.rows_total and vk.rows_total == vs.rows_total and list(vk.passes) == list(vs.passes)
    h = fresh()
    bufs = [(h.pinned_like(scan), h.pinned_like(src), x0) for scan, src, x0 in inputs]
    pp, pr, pl = h.pinned_like(pos), h.pinned_like(ref), h.pinned_like(lev)
    fis = [h.frame_inputs(scan, x0, x0.copy(), None, pp, pr, pl) for scan, _, x0 in bufs]
    for k in range(n_frames):
        h.image_upload_bgr(bufs[k][1])                     # while frame k - 1's updates still run
        h.frame_enqueue(fis[k], lprm, vprm, k & 1)
        if k:
            check(k - 1, h.state_download_wait((k - 1) & 1))
    check(n_frames - 1, h.state_download_wait((n_frames - 1) & 1))
    h.close()
    h = fresh()
    h.patches_upload(pos, ref, lev)
    for k in range(n_frames):
        scan, src, x0 = inputs[k]
        h.scan_upload(scan)
        h.state_upload(x0, x0.copy())
        h.lio_update_enqueue(lprm)
        h.image_upload_bgr(np.ascontiguousarray(halve(src)))
        h.patches_upload(pos, ref, lev)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
        h.state_download_enqueue(k & 1)
        if k:
            check(k - 1, h.state_download_wait((k - 1) & 1))
    check(n_frames - 1, h.state_download_wait((n_frames - 1) & 1))
    h.close()


# ------------------------------------------------------------------------------------------------ errors
def test_errors_keep_the_previous_image(flb):
    rows, (w, h_, W, H), bgr, gray = golden("texture_2x_strided")
    src = strided_view(rows, w, h_)
    hd = flb.Handle(device=0)
    raw = hd.L.flb_image_upload_bgr
    expect_error(flb, ERR_STATE, hd.image_upload_bgr, src)                       # no camera
    hd.camera_set(camera(W, H))
    expect_error(flb, ERR_STATE, hd.image_download)                             # no image yet
    hd.image_upload_bgr(src)

    def unchanged():
        g, c = hd.image_download()
        assert np.array_equal(g, gray) and np.array_equal(c, bgr)
    unchanged()
    a = np.ascontiguousarray(src)
    for bad in (lambda: hd.image_upload_bgr(a[:, :-2]), lambda: hd.image_upload_bgr(a[:-2]),
                lambda: hd.image_upload_bgr(a[:-1, :-1]), lambda: hd.image_upload_bgr(np.zeros((H + 1, W, 3), np.uint8)),
                lambda: hd.image_upload_bgr(np.zeros((4 * H, 4 * W, 3), np.uint8)),
                lambda: hd.image_upload_bgr(a, 2), lambda: hd.image_upload_bgr(a, -1),
                lambda: hd._ck(raw(hd.h, a.ctypes.data, w, h_, 3 * w - 1, CV4)),
                lambda: hd._ck(raw(hd.h, None, w, h_, 3 * w, CV4))):
        expect_error(flb, ERR_INVALID, bad)
        unchanged()
    # a download too small for the image
    g = np.zeros(W * H - 1, np.uint8)
    expect_error(flb, ERR_INVALID, lambda: hd._ck(hd.L.flb_image_download(hd.h, g.ctypes.data, None, W * H - 1, None, None)))
    # a gray upload: no colour frame, the NULL colouring and the colour download refuse
    hd.image_upload(gray)
    assert np.array_equal(hd.image_download(bgr=False)[0], gray)
    expect_error(flb, ERR_STATE, hd.image_download)
    seq = flb.synth.make_visual_sequence("T0", 1)
    fr = seq["frames"][0]
    expect_error(flb, ERR_STATE, hd.colorize, fr["Rcw"], fr["Pcw"], None, fr["pg"])
    expect_error(flb, ERR_STATE, hd.colorize, fr["Rcw"], fr["Pcw"], None, np.zeros((0, 3), np.float32))
    hd.image_upload_bgr(src)
    unchanged()
    assert hd.colorize(fr["Rcw"], fr["Pcw"], None, fr["pg"])[1].shape == (len(fr["pg"]),)
    # a camera of another size after the upload: the colour frame no longer matches it
    hd.camera_set(camera(W // 2, H // 2))
    expect_error(flb, ERR_STATE, hd.colorize, fr["Rcw"], fr["Pcw"], None, fr["pg"])
    hd.close()
