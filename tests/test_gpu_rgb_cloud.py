"""GPU tier: publish_frame_world_rgb's laserCloudWorldRGB built on the device as pcl::PointXYZRGB records
(flb_rgb_cloud) and the run's pcl_wait_save kept there (flb_rgb_save_*).

flb_rgb_cloud must equal flb_colorize_cloud's valid points, compacted in world-cloud order and packed in numpy, byte for
byte: over the visual-map scenarios with both world-cloud sources, with the colour frame of the image set (bgr NULL)
and a caller's bgr, at explicit poses and at the device state.  The save must equal the frame clouds concatenated in
call order, past one 2^20-record chunk too; its cap drops whole frames and counts them while the frame cloud is still
built.  Each FLB_ERR_STATE case is refused, and the LIO export survives the call."""
import ctypes as C

import numpy as np
import pytest

from test_vmap_select import SCENARIOS
from test_gpu_world_cloud import SOURCES, bgr_of, expect_error, source_cloud, visual_handle

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4


def packed_colorize(flb, h, Rcw, Pcw, bgr, xyz):
    """flb_colorize_cloud + compaction + packing: the records flb_rgb_cloud must return."""
    rgb, val = h.colorize_cloud(Rcw, Pcw, bgr)
    out = np.zeros(int(val.sum()), flb.capi.RGB_POINT)
    kept = xyz[val]
    out["x"], out["y"], out["z"] = kept[:, 0], kept[:, 1], kept[:, 2]
    out["w"] = 1.0
    out["r"], out["g"], out["b"] = rgb[val, 0], rgb[val, 1], rgb[val, 2]
    out["a"] = 255
    return out


def prm_of(flb, seq):
    return flb.capi.lio_params(dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"]), 3)


# ------------------------------------------------------------------------------------------------ the frame's cloud
@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("sc", SCENARIOS, ids=lambda s: f"{s[0]}-g{s[2]}-thr{s[3]}-ncc{s[4]}-step{s[6][0]}")
def test_rgb_cloud_equals_colorize_cloud(flb, po, sc, src):
    name, nf, grid, thr, ncc_en, ncc_thre, step, yaw = sc
    seq = flb.synth.make_visual_sequence(name, nf, step=step, yaw_step_deg=yaw)
    prm = prm_of(flb, seq)
    h = flb.Handle(device=0)
    h.camera_set(seq["cam"])
    h.image_upload(seq["frames"][0]["image"])
    h.vmap_reset(seq, grid_size=grid, outlier_threshold=thr, ncc_en=ncc_en, ncc_thre=ncc_thre)
    kept = 0
    for k, fr in enumerate(seq["frames"]):
        source_cloud(flb, h, src, fr["scan_body"], 80 + k)
        x = flb.capi.State18.make(fr["R"], fr["p"], cov=seq["cov"])
        h.state_upload(x, x.copy())
        n = h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED, fr["R"], fr["p"])
        xyz = h.world_cloud_download()
        assert n == len(xyz) > 0
        bgr = bgr_of(fr["image"], k)
        h.image_upload_bgr(bgr_of(fr["image"], k + 100))
        for img in (None, bgr):                              # the image set's colour frame, the caller's frame
            for pose in ((fr["Rcw"], fr["Pcw"]), (None, None)):
                ref = packed_colorize(flb, h, *pose, img, xyz)
                m = h.rgb_cloud(*pose, img)
                got = h.rgb_cloud_download()
                assert m == len(got) == len(ref)
                assert got.tobytes() == ref.tobytes()
                kept += m
    assert kept > 100
    h.close()


# ------------------------------------------------------------------------------------------------ the save
def body_in_view(flb, seq, fr, n, seed):
    """n body points whose world transform at (R, p) lies in front of the camera, inside its image (pinhole)."""
    cam = seq["cam"]
    rng = np.random.default_rng(seed)
    u, v, d = rng.uniform(-0.5, cam["width"], n), rng.uniform(-0.5, cam["height"], n), rng.uniform(1.0, 30.0, n)
    pc = np.stack([(u - cam["cx"]) / cam["fx"] * d, (v - cam["cy"]) / cam["fy"] * d, d], 1)
    pw = (pc - fr["Pcw"]) @ fr["Rcw"]
    return np.ascontiguousarray(((pw - fr["p"]) @ fr["R"] - seq["t_LI"]) @ seq["R_LI"], np.float32)


def run_frames(flb, seq, bodies, save_max=None, fidx=None):
    """One handle; per body: scan upload, world cloud, flb_rgb_cloud (frame fidx[k]'s pose, its image as the image
    set's colour frame).  Returns the frame clouds, the save's size and its whole download (or None without a save),
    and the handle."""
    prm = prm_of(flb, seq)
    h = visual_handle(flb, seq)
    if save_max is not None:
        h.rgb_save_begin(save_max)
    clouds = []
    for k, body in enumerate(bodies):
        fr = seq["frames"][k % len(seq["frames"]) if fidx is None else fidx[k]]
        h.scan_upload(body)
        h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
        h.image_upload_bgr(bgr_of(fr["image"], k))
        h.rgb_cloud(fr["Rcw"], fr["Pcw"])
        clouds.append(h.rgb_cloud_download())
    if save_max is None:
        return clouds, None, None, h
    return clouds, h.rgb_save_size(), h.rgb_save_download(), h


def test_save_is_the_frames_concatenated(flb, po):
    seq = flb.synth.make_visual_sequence("T0", 3)
    bodies = [fr["scan_body"] for fr in seq["frames"]] + [np.zeros((0, 3), np.float32), seq["frames"][0]["scan_body"]]
    clouds, size, whole, h = run_frames(flb, seq, bodies, save_max=1 << 40)
    h.close()
    ref, _, _, h2 = run_frames(flb, seq, bodies)
    h2.close()
    assert [c.tobytes() for c in clouds] == [c.tobytes() for c in ref]
    assert size["n"] == sum(len(c) for c in clouds) > 100 and size["dropped"] == 0
    assert size["device_bytes"] >= 16 << 20
    assert whole.tobytes() == np.concatenate(clouds).tobytes()


def test_save_past_one_chunk(flb, po):
    """Six frames of a 200 k-point scan cloud: more than 2^20 records, so the save spans two chunks; the whole save and
    slices across the chunk boundary equal the frame clouds concatenated."""
    seq = flb.synth.make_visual_sequence("T0", 2)
    bodies = [body_in_view(flb, seq, seq["frames"][k % 2], 200_000, 90 + k) for k in range(6)]
    clouds, size, whole, h = run_frames(flb, seq, bodies, save_max=1 << 40)
    cat = np.concatenate(clouds)
    assert size["n"] == len(cat) > 1 << 20 and size["dropped"] == 0
    assert size["device_bytes"] >= 2 * (16 << 20)
    assert whole.tobytes() == cat.tobytes()
    c = 1 << 20
    for first, count in [(c - 1, 2), (c - 300_000, 400_000), (len(cat) - 1, 1), (0, 0)]:
        assert h.rgb_save_download(first, count).tobytes() == cat[first:first + count].tobytes()
    h.close()


def test_save_cap_drops_whole_frames(flb, po):
    seq = flb.synth.make_visual_sequence("T0", 2)
    b1 = seq["frames"][1]["scan_body"]
    bodies, fidx = [seq["frames"][0]["scan_body"], b1, b1[: len(b1) // 3]], [0, 1, 1]   # the third: a part of the second
    ref, _, _, h = run_frames(flb, seq, bodies, fidx=fidx)
    h.close()
    n1, n2, n3 = map(len, ref)
    assert n2 > n3 > 10 and n1 > 10
    cap = n1 + n3                                            # the second frame passes the cap, the third fits
    clouds, size, whole, h = run_frames(flb, seq, bodies, save_max=cap, fidx=fidx)
    assert [c.tobytes() for c in clouds] == [c.tobytes() for c in ref]    # every frame cloud is still built
    assert size["n"] == n1 + n3 and size["dropped"] == n2
    assert whole.tobytes() == np.concatenate([ref[0], ref[2]]).tobytes()
    h.rgb_save_end()
    expect_error(flb, ERR_STATE, h.rgb_save_size)
    expect_error(flb, ERR_STATE, h.rgb_save_download, 0, 0)
    h.rgb_save_end()                                         # nothing open: nothing to do
    h.rgb_save_begin(1)                                      # a fresh save: a frame of more than one point is dropped
    assert h.rgb_cloud(seq["frames"][1]["Rcw"], seq["frames"][1]["Pcw"]) == n3
    assert h.rgb_save_size()["n"] == 0 and h.rgb_save_size()["dropped"] == n3
    h.close()


# ------------------------------------------------------------------------------------------------ errors
def test_errors(flb, po):
    seq = flb.synth.make_visual_sequence("T0", 2)
    prm = prm_of(flb, seq)
    fr = seq["frames"][1]
    bgr = bgr_of(fr["image"], 0)
    # no camera
    h = flb.Handle(device=0)
    h.scan_upload(fr["scan_body"])
    h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
    expect_error(flb, ERR_STATE, h.rgb_cloud, fr["Rcw"], fr["Pcw"], bgr)
    h.close()
    h = visual_handle(flb, seq)                              # camera, gray image, visual map
    expect_error(flb, ERR_STATE, h.rgb_cloud_download)      # nothing built yet
    # no world cloud
    expect_error(flb, ERR_STATE, h.rgb_cloud, fr["Rcw"], fr["Pcw"], bgr)
    h.scan_upload(fr["scan_body"])
    assert h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"]) > 0
    ok = lambda: h.rgb_cloud(fr["Rcw"], fr["Pcw"], bgr) > 0 and len(h.rgb_cloud_download()) > 0
    # no colour frame with bgr == NULL (the current image came from flb_image_upload)
    assert ok()
    expect_error(flb, ERR_STATE, h.rgb_cloud, fr["Rcw"], fr["Pcw"], None)
    expect_error(flb, ERR_STATE, h.rgb_cloud_download)      # on any error no cloud is held
    # a caller's bgr with a short stride
    assert ok()
    n = C.c_int()
    assert h.L.flb_rgb_cloud(h.h, None, None, bgr.ctypes.data_as(C.c_void_p), 3 * seq["cam"]["width"] - 1, C.byref(n)) == ERR_INVALID
    expect_error(flb, ERR_STATE, h.rgb_cloud_download)
    # no pose source: no pose given and no flb_vmap_reset
    h2 = flb.Handle(device=0)
    h2.camera_set(seq["cam"])
    h2.image_upload_bgr(bgr)
    h2.scan_upload(fr["scan_body"])
    h2.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
    expect_error(flb, ERR_STATE, h2.rgb_cloud, None, None, None)
    assert h2.rgb_cloud(fr["Rcw"], fr["Pcw"], None) > 0
    h2.close()
    # the world cloud refused: so is the coloured cloud
    assert ok()
    expect_error(flb, ERR_INVALID, h.world_cloud, prm, flb.capi.CLOUD_SCAN, fr["R"], np.asarray(fr["p"]) + [1e39, 0, 0])
    expect_error(flb, ERR_STATE, h.rgb_cloud, fr["Rcw"], fr["Pcw"], bgr)
    # a world cloud of 0 points: 0 records, no pose needed
    h.scan_upload(np.zeros((0, 3), np.float32))
    assert h.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"]) == 0
    assert h.rgb_cloud(None, None, bgr) == 0 and len(h.rgb_cloud_download()) == 0
    # the save's own refusals
    expect_error(flb, ERR_INVALID, h.rgb_save_begin, 0)
    expect_error(flb, ERR_STATE, h.rgb_save_size)
    h.rgb_save_begin(10)
    expect_error(flb, ERR_STATE, h.rgb_save_begin, 10)
    for first, count in [(-1, 0), (0, -1), (0, 1), (1, 0)]:
        expect_error(flb, ERR_INVALID, h.rgb_save_download, first, count)
    h.rgb_save_end()
    h.close()


# ------------------------------------------------------------------------------------------------ the LIO export survives
def lio_export(h, width=6):
    N = h.N
    bufs = [np.zeros((N, 3), np.float32), np.zeros((N, 5), np.int32), np.zeros((N, 5), np.float32), np.zeros((N, 4), np.float32),
            np.zeros(N, np.float32), np.zeros(N, np.uint8), np.zeros((N, width)), np.zeros(N), np.zeros(N, np.int32)]
    n = C.c_int()
    rc = h.L.flb_lio_export(h.h, *[b.ctypes.data_as(C.c_void_p) for b in bufs], C.byref(n))
    return rc, [b.tobytes() for b in bufs], n.value


def test_lio_export_survives(flb, po, frames):
    f = frames("T0")
    seq = flb.synth.make_visual_sequence("T0", 1)
    fr = seq["frames"][0]
    prm = flb.capi.lio_params(f, 3)
    out = []
    for colour in (False, True):
        h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
        h.camera_set(seq["cam"])
        h.image_upload_bgr(bgr_of(fr["image"], 0))
        h.map_upload(f["map_xyz"])
        h.scan_upload(f["scan_body"])
        h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_prop"], f["p_prop"])
        h.lio_pass(prm, f["R_prop"], f["p_prop"], True, export=False)
        if colour:
            h.rgb_cloud(fr["Rcw"], fr["Pcw"])
        out.append(lio_export(h))
        h.close()
    assert out[0][0] == out[1][0] == 0 and out[0][2] > 0
    assert out[0] == out[1]
