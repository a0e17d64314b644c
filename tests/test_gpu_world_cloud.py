"""GPU tier: the frame's world cloud on the device (pcl_wait_pub, src/laserMapping.cpp:1763-1772) and the visual-map
steps that read it (flb_world_cloud, flb_vmap_select_cloud, flb_vmap_grow_cloud, flb_colorize_cloud).

Every test compares handle A, which builds the cloud on the device and calls the *_cloud entry points, with handle B,
which calls the host-input entry points on the oracle's pointBodyToWorld of the same source at the same pose, with
B's pg_down = flb_voxel_grid(pg, leaf) on a scratch handle.  Everything must be byte-identical.  The multi-GPU refusal
of FLB_CLOUD_SCAN needs flb_comm_init / flb_p2p_attach and is not exercised on one GPU."""
import numpy as np
import pytest

from conftest import bits
from imu_util import product_inputs
from test_vmap_select import SCENARIOS

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
LEAF = 0.2
SOURCES = ["scan", "undistorted"]


def oracle_world(po, f, body, R, p):
    """pointBodyToWorld (double math, float store) of `body` with f's extrinsic, as the oracle's LIO pass exports it."""
    body = np.ascontiguousarray(body, np.float32)
    lio = po.Lio(body[:64].copy(), body)
    return lio.run_pass(po.lio_params(f, 1), np.asarray(R, np.float64), np.asarray(p, np.float64), True)["world"]


def undistort(flb, h, body, seed):
    """flb_imu_undistort of `body` (as the lidar points of one IMU frame, offsets spread over the scan); returns the
    host out_xyz.  Leaves the device state propagated."""
    f = flb.synth.make_imu_frame(seed=seed, n_points=0)
    P, Cc, x = product_inputs(flb, f)
    h.state_upload(x, x.copy())
    off = np.sort(np.random.default_rng(seed).uniform(0.0, 100.0, len(body))).astype(np.float32)
    packed = np.concatenate([np.asarray(body, np.float32).reshape(-1, 3), off[:, None]], 1)
    out, _ = h.imu_undistort(P, Cc, f["v_imu"], f["pcl_beg_time"], f["pcl_end_time"], packed, offset_index=3)
    return out


def source_cloud(flb, h, src, body, seed):
    """Make `src` the current source of h: the scan upload or the undistortion output.  Returns the host cloud."""
    if src == "scan":
        h.scan_upload(body)
        return np.asarray(body, np.float32)
    return undistort(flb, h, body, seed)


def ikfom_params(flb, f):
    """An IKFoM-style extrinsic (the estimated offset_R_L_I / offset_T_L_I, not the configured one)."""
    prm = flb.capi.lio_params(f, 3)
    prm.R_LI[:] = (np.asarray(f["R_LI"]) @ flb.synth.exp_so3(np.array([0.021, -0.013, 0.034]))).ravel()
    prm.t_LI[:] = np.asarray(f["t_LI"]) + np.array([0.07, -0.045, 0.012])
    return prm


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def assert_no_cloud(flb, h, fr, bgr):
    """Every world-cloud consumer refuses with FLB_ERR_STATE."""
    expect_error(flb, ERR_STATE, h.vmap_select_cloud, fr["Rcw"], fr["Pcw"], LEAF)
    expect_error(flb, ERR_STATE, h.vmap_select_cloud, fr["Rcw"], fr["Pcw"], LEAF, blocking=False)
    expect_error(flb, ERR_STATE, h.vmap_grow_cloud, fr["Rcw"], fr["Pcw"], 0)
    expect_error(flb, ERR_STATE, h.colorize_cloud, fr["Rcw"], fr["Pcw"], bgr)
    expect_error(flb, ERR_STATE, h.world_cloud_download)


def bgr_of(img, k):
    rng = np.random.default_rng(10 + k)
    return np.ascontiguousarray(np.stack([img, np.roll(img, 3, 1), 255 - img], -1) ^ rng.integers(0, 8, img.shape + (3,), dtype=np.uint8))


# ------------------------------------------------------------------------------------------------ the cloud itself
@pytest.mark.parametrize("pose", ["lio_update", "lio_update_enqueue", "explicit_ikfom"])
@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("name", ["T0", "C2"])
def test_world_cloud_matches_oracle(flb, po, frames, name, src, pose):
    f = frames(name)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.map_upload(f["map_xyz"])
    h.scan_upload(f["scan_body"])                      # the LIO update's scan
    cloud = source_cloud(flb, h, src, f["scan_body"], 31)
    prm = flb.capi.lio_params(f, 3)
    x = flb.capi.State18.from_frame(f)
    if pose == "lio_update":
        h.lio_update(prm, x, x.copy())
        n = h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED)
        R, p = x.R, x.p
    elif pose == "lio_update_enqueue":
        h.state_upload(x, x.copy())
        h.lio_update_enqueue(prm)
        n = h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED)   # no synchronise between
        x, _, _ = h.state_download()
        R, p = x.R, x.p
    else:
        prm = ikfom_params(flb, f)
        R, p = f["R_true"], f["p_true"]
        n = h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED, R, p)
    ref = oracle_world(po, dict(f, R_LI=np.array(prm.R_LI[:]).reshape(3, 3), t_LI=np.array(prm.t_LI[:])), cloud, R, p)
    got = h.world_cloud_download()
    assert n == len(cloud) == len(got)
    assert got.tobytes() == np.ascontiguousarray(ref, np.float32).tobytes()
    h.close()


# ------------------------------------------------------------------------------------------------ visual-map sequences
def run_pair(flb, po, seq, grid, thr, ncc_en, ncc_thre, src, reclaim, blocking=True):
    """detect() per frame (select -> grow -> VIO update -> add_observations -> colorize) on A from the device cloud and
    on B from the host cloud.  Returns per-handle lists of per-frame outputs and the final dumps."""
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    vprm = flb.capi.vio_params(f, 4)
    L = (seq["cam"]["width"] // grid) * (seq["cam"]["height"] // grid)
    hs = [flb.Handle(device=0) for _ in range(2)]
    scratch = flb.Handle(device=0)
    for h in hs:
        h.camera_set(seq["cam"])
        h.image_upload(seq["frames"][0]["image"])
        h.vmap_reset(seq, grid_size=grid, outlier_threshold=thr, ncc_en=ncc_en, ncc_thre=ncc_thre)
    out = [[], []]
    for k, fr in enumerate(seq["frames"]):
        bgr = bgr_of(fr["image"], k)
        x0 = flb.capi.State18.make(fr["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr["p"] + [0.02, -0.015, 0.01],
                                   cov=seq["cov"])
        clouds = [source_cloud(flb, h, src, fr["scan_body"], 40 + k) for h in hs]
        assert clouds[0].tobytes() == clouds[1].tobytes()
        pg = oracle_world(po, f, clouds[1], fr["R"], fr["p"])
        pg_down = scratch.voxel_grid(pg, LEAF)
        for i, h in enumerate(hs):
            h.image_upload(fr["image"])
            if i == 0:
                assert h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED, fr["R"], fr["p"]) == len(pg)
                h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF, blocking=blocking)
            else:
                h.vmap_select(fr["Rcw"], fr["Pcw"], pg_down, blocking=blocking)
            s = h.vmap_selected()
            s["map_value"] = h.vmap_map_value(L)
            if i == 0:
                h.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], k)
            else:
                h.vmap_grow(fr["Rcw"], fr["Pcw"], pg, k)
            g = h.vmap_counts()["last_added"]
            mv = h.vmap_map_value(L)
            h.state_upload(x0, x0.copy())
            if k > 0:
                h.vio_update_enqueue(vprm)
            h.vmap_add_observations(None, None, k)
            a = h.vmap_counts()["last_added"]
            x, _, vrep = h.state_download()
            errs = h.vio_errors() if k > 0 else np.zeros(0, np.float32)
            rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"], bgr) if i == 0 else h.colorize(fr["Rcw"], fr["Pcw"], bgr, pg)
            if reclaim:
                h.vmap_reclaim()
            out[i].append(dict(sel=s, grow=g, mv=mv, obs=a, x=bytes(x), vrep=bytes(vrep), errs=errs, rgb=rgb, val=val))
        out[0][-1]["world"] = hs[0].world_cloud_download()
        out[1][-1]["world"] = pg
    dumps = [h.vmap_dump() for h in hs]
    for h in hs + [scratch]:
        h.close()
    return out, dumps


def assert_pair_equal(out, dumps):
    for fa, fb in zip(*out):
        sa, sb = fa["sel"], fb["sel"]
        for key in ("index", "point", "search_level", "error", "pos", "patch", "map_value"):
            assert sa[key].tobytes() == sb[key].tobytes(), key
        assert bits(fa["mv"]).tobytes() == bits(fb["mv"]).tobytes()
        assert fa["grow"] == fb["grow"] and fa["obs"] == fb["obs"]
        assert fa["x"] == fb["x"] and fa["vrep"] == fb["vrep"]
        assert fa["errs"].tobytes() == fb["errs"].tobytes()
        assert fa["rgb"].tobytes() == fb["rgb"].tobytes() and (fa["val"] == fb["val"]).all()
        assert fa["world"].tobytes() == np.ascontiguousarray(fb["world"], np.float32).tobytes()
    da, db = dumps
    for key in da:
        assert da[key].tobytes() == db[key].tobytes(), key


@pytest.mark.parametrize("reclaim", [False, True])
@pytest.mark.parametrize("src", SOURCES)
@pytest.mark.parametrize("sc", SCENARIOS, ids=lambda s: f"{s[0]}-g{s[2]}-thr{s[3]}-ncc{s[4]}-step{s[6][0]}")
def test_visual_map_sequence_equals_host_path(flb, po, sc, src, reclaim):
    name, nf, grid, thr, ncc_en, ncc_thre, step, yaw = sc
    seq = flb.synth.make_visual_sequence(name, nf, step=step, yaw_step_deg=yaw)
    out, dumps = run_pair(flb, po, seq, grid, thr, ncc_en, ncc_thre, src, reclaim)
    assert_pair_equal(out, dumps)
    # the sequence really selects, grows, updates and colours
    assert min(len(f["sel"]["index"]) for f in out[0][1:]) > 10
    assert sum(f["grow"] for f in out[0]) > 0 and sum(f["val"].sum() for f in out[0]) > 100
    if step[0] > 1.0:
        assert (np.concatenate([f["sel"]["search_level"] for f in out[0]]) > 0).sum() > 0


@pytest.mark.parametrize("src", SOURCES)
def test_enqueue_only_select_equals_blocking(flb, po, src):
    """flb_vmap_select_cloud without a count, then flb_vio_update_enqueue (the patch count never visits the host)."""
    seq = flb.synth.make_visual_sequence("T0", 3)
    a, da = run_pair(flb, po, seq, 16, 300.0, 0, 0.0, src, False, blocking=False)
    b, db = run_pair(flb, po, seq, 16, 300.0, 0, 0.0, src, False, blocking=True)
    assert_pair_equal(a, da)
    assert_pair_equal((a[0], b[0]), (da[0], db[0]))


# ------------------------------------------------------------------------------------------------ isolation
def visual_handle(flb, seq):
    h = flb.Handle(device=0)
    h.camera_set(seq["cam"])
    h.image_upload(seq["frames"][0]["image"])
    h.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
    return h


def test_map_add_scan_after_select_cloud(flb, po):
    """flb_vmap_select_cloud filters in buffers of its own: the scan slot survives, flb_map_add_scan still works."""
    seq = flb.synth.make_visual_sequence("T0", 2)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    fr0, fr = seq["frames"]
    a = visual_handle(flb, seq)
    b = flb.Handle(device=0)
    for h in (a, b):
        h.map_upload(fr0["pg"])
    a.scan_upload(fr["scan_body"])
    a.world_cloud(prm, flb.capi.CLOUD_SCAN, fr["R"], fr["p"])
    a.image_upload(fr["image"])
    a.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF)
    a.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], 1)
    a.map_add_scan(prm, 0.5, fr["R"], fr["p"])
    b.map_add_points(oracle_world(po, f, fr["scan_body"], fr["R"], fr["p"]), 0.5)
    ma, mb = a.map_download(), b.map_download()
    assert len(ma) > len(fr0["pg"]) // 2 and ma.tobytes() == mb.tobytes()
    assert a.map_grid_info() == b.map_grid_info()
    a.close()
    b.close()


@pytest.mark.parametrize("between", ["scan_upload", "imu_undistort_0"])
@pytest.mark.parametrize("src", SOURCES)
def test_cloud_is_a_copy(flb, po, src, between):
    """A scan upload, or an undistortion of 0 points, between flb_world_cloud and its consumers changes nothing."""
    seq = flb.synth.make_visual_sequence("T0", 2)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    fr0, fr = seq["frames"]
    res = []
    for disturb in (False, True):
        h = visual_handle(flb, seq)
        h.vmap_grow(fr0["Rcw"], fr0["Pcw"], fr0["pg"], 0)
        source_cloud(flb, h, src, fr["scan_body"], 50)
        h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED, fr["R"], fr["p"])
        w = h.world_cloud_download()
        if disturb:
            if between == "scan_upload":
                h.scan_upload(fr0["scan_body"][:1000])
            else:
                undistort(flb, h, np.zeros((0, 3), np.float32), 51)
        h.image_upload(fr["image"])
        n = h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF)
        s = h.vmap_selected()
        h.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], 1)
        rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"], bgr_of(fr["image"], 1))
        res.append((w.tobytes(), h.world_cloud_download().tobytes(), n, s["index"].tobytes(), s["patch"].tobytes(), rgb.tobytes(),
                    val.tobytes(), h.vmap_dump()["pos"].tobytes()))
        h.close()
    assert res[0][0] == res[0][1] == res[1][0] == res[1][1]
    assert res[0][2] > 10 and res[0] == res[1]


# ------------------------------------------------------------------------------------------------ errors
def test_errors(flb, po):
    seq = flb.synth.make_visual_sequence("T0", 2)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    fr0, fr = seq["frames"]
    bgr = bgr_of(fr["image"], 0)
    SCAN, UND = flb.capi.CLOUD_SCAN, flb.capi.CLOUD_UNDISTORTED
    h = visual_handle(flb, seq)
    # no source at all
    expect_error(flb, ERR_STATE, h.world_cloud, prm, SCAN, fr["R"], fr["p"])
    expect_error(flb, ERR_STATE, h.world_cloud, prm, UND, fr["R"], fr["p"])
    assert_no_cloud(flb, h, fr, bgr)
    h.scan_upload(fr["scan_body"])

    def ok():
        assert h.world_cloud(prm, SCAN, fr["R"], fr["p"]) == len(fr["scan_body"])
        assert len(h.world_cloud_download()) == len(fr["scan_body"])

    # no pose and no device state
    ok()
    expect_error(flb, ERR_STATE, h.world_cloud, prm, SCAN)
    assert_no_cloud(flb, h, fr, bgr)
    # a bad source, exactly one of R / p, no parameters
    for bad in (lambda: h.world_cloud(prm, 2, fr["R"], fr["p"]), lambda: h.world_cloud(prm, -1, fr["R"], fr["p"]),
                lambda: h.world_cloud(prm, SCAN, fr["R"], None), lambda: h.world_cloud(prm, SCAN, None, fr["p"]),
                lambda: h.world_cloud(None, SCAN, fr["R"], fr["p"])):
        ok()
        expect_error(flb, ERR_INVALID, bad)
        assert_no_cloud(flb, h, fr, bgr)
    # a transformed point that is not finite (float overflow) or beyond the visual map's 5e5 limit
    for off in ([1e39, 0.0, 0.0], [0.0, -6.0e5, 0.0], [0.0, 0.0, 5.0e5 + 1e3]):
        ok()
        expect_error(flb, ERR_INVALID, h.world_cloud, prm, SCAN, fr["R"], np.asarray(fr["p"]) + np.array(off))
        assert_no_cloud(flb, h, fr, bgr)
    # flb_voxel_grid used the scan slot as scratch
    ok()
    h.voxel_grid(fr["pg"][:100], LEAF)
    expect_error(flb, ERR_STATE, h.world_cloud, prm, SCAN, fr["R"], fr["p"])
    assert_no_cloud(flb, h, fr, bgr)
    # an undistortion that failed after one that succeeded
    undistort(flb, h, fr["scan_body"], 60)
    assert h.world_cloud(prm, UND, fr["R"], fr["p"]) == len(fr["scan_body"])
    fi = flb.synth.make_imu_frame(seed=61, n_points=0)
    P, Cc, _ = product_inputs(flb, fi)
    v = fi["v_imu"].copy()
    v[2, 0] = v[1, 0] - 1.0                                  # IMU time running backwards
    expect_error(flb, ERR_INVALID, h.imu_undistort, P, Cc, v, fi["pcl_beg_time"], fi["pcl_end_time"], np.zeros((4, 4), np.float32))
    expect_error(flb, ERR_STATE, h.world_cloud, prm, UND, fr["R"], fr["p"])
    assert_no_cloud(flb, h, fr, bgr)
    # a leaf too small for the cloud's extent: refused like flb_voxel_grid refuses it; the cloud stays usable
    h.scan_upload(fr["scan_body"])
    ok()
    scratch = flb.Handle(device=0)
    expect_error(flb, ERR_INVALID, scratch.voxel_grid, oracle_world(po, f, fr["scan_body"], fr["R"], fr["p"]), 1e-4)
    expect_error(flb, ERR_INVALID, h.vmap_select_cloud, fr["Rcw"], fr["Pcw"], 1e-4)
    expect_error(flb, ERR_INVALID, h.vmap_select_cloud, fr["Rcw"], fr["Pcw"], 0.0)
    assert h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF) >= 0
    scratch.close()
    h.close()


@pytest.mark.parametrize("src", SOURCES)
def test_empty_source_behaves_like_n0(flb, po, src):
    seq = flb.synth.make_visual_sequence("T0", 2)
    f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], cfg=seq["cfg"])
    prm = flb.capi.lio_params(f, 3)
    fr0, fr = seq["frames"]
    hs = [visual_handle(flb, seq) for _ in range(2)]
    L = (seq["cam"]["width"] // 16) * (seq["cam"]["height"] // 16)
    res = []
    for i, h in enumerate(hs):
        h.vmap_grow(fr0["Rcw"], fr0["Pcw"], fr0["pg"], 0)
        h.image_upload(fr["image"])
        if i == 0:
            source_cloud(flb, h, src, np.zeros((0, 3), np.float32), 70)
            assert h.world_cloud(prm, flb.capi.CLOUD_SCAN if src == "scan" else flb.capi.CLOUD_UNDISTORTED, fr["R"], fr["p"]) == 0
            assert len(h.world_cloud_download()) == 0
            n = h.vmap_select_cloud(fr["Rcw"], fr["Pcw"], LEAF)
            h.vmap_grow_cloud(fr["Rcw"], fr["Pcw"], 1)
            rgb, val = h.colorize_cloud(fr["Rcw"], fr["Pcw"], bgr_of(fr["image"], 1))
        else:
            n = h.vmap_select(fr["Rcw"], fr["Pcw"], np.zeros((0, 3), np.float32))
            h.vmap_grow(fr["Rcw"], fr["Pcw"], np.zeros((0, 3), np.float32), 1)
            rgb, val = h.colorize(fr["Rcw"], fr["Pcw"], bgr_of(fr["image"], 1), np.zeros((0, 3), np.float32))
        s = h.vmap_selected()
        d = h.vmap_dump()
        res.append((n, s["index"].tobytes(), s["patch"].tobytes(), h.vmap_map_value(L).tobytes(), rgb.shape, val.shape,
                    d["pos"].tobytes(), d["obs"].tobytes(), d["ft_geo"].tobytes()))
        h.close()
    assert res[0] == res[1]
