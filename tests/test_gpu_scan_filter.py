"""GPU tier: the LIO scan built on the device from the undistorted cloud (downSizeFilterSurf -> feats_down_body,
src/laserMapping.cpp:1398-1399: flb_scan_from_undistorted), flb_imu_undistort without a host copy of its points
(out_xyz = NULL), and the first frame's map from the scan (ikdtree.Build(feats_down_body), :1411-1419:
flb_map_upload_scan).

Every comparison is against the host chain on a second handle: flb_imu_undistort with out_xyz -> flb_voxel_grid on a
scratch handle -> flb_scan_upload (and flb_map_upload of the same host points).  Everything must be byte-identical.
The multi-GPU refusal (after flb_comm_init / flb_p2p_attach each rank holds a shard of the scan) needs two ranks and
is not exercised on one GPU."""
import numpy as np
import pytest

from imu_util import product_inputs

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
LEAVES = [0.15, 0.5]          # filter_size_surf of config/avia.yaml, mid360.yaml, MARS_LVIG.yaml / of NTU_VIRAL.yaml


def imu_inputs(flb, seed):
    fi = flb.synth.make_imu_frame(seed=seed, n_points=0)
    P, Cc, x = product_inputs(flb, fi)
    return fi, P, Cc, x


def raw_points(body, seed):
    """`body` as the lidar points of one IMU frame: time offsets (ms) spread over the scan, in time order."""
    off = np.sort(np.random.default_rng(seed).uniform(0.0, 100.0, len(body))).astype(np.float32)
    return np.concatenate([np.asarray(body, np.float32).reshape(-1, 3), off[:, None]], 1)


def undistort(flb, h, body, seed, download=True):
    """flb_imu_undistort of `body` on h (state uploaded first); returns (out_xyz or None, poses, carry, state)."""
    fi, P, Cc, x = imu_inputs(flb, seed)
    h.state_upload(x, x.copy())
    out, poses = h.imu_undistort(P, Cc, fi["v_imu"], fi["pcl_beg_time"], fi["pcl_end_time"], raw_points(body, seed), offset_index=3,
                                 download=download)
    xs, _, _ = h.state_download()
    return out, poses, bytes(Cc), bytes(xs)


def host_chain(flb, h, scratch, body, leaf, seed):
    """undistort with out_xyz -> flb_voxel_grid on the scratch handle -> flb_scan_upload.  Returns the scan's points."""
    out, _, _, _ = undistort(flb, h, body, seed)
    down = scratch.voxel_grid(out, leaf)
    h.scan_upload(down)
    return down


def device_chain(flb, h, body, leaf, seed):
    undistort(flb, h, body, seed, download=False)
    return h.scan_from_undistorted(leaf)


def expect_error(flb, code, fn, *a, **k):
    with pytest.raises(flb.capi.FlbError) as e:
        fn(*a, **k)
    assert e.value.code == code, e.value


def lio_outputs(flb, h, f, prm):
    """Everything that reads the scan: a LIO pass export at a fixed pose, the update's posterior and report, the map
    after flb_map_add_scan at the device posterior, and the scan as a world cloud."""
    R, p = f["R_true"], f["p_true"]
    ps = h.lio_pass(prm, R, p, True)
    x = flb.capi.State18.from_frame(f)
    rep = h.lio_update(prm, x, x.copy())
    h.map_add_scan(prm, 0.5)
    n = h.world_cloud(prm, flb.capi.CLOUD_SCAN, R, p)
    return dict(order=h.debug_scan_order().tobytes(), world=ps["world"].tobytes(), nn_idx=ps["nn_idx"].tobytes(),
                pabcd=ps["pabcd"].tobytes(), sel=ps["rowmask"].tobytes(), x=bytes(x), rep=bytes(rep),
                map=h.map_download().tobytes(), wc_n=n, wc=h.world_cloud_download().tobytes())


def handles(flb, f, n=2):
    hs = [flb.Handle(device=0, cell_size=f["cfg"].cell_size) for _ in range(n)]
    for h in hs:
        h.map_upload(f["map_xyz"])
    return hs


# ------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("leaf", LEAVES)
@pytest.mark.parametrize("name", ["T0", "C2", "C3"])
def test_scan_from_undistorted_equals_host_chain(flb, frames, name, leaf, mode):
    """T0 (600 raw points), C2 (24 k; 14 k leaves at 0.15: the one-block ordering in automatic mode) and a C3-sized raw
    cloud (100 k; 41 k leaves at 0.15: the device-wide ordering), under every flb_debug_set_scan_sort mode."""
    f = frames(name)
    prm = flb.capi.lio_params(f, 3)
    a, b = handles(flb, f)
    scratch = flb.Handle(device=0)
    for h in (a, b):
        h.debug_set_scan_sort(mode)
    n = device_chain(flb, a, f["scan_body"], leaf, 7)
    down = host_chain(flb, b, scratch, f["scan_body"], leaf, 7)
    assert n == len(down) == a.N == b.N and n > 5
    if name == "C2" and leaf == 0.15:
        assert n <= 512 * 33
    if name == "C3" and leaf == 0.15:
        assert n > 1024 * 25
    oa, ob = lio_outputs(flb, a, f, prm), lio_outputs(flb, b, f, prm)
    for key in ob:
        assert oa[key] == ob[key], key
    assert oa["wc_n"] == n
    for h in (a, b, scratch):
        h.close()


# ------------------------------------------------------------------------------------------------ sequence
def test_sequence_interleaved_with_host_uploads(flb, frames):
    """Eight frames that alternate the two scan sets, the device filter and flb_scan_upload taking turns on handle A with
    an flb_voxel_grid call between undistortion and filter (it uses the scan slot as scratch, never the filter's
    buffers); the LIO update is enqueued and the map grown at the device posterior.  Every frame equals the host chain."""
    f = frames("C2")
    prm = flb.capi.lio_params(f, 3)
    a, b = handles(flb, f)
    scratch = flb.Handle(device=0)
    bodies = [f["scan_body"], frames("T1")["scan_body"], f["scan_body"][::3]]
    x0 = flb.capi.State18.from_frame(f)
    for k in range(8):
        body = np.asarray(bodies[k % 3], np.float32) @ flb.synth.exp_so3(np.array([0.0, 0.0, 0.01 * k])).T.astype(np.float32)
        leaf = LEAVES[k % 2]
        res = []
        for i, h in enumerate((a, b)):
            if i == 0 and k % 4 != 3:
                undistort(flb, h, body, 20 + k, download=False)
                h.voxel_grid(bodies[(k + 1) % 3][:5000], 0.3)
                n = h.scan_from_undistorted(leaf)
            else:                                            # B, and every fourth frame of A: the host chain
                n = len(host_chain(flb, h, scratch, body, leaf, 20 + k))
            h.state_upload(x0, x0.copy())
            h.lio_update_enqueue(prm)
            h.map_add_scan(prm, 0.5)
            x, rep, _ = h.state_download()
            res.append((n, h.debug_scan_order().tobytes(), bytes(x), bytes(rep), h.map_download().tobytes()))
        assert res[0] == res[1], k
        assert res[0][0] > 5
    for h in (a, b, scratch):
        h.close()


# ------------------------------------------------------------------------------------------------ out_xyz = NULL
@pytest.mark.parametrize("n_points", [0, 600, 24000])
def test_undistort_without_download(flb, frames, n_points):
    f = frames("C2")
    body = f["scan_body"][:n_points]
    prm = flb.capi.lio_params(f, 3)
    res = []
    for download in (True, False):
        h = flb.Handle(device=0)
        out, poses, carry, xs = undistort(flb, h, body, 30, download=download)
        assert (out is None) != download
        n = h.world_cloud(prm, flb.capi.CLOUD_UNDISTORTED, f["R_true"], f["p_true"])
        res.append((poses.tobytes(), carry, xs, n, h.world_cloud_download().tobytes()))
        h.close()
    assert res[0] == res[1]
    assert res[0][3] == n_points and len(res[0][0]) > 0


# ------------------------------------------------------------------------------------------------ flb_map_upload_scan
@pytest.mark.parametrize("source", ["device", "host"])
@pytest.mark.parametrize("name,leaf", [("T0", 0.15), ("C2", 0.5)])
def test_map_upload_scan_equals_map_upload(flb, frames, name, leaf, source):
    f = frames(name)
    c2 = frames("C2")
    prm = flb.capi.lio_params(f, 3)
    a, b = [flb.Handle(device=0, cell_size=f["cfg"].cell_size) for _ in range(2)]
    scratch = flb.Handle(device=0)
    if source == "device":
        device_chain(flb, a, f["scan_body"], leaf, 9)
    else:
        a.scan_upload(scratch.voxel_grid(undistort(flb, scratch, f["scan_body"], 9)[0], leaf))
    down = host_chain(flb, b, scratch, f["scan_body"], leaf, 9)
    a.map_upload_scan()
    b.map_upload(down)
    assert a.M == b.M == len(down)
    assert a.map_download().tobytes() == b.map_download().tobytes() == down.tobytes()
    assert a.map_grid_info() == b.map_grid_info()
    q = np.ascontiguousarray(np.concatenate([c2["scan_body"][::7], down + 0.05]), np.float32)
    ia, da = a.knn(q)
    ib, db = b.knn(q)
    assert ia.tobytes() == ib.tobytes() and da.tobytes() == db.tobytes()
    assert (ia[:, 0] >= 0).sum() > 100
    # the first frame's update against the map built from its own scan (body frame, identity pose)
    x = [flb.capi.State18.make(np.eye(3), np.zeros(3), cov=f["cov"]) for _ in range(2)]
    reps = [h.lio_update(prm, xi, xi.copy()) for h, xi in zip((a, b), x)]
    assert bytes(x[0]) == bytes(x[1]) and bytes(reps[0]) == bytes(reps[1])
    for h in (a, b, scratch):
        h.close()


# ------------------------------------------------------------------------------------------------ errors
def test_errors_leave_the_previous_scan(flb, frames):
    f = frames("T0")
    prm = flb.capi.lio_params(f, 3)
    h, twin = handles(flb, f)
    scratch = flb.Handle(device=0)
    # no undistortion output at all; no scan for flb_map_upload_scan
    expect_error(flb, ERR_STATE, h.scan_from_undistorted, 0.5)
    expect_error(flb, ERR_STATE, h.map_upload_scan)
    for hh in (h, twin):
        hh.scan_upload(f["scan_body"])

    def assert_current():
        """The scan uploaded first is still current: a LIO update on it equals the twin's, which saw none of the failed
        calls, and so does the scan order."""
        out = []
        for hh in (h, twin):
            x = flb.capi.State18.from_frame(f)
            rep = hh.lio_update(prm, x, x.copy())
            out.append((hh.debug_scan_order().tobytes(), bytes(x), bytes(rep)))
        assert out[0] == out[1]
        assert len(out[0][0]) == 4 * len(f["scan_body"])

    assert_current()
    # a bad leaf
    undistort(flb, h, f["scan_body"], 40, download=False)
    for leaf in (0.0, -0.5, float("nan")):
        expect_error(flb, ERR_INVALID, h.scan_from_undistorted, leaf)
        assert_current()
    # a non-finite point: the host chain fails in flb_voxel_grid
    for bad in (np.nan, np.inf, -np.inf):
        body = np.array(f["scan_body"], np.float32)
        body[len(body) // 2, 1] = bad
        out, _, _, _ = undistort(flb, scratch, body, 41)
        expect_error(flb, ERR_INVALID, scratch.voxel_grid, out, 0.5)
        undistort(flb, h, body, 41, download=False)
        expect_error(flb, ERR_INVALID, h.scan_from_undistorted, 0.5)
        assert_current()
    # PCL's index-overflow case: a leaf too small for the cloud's extent
    body = np.array(f["scan_body"], np.float32)
    body[0] = [-3.0e4, -3.0e4, -3.0e4]
    body[1] = [3.0e4, 3.0e4, 3.0e4]
    out, _, _, _ = undistort(flb, scratch, body, 42)
    expect_error(flb, ERR_INVALID, scratch.voxel_grid, out, 0.01)
    undistort(flb, h, body, 42, download=False)
    expect_error(flb, ERR_INVALID, h.scan_from_undistorted, 0.01)
    assert_current()
    # a failed undistortion after a successful one
    undistort(flb, h, f["scan_body"], 43, download=False)
    fi, P, Cc, x = imu_inputs(flb, 44)
    v = fi["v_imu"].copy()
    v[2, 0] = v[1, 0] - 1.0                                  # IMU time running backwards
    expect_error(flb, ERR_INVALID, h.imu_undistort, P, Cc, v, fi["pcl_beg_time"], fi["pcl_end_time"], raw_points(f["scan_body"], 44),
                 download=False)
    expect_error(flb, ERR_STATE, h.scan_from_undistorted, 0.5)
    assert_current()
    # flb_voxel_grid used the scan slot as scratch: no scan for flb_map_upload_scan
    h.voxel_grid(f["scan_body"], 0.5)
    expect_error(flb, ERR_STATE, h.map_upload_scan)
    # zero points: an empty scan, as flb_scan_upload of nothing; flb_map_upload_scan refuses it
    undistort(flb, h, np.zeros((0, 3), np.float32), 45, download=False)
    assert h.scan_from_undistorted(0.5) == 0 and h.N == 0
    assert len(h.debug_scan_order()) == 0
    assert h.world_cloud(prm, flb.capi.CLOUD_SCAN, f["R_true"], f["p_true"]) == 0
    expect_error(flb, ERR_INVALID, h.map_upload_scan)
    # and the handle goes on: the next frame's scan equals the host chain's
    n = device_chain(flb, h, f["scan_body"], 0.15, 46)
    down = host_chain(flb, twin, scratch, f["scan_body"], 0.15, 46)
    assert n == len(down) and h.debug_scan_order().tobytes() == twin.debug_scan_order().tobytes()
    for hh in (h, twin, scratch):
        hh.close()
