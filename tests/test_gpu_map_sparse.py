"""GPU tier: the sparse cell index of the device map.  On the dense grid's cell geometry it must give bit-identical
results to the dense table in every kNN consumer and in map maintenance; on a map of km extent (where the dense table
enlarges its cell) it keeps the configured cell and stays exact."""
import numpy as np
import pytest

from conftest import bits
from golden_util import ADD_POINTS_CASES, DELETE_BOXES, assert_digest, load_ref_golden, rows, world_scan
from test_map_sparse_index import large_extent_map

pytestmark = pytest.mark.gpu

DENSE, SPARSE = 1, 2


def _handle(flb, f, mode, **kw):
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size, **kw)
    h.debug_set_map_index(mode)
    return h


def _lio(flb, h, f, early=False):
    x = flb.capi.State18.from_frame(f)
    rep = h.lio_update(flb.capi.lio_params(f, 3, early_stop=early), x, x.copy())
    return x, rep


@pytest.mark.parametrize("name", ["T0", "T1", "C2"])
def test_forced_sparse_equals_dense(flb, frames, name):
    f = frames(name)
    rng = np.random.default_rng(4)
    m = f["map_xyz"]
    q = np.concatenate([m[rng.integers(0, len(m), 4000)] + rng.normal(0, 0.3, (4000, 3)),
                        rng.uniform(m.min(0) - 5, m.max(0) + 5, (1000, 3))]).astype(np.float32)
    out = {}
    for mode in (DENSE, SPARSE):
        for persistent in (1, 0):
            h = _handle(flb, f, mode, persistent=persistent)
            h.load_frame(f)
            assert h.map_grid_info()["sparse"] == (mode == SPARSE)
            assert h.map_grid_info()["cell_size"] == np.float32(f["cfg"].cell_size)
            x, rep = _lio(flb, h, f)
            res = [x.vector(), np.array(x.cov[:]), (rep.passes, rep.knn_passes, rep.n_eff_last, rep.rows_total, rep.converged_last)]
            if persistent:
                res += list(h.knn(q)) + [h.map_download()]
            out[mode, persistent] = res
            h.close()
    for persistent in (1, 0):
        d, s = out[DENSE, persistent], out[SPARSE, persistent]
        assert (bits(s[0]) == bits(d[0])).all() and (bits(s[1]) == bits(d[1])).all() and s[2] == d[2]
    d, s = out[DENSE, 1], out[SPARSE, 1]
    assert (s[3] == d[3]).all() and (bits(s[4]) == bits(d[4])).all()
    assert s[5].tobytes() == d[5].tobytes()


def test_forced_sparse_ikfom_and_batch_equal_dense(flb, po, frames):
    import ctypes as C
    f = frames("C2")
    res = {}
    for mode in (DENSE, SPARSE):
        h = _handle(flb, f, mode)
        h.map_upload(f["map_xyz"])
        h.scan_upload(f["scan_body"])
        xg = flb.capi.StateIkfom()
        C.memmove(C.byref(xg), C.byref(po.state_ikfom_from_frame(f)), C.sizeof(xg))
        prm = flb.capi.IkfomParams()
        prm.laser_point_cov = f["cfg"].laser_point_cov
        prm.max_iteration = 4
        prm.limit[:] = [0.001] * 23
        rep = h.lio_update_ikfom(prm, xg)
        res[mode, "ikfom"] = (xg.vector(), np.array(xg.cov), (rep.passes, rep.knn_passes, rep.n_eff_last, rep.rows_total))
        h.close()
        # a C2 x 4 batch (kernel-per-pass batched frames)
        from test_gpu_batch import _frames
        fr = _frames(flb, f, 4)
        hb = _handle(flb, f, mode)
        hb.load_frame(f)
        hb.batch_begin(4, max(len(s) for s, _ in fr))
        for b, (scan, x) in enumerate(fr):
            hb.batch_set_frame(b, scan, x, x.copy())
        hb.batch_update_enqueue(flb.capi.lio_params(f, 3, early_stop=False), flb.capi.vio_params(f, 3, early_stop=False))
        res[mode, "batch"] = [(xb.vector(), np.array(xb.cov[:])) for xb, _, _ in (hb.batch_state_download(b) for b in range(4))]
        hb.close()
    d, s = res[DENSE, "ikfom"], res[SPARSE, "ikfom"]
    assert (bits(s[0]) == bits(d[0])).all() and (bits(s[1]) == bits(d[1])).all() and s[2] == d[2]
    for (xs, cs), (xd, cd) in zip(res[SPARSE, "batch"], res[DENSE, "batch"]):
        assert (bits(xs) == bits(xd)).all() and (bits(cs) == bits(cd)).all()


@pytest.mark.parametrize("k", range(len(ADD_POINTS_CASES)), ids=[f"{n}-{ds}" for n, ds in ADD_POINTS_CASES])
def test_forced_sparse_map_maintenance(flb, k):
    """The batches of test_gpu_map_maintenance on a sparse-index map: the reference ikd-Tree's rows after every batch,
    and the dense handle's exact array (same order, so nn indices keep their meaning)."""
    name, ds = ADD_POINTS_CASES[k]
    g = load_ref_golden()
    f = flb.synth.make_frame(name)
    hs, hd = _handle(flb, f, SPARSE), _handle(flb, f, DENSE)
    for h in (hs, hd):
        h.map_upload(f["map_xyz"])
    rng = np.random.default_rng(3)
    new = world_scan(f)
    batches = [new, new + rng.normal(0, 0.02, new.shape).astype(np.float32),
               rng.uniform(f["map_xyz"].min(0), f["map_xyz"].max(0), (len(new) // 4, 3)).astype(np.float32)]
    for j, b in enumerate(batches):
        hs.map_add_points(b, ds)
        hd.map_add_points(b, ds)
        got = hs.map_download()
        assert len(got) == int(g[f"add{k}_n{j}"])
        assert_digest(g, f"add{k}_rows{j}", rows(got))
        assert got.tobytes() == hd.map_download().tobytes()
        assert hs.map_grid_info()["sparse"] == 1
    q = (new[rng.integers(0, len(new), 2000)] + rng.normal(0, 0.1, (2000, 3))).astype(np.float32)
    (si, sd), (di, dd) = hs.knn(q), hd.knn(q)
    assert (si == di).all() and (bits(sd) == bits(dd)).all()
    hs.close()
    hd.close()


def test_forced_sparse_delete_boxes(flb):
    g = load_ref_golden()
    f = flb.synth.make_frame("T1")
    h = _handle(flb, f, SPARSE)
    h.map_upload(f["map_xyz"])
    h.map_delete_boxes(DELETE_BOXES(f))
    got = h.map_download()
    assert len(got) == int(g["del_left"])
    assert_digest(g, "del_rows", rows(got))
    assert h.map_grid_info()["sparse"] == 1
    h.close()


def _far_frame(flb, f, off):
    """The frame's map replaced by the large-extent map, its pose moved by `off` (into a far copy of the room)."""
    m, offs = large_extent_map(f["map_xyz"])
    g = dict(f)
    g["map_xyz"] = m
    g["p_prop"] = f["p_prop"] + offs[off]
    return g


def test_large_extent_sparse_vs_coarsened_dense(flb, frames):
    f = frames("C2")
    g = _far_frame(flb, f, 3)
    ha = _handle(flb, f, SPARSE)
    hd = flb.Handle(device=0, cell_size=f["cfg"].cell_size)       # automatic: the dense table, cell enlarged
    for h in (ha, hd):
        h.map_upload(g["map_xyz"])
        h.scan_upload(g["scan_body"])
    ia, id_ = ha.map_grid_info(), hd.map_grid_info()
    assert ia["sparse"] == 1 and ia["cell_size"] == np.float32(0.6)
    assert id_["sparse"] == 0 and id_["cell_size"] > 0.6 and id_["cells"] <= 2 ** 25
    rng = np.random.default_rng(8)
    m = g["map_xyz"]
    q = (m[rng.integers(0, len(m), 5000)] + rng.normal(0, 0.3, (5000, 3))).astype(np.float32)
    (ai, ad), (di, dd) = ha.knn(q), hd.knn(q)
    assert (bits(ad) == bits(dd)).all()
    ok = ai >= 0
    assert (ok == (di >= 0)).all()
    ma, md = ha.map_download(), hd.map_download()
    assert (ma[ai[ok]] == md[di[ok]]).all()
    xa, ra = _lio(flb, ha, g)
    xd, rd = _lio(flb, hd, g)
    assert ra.n_eff_last > 1000
    assert (bits(xa.vector()) == bits(xd.vector())).all()
    ha.close()
    hd.close()


def test_large_extent_add_points_trajectory(flb, frames):
    """Frames moving between far rooms: the sparse map stays incremental, the dense one leaves its box and rebuilds;
    both must hold the same point set, before and after the far rooms are deleted."""
    f = frames("T1")
    m, offs = large_extent_map(f["map_xyz"])
    ha = _handle(flb, f, SPARSE)
    hd = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    for h in (ha, hd):
        h.map_upload(m[: len(f["map_xyz"]) * 3])     # three rooms: the last two are added along the trajectory
    assert ha.map_grid_info()["sparse"] == 1
    scan = world_scan(f)
    rng = np.random.default_rng(2)
    for step in range(8):
        o = offs[[0, 3, 4, 1, 4, 2, 3, 0][step]]
        b = (scan + o + rng.normal(0, 0.05, scan.shape)).astype(np.float32)
        if step == 2:
            b = np.concatenate([b, f["map_xyz"] + offs[4]]).astype(np.float32)
        ha.map_add_points(b, 0.3)
        hd.map_add_points(b, 0.3)
        assert ha.map_grid_info()["sparse"] == 1
        assert (rows(ha.map_download()) == rows(hd.map_download())).all()
    assert hd.map_grid_info()["cell_size"] > 0.6
    # delete everything outside the first room: the dense rebuild goes back to the configured cell
    lo, hi = f["map_xyz"].min(0) - 50, f["map_xyz"].max(0) + 50
    far = np.array([[-1e5, -1e5, -1e5, lo[0], 1e5, 1e5], [hi[0], -1e5, -1e5, 1e5, 1e5, 1e5],
                    [lo[0], -1e5, -1e5, hi[0], lo[1], 1e5], [lo[0], hi[1], -1e5, hi[0], 1e5, 1e5]], np.float32)
    ha.map_delete_boxes(far)
    hd.map_delete_boxes(far)
    assert ha.map_grid_info()["sparse"] == 1
    assert hd.map_grid_info()["cell_size"] == np.float32(0.6)
    assert (rows(ha.map_download()) == rows(hd.map_download())).all()
    ha.close()
    hd.close()


def test_sparse_rejects_points_beyond_key_range(flb, frames):
    f = frames("T0")
    h = _handle(flb, f, SPARSE)
    h.map_upload(f["map_xyz"])
    before = h.map_download()
    bad = np.array([[0.0, 0.0, 0.0], [7.0e5, 0.0, 0.0]], np.float32)       # 2^20 cells of 0.6 m = 629 km
    with pytest.raises(flb.FlbError) as e:
        h.map_add_points(bad, 1.0)
    assert e.value.code == -1
    assert h.map_download().tobytes() == before.tobytes()
    h.map_add_points(bad[:1], 1.0)                                          # the handle is still usable
    assert h.map_grid_info()["sparse"] == 1
    with pytest.raises(flb.FlbError):
        h.debug_set_map_index(3)
    h.close()
