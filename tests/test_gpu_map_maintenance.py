"""GPU tier, SURVEY.md section 8 row f1: device-resident map maintenance against the reference's own ikd-Tree
(results stored by tests/golden/make_golden_ref.py): Add_Points(downsample = true) (ikd_Tree.cpp:382-457) and
Delete_Point_Boxes (:501-521)."""
import numpy as np
import pytest

from conftest import bits
from golden_util import ADD_POINTS_CASES, DELETE_BOXES, assert_digest, load_ref_golden, rows, world_scan

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("k", range(len(ADD_POINTS_CASES)), ids=[f"{n}-{ds}" for n, ds in ADD_POINTS_CASES])
def test_add_points_matches_reference_ikdtree(flb, po, k):
    name, ds = ADD_POINTS_CASES[k]
    g = load_ref_golden()
    f = flb.synth.make_frame(name)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.map_upload(f["map_xyz"])
    rng = np.random.default_rng(3)
    new = world_scan(f)
    # three successive batches (the second re-observes the same surfaces, the third is far-field clutter)
    batches = [new, new + rng.normal(0, 0.02, new.shape).astype(np.float32),
               rng.uniform(f["map_xyz"].min(0), f["map_xyz"].max(0), (len(new) // 4, 3)).astype(np.float32)]
    for j, b in enumerate(batches):
        h.map_add_points(b, ds)
        got = h.map_download()
        assert len(got) == int(g[f"add{k}_n{j}"])
        assert_digest(g, f"add{k}_rows{j}", rows(got))
    # the refreshed device grid answers kNN exactly like the refreshed reference tree
    q = (new[rng.integers(0, len(new), 2000)] + rng.normal(0, 0.1, (2000, 3))).astype(np.float32)
    gi, gd = h.knn(q)
    ok = np.unpackbits(g[f"add{k}_ok"], count=len(q)).astype(bool)
    assert ok.sum() > 1500
    assert_digest(g, f"add{k}_d2", gd[ok])
    m = h.map_download()
    # neighbour identity by coordinates (index spaces differ)
    # reference returns indices of ITS build order only for original points; compare coordinates instead
    got_nb = m[gi[ok]]
    d = (q[ok][:, None, :] - got_nb).astype(np.float32)
    rec = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    assert (bits(rec) == bits(gd[ok])).all()
    assert len(m) == int(g[f"add{k}_n2"])
    h.close()


def test_delete_boxes_matches_reference_ikdtree(flb, po):
    g = load_ref_golden()
    f = flb.synth.make_frame("T1")
    h = flb.Handle(device=0)
    h.map_upload(f["map_xyz"])
    n_ref = int(g["del_n"])
    h.map_delete_boxes(DELETE_BOXES(f))
    got = h.map_download()
    assert n_ref > 100 and len(got) == int(g["del_left"]) == len(f["map_xyz"]) - n_ref
    assert_digest(g, "del_rows", rows(got))
    # LIO still runs on the pruned map and agrees with the oracle on the same point set
    h.scan_upload(f["scan_body"])
    lio = po.Lio(got, f["scan_body"])
    xo = po.state_from_frame(f)
    lio.update(po.lio_params(f, 3), xo, xo.copy())
    xg = flb.capi.State18.from_frame(f)
    h.lio_update(flb.capi.lio_params(f, 3), xg, xg.copy())
    assert np.abs(xg.vector() - xo.vector()).max() / np.abs(xo.vector()).max() < 1e-9
    h.close()


def test_map_maintenance_argument_errors(flb):
    h = flb.Handle(device=0)
    with pytest.raises(flb.FlbError) as e:
        h.map_add_points(np.zeros((3, 3), np.float32), 0.3)
    assert e.value.code == -4
    f = flb.synth.make_frame("T0")
    h.map_upload(f["map_xyz"])
    with pytest.raises(flb.FlbError) as e:
        h.map_add_points(np.full((3, 3), np.inf, np.float32), 0.3)
    assert e.value.code == -1
    with pytest.raises(flb.FlbError) as e:
        h.map_add_points(np.zeros((3, 3), np.float32), 0.0)
    assert e.value.code == -1
    h.close()
