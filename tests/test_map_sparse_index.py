"""CPU tier: the sparse cell index of the device map (flb_device.cuh: cell keys, hash probe, knn5_grid<true>) compiled
for the host (tests/hostemu/sparse_index.cpp).  On the dense grid's cell geometry both indexes must return bit-identical neighbours;
on a map of km extent the sparse index must stay exact against brute force."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import bits
from golden_util import lattice_fixture
from test_hostemu_device_math import grid_build


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def sparse_emu(tmp_path_factory):
    """tests/hostemu/sparse_index.cpp built for the host (into a temporary directory)."""
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "sparse_index.cpp")
    so = str(tmp_path_factory.mktemp("sparse_emu") / "libsparse_index.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    return C.CDLL(so)


def sparse_build(lib, map_xyz, gridf):
    """Points sorted (stably) by 64-bit cell key, as rebuild_sparse orders them."""
    m = np.ascontiguousarray(map_xyz, np.float32)
    keys = np.empty(len(m), np.uint64)
    lib.emu_sparse_keys(_p(gridf), _p(m), len(m), _p(keys))
    order = np.argsort(keys, kind="stable")
    pts4 = np.zeros((len(m), 4), np.float32)
    pts4[:, :3] = m[order]
    pts4[:, 3] = order.astype(np.int32).view(np.float32)
    return np.ascontiguousarray(keys[order]), pts4, order


def knn_dense(hostemu, gridf, gridi, cell_start, pts4, q):
    pos = np.empty((len(q), 5), np.int32)
    d2 = np.empty((len(q), 5), np.float32)
    hostemu.emu_knn(_p(gridf), _p(gridi), _p(cell_start), _p(pts4), _p(q), len(q), _p(pos), _p(d2))
    return pos, d2


def knn_sparse(lib, gridf, max_ring, keys, pts4, q):
    q = np.ascontiguousarray(q, np.float32)
    pos = np.empty((len(q), 5), np.int32)
    d2 = np.empty((len(q), 5), np.float32)
    lib.emu_knn_sparse(_p(gridf), int(max_ring), _p(keys), _p(pts4), len(pts4), _p(q), len(q), _p(pos), _p(d2))
    return pos, d2


def _queries(m, n, seed):
    rng = np.random.default_rng(seed)
    lo, hi = m.min(0), m.max(0)
    near = m[rng.integers(0, len(m), n)] + rng.normal(0, 0.3, (n, 3))
    box = rng.uniform(lo - 6, hi + 6, size=(n // 2, 3))
    far = rng.uniform(-1e4, 1e4, size=(50, 3))
    return np.concatenate([near, box, far]).astype(np.float32)


@pytest.mark.parametrize("name", ["T0", "T1", "C1", "C2"])
def test_sparse_matches_dense_bitwise(hostemu, sparse_emu, frames, name):
    f = frames(name)
    m = f["map_xyz"]
    gridf, gridi, cell_start, pts4_d, order_d = grid_build(m, f["cfg"].cell_size)
    keys, pts4_s, order_s = sparse_build(sparse_emu, m, gridf)
    assert (order_s == order_d).all()              # key order == dense cell-id order, same within-cell order
    q = _queries(m, 3000, 7)
    pd, dd = knn_dense(hostemu, gridf, gridi, cell_start, pts4_d, q)
    ps, ds = knn_sparse(sparse_emu, gridf, gridi[3], keys, pts4_s, q)
    assert (ps == pd).all()
    assert (bits(ds) == bits(dd)).all()


def test_sparse_matches_dense_exact_ties(hostemu, sparse_emu):
    lat, q = lattice_fixture()
    gridf, gridi, cell_start, pts4_d, _ = grid_build(lat, 0.6)
    keys, pts4_s, _ = sparse_build(sparse_emu, lat, gridf)
    pd, dd = knn_dense(hostemu, gridf, gridi, cell_start, pts4_d, q)
    ps, ds = knn_sparse(sparse_emu, gridf, gridi[3], keys, pts4_s, q)
    assert (ps == pd).all() and (bits(ds) == bits(dd)).all()


def large_extent_map(m, spread=1500.0):
    """The room plus translated copies about +-spread metres away (a dense 0.6 m grid over it needs > 2^25 cells)."""
    offs = np.array([[0, 0, 0], [spread, 0, 0], [-spread, spread, 0], [0, -spread, 0], [spread, spread, 0]], np.float32)
    return np.concatenate([m + o for o in offs]).astype(np.float32), offs


def test_sparse_large_extent_exact(sparse_emu, po, frames):
    f = frames("T1")
    m, offs = large_extent_map(f["map_xyz"])
    lo = m.min(0)
    cell = np.float32(0.6)
    gridf = np.array([lo[0], lo[1], lo[2], cell, np.float32(1.0) / cell, 5.0], np.float32)
    dims = np.floor((m.max(0).astype(np.float64) - lo) / 0.6) + 1
    assert np.prod(dims) > 2 ** 25
    keys, pts4, order = sparse_build(sparse_emu, m, gridf)
    rng = np.random.default_rng(9)
    base = _queries(f["map_xyz"], 600, 3)
    q = (base + offs[rng.integers(0, len(offs), len(base))]).astype(np.float32)
    pos, d2 = knn_sparse(sparse_emu, gridf, int(np.ceil(np.sqrt(5.0) / 0.6)) + 1, keys, pts4, q)
    bi, bd = po.knn_brute(m, q)
    ok = bd[:, 4] <= 5.0
    assert ok.any() and (~ok).any()
    assert (bits(d2[ok]) == bits(bd[ok])).all()
    idx = np.where(pos >= 0, order[np.maximum(pos, 0)], -1)
    assert (m[idx[ok]] == m[bi[ok]]).all()
    assert (~(d2[~ok][:, 4] <= 5.0)).all()


def test_sparse_find_every_cell(sparse_emu, frames):
    f = frames("T1")
    m, _ = large_extent_map(f["map_xyz"], 500.0)
    lo = m.min(0)
    gridf = np.array([lo[0], lo[1], lo[2], 0.6, np.float32(1.0) / np.float32(0.6), 5.0], np.float32)
    keys, _, _ = sparse_build(sparse_emu, m, gridf)
    ukeys, first, counts = np.unique(keys, return_index=True, return_counts=True)
    mask21 = np.uint64((1 << 21) - 1)
    cells = np.stack([(ukeys & mask21), (ukeys >> np.uint64(21)) & mask21, ukeys >> np.uint64(42)], 1).astype(np.int64) - (1 << 20)
    cells = np.ascontiguousarray(cells, np.int32)
    se = np.empty((len(cells), 2), np.int32)
    sparse_emu.emu_sparse_find(_p(keys), len(keys), _p(cells), len(cells), _p(se))
    assert (se[:, 0] == first).all() and (se[:, 1] == first + counts).all()
    # absent cells (and cells beyond the key range) are empty runs
    rng = np.random.default_rng(1)
    probe = rng.integers(-3000, 3000, size=(20000, 3)).astype(np.int32)
    probe = np.concatenate([probe, np.array([[1 << 20, 0, 0], [0, -(1 << 20) - 1, 0], [0, 0, 1 << 22]], np.int32)])
    occupied = set(map(tuple, cells.tolist()))
    absent = np.ascontiguousarray([c for c in probe.tolist() if tuple(c) not in occupied], np.int32)
    se = np.empty((len(absent), 2), np.int32)
    sparse_emu.emu_sparse_find(_p(keys), len(keys), _p(absent), len(absent), _p(se))
    assert (se == 0).all()
