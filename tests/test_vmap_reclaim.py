"""CPU tier: the reclaim rules of the device visual map (flb_device.cuh: live test, rank remap, free-slot choice),
compiled for the host (tests/hostemu/vmap_reclaim.cpp) in the order the flb_vmap_reclaim kernels apply them, against a
numpy restatement of the reference's lifetimes: a Feature lives while a Point's observation list holds it, a keyframe
image while a live Feature refers to it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def reclaim_emu(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "vmap_reclaim.cpp")
    so = str(tmp_path_factory.mktemp("reclaim_emu") / "libvmap_reclaim.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emu_vm_reclaim.restype = C.c_int
    L.emu_vm_reclaim.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_vm_next_slots.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return L


def make_map(rng, n_points, n_feats, tail, dead_frac):
    """Observation lists as the device keeps them: every feature belongs to at most one point, newest first; the
    entries past n_obs are stale ids (left behind by evictions) that must be ignored."""
    n_obs = rng.choice([0, 1, 5, 19, 20], size=n_points, p=[0.15, 0.2, 0.25, 0.15, 0.25]).astype(np.int32)
    ids = rng.permutation(n_feats)
    n_named = min(int(n_obs.sum()), int(round(n_feats * (1.0 - dead_frac))))
    obs = rng.integers(0, max(n_feats, 1), size=(n_points, 20)).astype(np.int32)
    k = 0
    for j in range(n_points):
        m = min(int(n_obs[j]), n_named - k)
        n_obs[j] = m
        obs[j, :m] = ids[k:k + m]
        k += m
    feat_img = rng.integers(0, max(tail, 1), size=n_feats).astype(np.int32)
    return n_obs, obs, feat_img


def numpy_reclaim(n_obs, obs, feat_img, tail, pinned):
    n_feats = len(feat_img)
    live = np.zeros(n_feats, bool)
    for j in range(len(n_obs)):
        live[obs[j, :n_obs[j]]] = True
    rank = np.concatenate([[0], np.cumsum(live)]).astype(np.int32)
    new_obs = np.full_like(obs, -1)
    for j in range(len(n_obs)):
        new_obs[j, :n_obs[j]] = rank[obs[j, :n_obs[j]]]
    kept = feat_img[live]
    used = set(kept.tolist()) | {pinned}
    free = sorted((s for s in range(tail) if s not in used), reverse=True)      # lowest free slot on top
    return rank, new_obs, kept, np.array(free, np.int32)


def run_emu(L, n_obs, obs, feat_img, tail, pinned):
    n_feats = len(feat_img)
    obs_io = np.ascontiguousarray(obs, np.int32).copy()
    img_io = np.ascontiguousarray(feat_img, np.int32).copy()
    rank = np.zeros(n_feats + 1, np.int32)
    stack = np.zeros(max(tail, 1), np.int32)
    n_free = np.zeros(1, np.int32)
    n_live = L.emu_vm_reclaim(len(n_obs), _p(np.ascontiguousarray(n_obs, np.int32)), _p(obs_io), n_feats, _p(img_io), tail, pinned,
                              _p(rank), _p(stack), _p(n_free))
    return n_live, rank, obs_io, img_io[:n_live], stack[:n_free[0]]


CASES = [
    # n_points, n_feats, tail, dead fraction, pinned
    (0, 0, 0, 0.0, -1),            # empty map
    (1, 1, 1, 0.0, 0),
    (300, 2000, 60, 0.3, 59),
    (300, 2000, 60, 0.0, -1),      # nothing to reclaim
    (300, 2000, 60, 1.0, 12),      # every feature dead: every slot but the pinned one frees
    (2000, 30000, 700, 0.6, 3),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"pts{c[0]}-ft{c[1]}-slots{c[2]}-dead{c[3]}")
def test_reclaim_rules_match_numpy(reclaim_emu, case):
    n_points, n_feats, tail, dead, pinned = case
    rng = np.random.default_rng(n_points * 7 + n_feats)
    n_obs, obs, feat_img = make_map(rng, n_points, n_feats, tail, dead)
    if tail > 4:
        feat_img[feat_img == 4] = 5            # a frame with no features at all ...
        gone = feat_img == 2                   # ... and one whose features are all dead
        for j in range(n_points):
            keep = ~gone[obs[j, :n_obs[j]]]
            lst = obs[j, :n_obs[j]][keep]
            obs[j, :len(lst)] = lst
            n_obs[j] = len(lst)
    rank_e, obs_e, kept_e, free_e = numpy_reclaim(n_obs, obs, feat_img, tail, pinned)
    n_live, rank, obs_g, kept, free = run_emu(reclaim_emu, n_obs, obs, feat_img, tail, pinned)
    assert n_live == rank_e[-1]
    assert (rank == rank_e).all()
    assert (obs_g == obs_e).all()
    assert (kept == kept_e).all()
    assert (free == free_e).all()
    if tail > 4:
        assert 2 in free.tolist() or pinned == 2
        assert 4 in free.tolist() or pinned == 4
    # a second reclaim of the compacted map changes nothing
    n2, rank2, obs2, kept2, free2 = run_emu(reclaim_emu, n_obs, obs_g, kept, tail, pinned)
    assert n2 == n_live and (rank2 == np.arange(n_live + 1)).all() and (obs2 == obs_g).all() and (kept2 == kept).all()
    assert (free2 == free).all()


def test_next_slot_prefers_free_stack(reclaim_emu):
    rng = np.random.default_rng(3)
    for n_free, tail in ((0, 0), (0, 17), (5, 40), (40, 40)):
        stack = np.ascontiguousarray(np.sort(rng.choice(max(tail, 1), n_free, replace=False))[::-1], np.int32)
        out = np.zeros(n_free + 6, np.int32)
        reclaim_emu.emu_vm_next_slots(n_free, _p(stack), tail, len(out), _p(out))
        expect = list(stack[::-1]) + list(range(tail, tail + 6))
        assert out.tolist() == expect
