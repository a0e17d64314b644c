"""Generate tests/golden/ikdtree_ref.npz: what the reference's own ikd-Tree (oracle/_ref, ikd_Tree.cpp) and the CPU path
built on it return on the seeded synthetic inputs of the tests that compare against it.  Those tests then run anywhere,
without the reference tree.  Needs oracle/_ref/libikdtree_ref.so, which build() compiles whenever the reference tree
is available (oracle/pyoracle.py: reference_dir); from the repo root:

    python __graft_entry__.py
    python tests/golden/make_golden_ref.py

Large outputs are kept as SHA-256 digests of their exact bytes (tests/golden_util.digest): the tests assert bit
equality, which a digest decides as well as the full array.  Each case runs in a child process of its own: the
reference's KD_TREE starts a background thread per tree that is never joined, and processes holding several have crashed.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fastlivo_loader  # noqa: E402
from golden_util import digest, rows, ADD_POINTS_CASES, DELETE_BOXES, lattice_fixture, world_scan  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "ikdtree_ref.npz")


def case_brute(flb, po, name):
    # tests/test_oracle_properties.py::test_brute_knn_equals_reference_ikdtree
    f = flb.synth.make_frame(name)
    rng = np.random.default_rng(1)
    q = (f["map_xyz"][rng.integers(0, len(f["map_xyz"]), 3000)] + rng.normal(0, 0.25, (3000, 3))).astype(np.float32)
    ri, rd = po.IkdTreeRef(f["map_xyz"]).knn(q, nthreads=4)
    return {f"brute_{name}_digest": digest(ri, rd)}


def case_knn_T1(flb, po):
    # tests/test_gpu_parity.py::test_knn_vs_reference_ikdtree
    f = flb.synth.make_frame("T1")
    rng = np.random.default_rng(17)
    q = (f["map_xyz"][rng.integers(0, len(f["map_xyz"]), 5000)] + rng.normal(0, 0.3, (5000, 3))).astype(np.float32)
    ri, rd = po.IkdTreeRef(f["map_xyz"]).knn(q)
    ok = rd[:, 4] <= 5.0
    return {"knn_T1_ok": np.packbits(ok), "knn_T1_digest": digest(ri[ok], rd[ok])}


def case_ties(flb, po):
    # tests/test_gpu_parity.py::test_knn_exact_ties_vs_reference_ikdtree
    lat, q = lattice_fixture()
    ri, rd = po.IkdTreeRef(lat).knn(q)
    return {"ties_idx": ri, "ties_d2": rd}


def case_add_points(flb, po, k):
    # tests/test_gpu_map_maintenance.py::test_add_points_matches_reference_ikdtree
    name, ds = ADD_POINTS_CASES[k]
    f = flb.synth.make_frame(name)
    tree = po.IkdTreeRef(f["map_xyz"])
    rng = np.random.default_rng(3)
    new = world_scan(f)
    batches = [new, new + rng.normal(0, 0.02, new.shape).astype(np.float32),
               rng.uniform(f["map_xyz"].min(0), f["map_xyz"].max(0), (len(new) // 4, 3)).astype(np.float32)]
    out = {}
    for j, b in enumerate(batches):
        tree.add_points(b, ds)
        ref = tree.points()
        out[f"add{k}_n{j}"] = np.int64(len(ref))
        out[f"add{k}_rows{j}"] = digest(rows(ref))
    q = (new[rng.integers(0, len(new), 2000)] + rng.normal(0, 0.1, (2000, 3))).astype(np.float32)
    _, rd = tree.knn(q, nthreads=8)
    ok = rd[:, 4] <= 5.0
    out[f"add{k}_ok"] = np.packbits(ok)
    out[f"add{k}_d2"] = digest(rd[ok])
    return out


def case_delete_boxes(flb, po):
    # tests/test_gpu_map_maintenance.py::test_delete_boxes_matches_reference_ikdtree
    f = flb.synth.make_frame("T1")
    tree = po.IkdTreeRef(f["map_xyz"])
    n = tree.delete_boxes(DELETE_BOXES(f))
    ref = tree.points()
    return {"del_n": np.int64(n), "del_left": np.int64(len(ref)), "del_rows": digest(rows(ref))}


def case_full_frame(flb, po, name):
    # tests/test_gpu_full_size.py::test_full_size_frame_matches_cpu_path: the CPU path (oracle + the reference's tree)
    f = flb.synth.make_frame(name)
    cfg = f["cfg"]
    lio = po.Lio(f["map_xyz"], f["scan_body"], po.IkdTreeRef(f["map_xyz"]))
    x = po.state_from_frame(f)
    lrep = lio.update(po.lio_params(f, cfg.lio_passes - 1, nthreads=8, early_stop=False), x, x.copy())
    out = {f"full_{name}_lio": np.array([lrep.passes, lrep.knn_passes, lrep.n_eff_last, lrep.rows_total], np.int64)}
    if cfg.n_patch:
        vio = po.Vio(f["image"], f["patch_pos"], f["patch_ref"], f["patch_level"], f["cam"])
        vrep = vio.update(po.vio_params(f, cfg.vio_passes, early_stop=False, force_all_passes=True), x, x.copy())
        out[f"full_{name}_vio"] = np.array([*vrep.passes, vrep.rows_total], np.int64)
        out[f"full_{name}_vio_err"] = np.array(list(vrep.last_error), np.float32)
    out[f"full_{name}_x"] = x.vector()
    out[f"full_{name}_P"] = x.P
    return out


def case_full_knn(flb, po):
    # tests/test_gpu_full_size.py::test_full_size_knn_and_pass_properties: the reference's kNN of the C2 scan's world
    # points at the prior pose (the product's world points are asserted bit-exact against the oracle's elsewhere)
    f = flb.synth.make_frame("C2")
    tree = po.IkdTreeRef(f["map_xyz"])
    o = po.Lio(f["map_xyz"], f["scan_body"], tree).run_pass(po.lio_params(f, 2), f["R_prop"], f["p_prop"], True)
    ri, rd = tree.knn(o["world"], nthreads=8)
    ok = rd[:, 4] <= 5.0
    return {"fullknn_world": digest(o["world"]), "fullknn_ok": np.packbits(ok), "fullknn_digest": digest(ri[ok], rd[ok])}


def case_ikfom_C2(flb, po):
    # tests/test_ikfom.py::test_gpu_ikfom_update_parity[C2-3-0.001]
    f = flb.synth.make_frame("C2")
    lio = po.Lio(f["map_xyz"], f["scan_body"], po.IkdTreeRef(f["map_xyz"]))
    x = po.state_ikfom_from_frame(f)
    rep = lio.update_ikfom(po.ikfom_params(f, 3, limit=0.001), x)
    return {"ikfom_C2_rep": np.array([rep.passes, rep.knn_passes, rep.n_eff_last, rep.rows_total, rep.converged_last], np.int64),
            "ikfom_C2_x": x.vector(), "ikfom_C2_cov": x.cov}


CASES = {"brute_T0": (case_brute, "T0"), "brute_T1": (case_brute, "T1"), "knn_T1": (case_knn_T1,), "ties": (case_ties,),
         **{f"add{k}": (case_add_points, k) for k in range(len(ADD_POINTS_CASES))}, "delete_boxes": (case_delete_boxes,),
         **{f"full_{n}": (case_full_frame, n) for n in ("C1", "C2", "C3", "C4")}, "full_knn": (case_full_knn,),
         "ikfom_C2": (case_ikfom_C2,)}


def main():
    if len(sys.argv) == 3:                    # child: one case into one .npz
        flb, po = fastlivo_loader.load(), fastlivo_loader.oracle()
        if po.ref_lib() is None:
            raise SystemExit("oracle/_ref/libikdtree_ref.so is not built")
        fn, *a = CASES[sys.argv[1]]
        np.savez(sys.argv[2], **fn(flb, po, *a))
        sys.stdout.flush()
        os._exit(0)                           # do not run the trees' destructors / thread teardown
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for name in CASES:
            p = os.path.join(d, name + ".npz")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), name, p])
            out.update(dict(np.load(p)))
            print("case", name)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
