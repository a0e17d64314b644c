"""GPU tier: the host point uploads pinned to fixed values.  Every entry point that takes a caller's xyz array with a
stride -- flb_map_upload, flb_map_add_points, flb_scan_upload (from pageable and from flb_host_alloc memory, and through
flb_frame_enqueue and flb_batch_set_frame), flb_voxel_grid, flb_visual_candidates, flb_vmap_select, flb_vmap_grow and
flb_colorize -- runs at strides 3, 4 and 12 and at sizes that put points in every lane of the host fold and in its scalar
tail.  Then the refusals: NaN, +inf and -inf on each axis at the first, a middle and the last point and in the tail, two
bad points (the first one is named), the visual map's +-5e5 limit and one ulp beyond, and a point beyond
flb_map_add_points' bounds together with a non-finite one.  A cloud whose minimum on one axis is reached by both +0.0 and
-0.0 checks that the map, its cell index and the kNN do not depend on which zero the bounds pick.  After every call it
records the return code, the error text, the launch count and a digest of the outputs (the map, its grid info and a kNN
of fixed queries; the scan order and the scan at a fixed pose; the centroids; the candidates; the selected patches; the
colours), so any change to what a call accepts, refuses, reports or leaves behind shows.

EXPECTED was recorded on an NVIDIA H100 80GB HBM3 (700 W power limit, 132 SMs) with the host code that packed and
checked the points in a loop of each entry point's own.  The LIO update behind flb_frame_enqueue sizes its grid from the
SM count, so the values hold for that card: the test checks the device name and SM count first."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

STRIDES = (3, 4, 12)
SIZES = (0, 1, 7, 8, 9, 23, 24, 25, 3000)       # 24 floats (8 points) a fold step: every lane, and the scalar tail
FEW = (1, 9, 25, 3000)
NB = 30                                          # the refusal cloud: points 0-23 in the vector body, 24-29 in the tail
BAD_AT = (("first", 0), ("middle", 11), ("tail", 25), ("last", NB - 1))
BAD_VAL = (("nan", np.nan), ("+inf", np.inf), ("-inf", -np.inf))
LIM = np.float32(5.0e5)
BEYOND = np.nextafter(LIM, np.float32(np.inf))


def digest(*objs):
    """sha256 (16 hex digits) over numpy arrays, ctypes structures and bytes, in order."""
    m = hashlib.sha256()
    for o in objs:
        if isinstance(o, (np.ndarray, np.generic)):
            m.update(np.ascontiguousarray(o).tobytes())
        elif isinstance(o, (bytes, bytearray)):
            m.update(o)
        else:
            m.update(bytes(o))
    return m.hexdigest()[:16]


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.name, p.multi_processor_count


def strided(pts, stride):
    """pts (n, 3) as an (n, stride) float32 array: xyz first, the rest a filler the calls must skip."""
    a = np.full((len(pts), stride), 7.25, np.float32)
    a[:, :3] = pts
    return a


def take(pts, n):
    """n points cycled from pts, each pass shifted by 1 cm so no two are equal."""
    reps = -(-n // len(pts)) if n else 0
    return np.concatenate([pts + np.float32(0.01 * r) for r in range(reps)] or [pts[:0]])[:n].astype(np.float32)


def with_bad(pts, at, axis, v):
    b = pts.copy()
    b[at, axis] = v
    return b


def refusals(pts, axes=(0, 1, 2)):
    """(label, cloud) of NB points with one non-finite coordinate, then two."""
    base = take(pts, NB)
    out = [(f"{vn}-{'xyz'[ax]}-{wn}", with_bad(base, at, ax, v)) for vn, v in BAD_VAL for ax in axes for wn, at in BAD_AT]
    return out + [("two-bad-3-17", with_bad(with_bad(base, 17, 2, -np.inf), 3, 1, np.nan))]


def signed_zero(pts):
    """pts moved so x's minimum is 0, reached by -0.0 and +0.0: (label, cloud) with either zero first in point order,
    and the other in a lower lane of the fold (point 5 is float 15, point 10 float 30 = lane 6)."""
    b = take(pts, 40)
    b[:, 0] -= b[:, 0].min() - np.float32(0.5)
    out = []
    for name, first, second in (("neg-first", -0.0, 0.0), ("pos-first", 0.0, -0.0)):
        c = b.copy()
        c[5, 0], c[10, 0], c[37, 0] = first, second, first
        out.append((f"signed-zero-{name}", c))
    return out


def run_sequence(flb):
    """[(label, rc, error text or None, launches, digest of the call's outputs)] after every call of the sequence."""
    cp = flb.capi
    L = cp.lib()
    f = flb.synth.make_frame("T0")
    cfg = f["cfg"]
    mp, sc = np.ascontiguousarray(f["map_xyz"], np.float32), np.ascontiguousarray(f["scan_body"], np.float32)
    lprm = cp.lio_params(f, cfg.lio_passes - 1)
    R, p = np.ascontiguousarray(f["R_prop"], np.float64), np.ascontiguousarray(f["p_prop"], np.float64)
    x0 = cp.State18.from_frame(f)
    queries = np.ascontiguousarray(mp[::97] + np.float32(0.03))
    out = []

    def state():
        s = cp.State18()
        C.memmove(C.byref(s), C.byref(x0), C.sizeof(s))
        return s

    def step(h, label, call, outs=list):
        """call() -> rc; outs() -> the outputs, read after the call's launch count and error text."""
        l0 = h.launch_count()
        rc = call()
        launches = h.launch_count() - l0
        err = L.flb_last_error(h.h).decode() if rc else None
        out.append((label, rc, err, launches, digest(*outs())))

    def map_state(h):
        n = L.flb_map_size(h.h)
        xyz, m = np.zeros((max(n, 1), 3), np.float32), C.c_int(-7)
        rc0 = L.flb_map_download(h.h, cp._p(xyz), n, C.byref(m))
        cs, sp, nc, nb = C.c_double(), C.c_int(), C.c_int64(), C.c_int64()
        rc1 = L.flb_map_grid_info(h.h, C.byref(cs), C.byref(sp), C.byref(nc), C.byref(nb))
        idx, d2 = np.full((len(queries), 5), -7, np.int32), np.full((len(queries), 5), -7, np.float32)
        rc2 = L.flb_knn(h.h, cp._p(queries), len(queries), cp._p(idx), cp._p(d2))
        return [np.int32([n, m.value, rc0, rc1, rc2, sp.value, nc.value, nb.value]), np.float64(cs.value), xyz, idx, d2]

    def scan_state(h):
        order = np.full(4096, -7, np.int32)
        rc0 = L.flb_debug_scan_order(h.h, cp._p(order), len(order))
        nw = C.c_int(-7)
        rc1 = L.flb_world_cloud(h.h, C.byref(lprm), cp._p(R), cp._p(p), cp.CLOUD_SCAN, C.byref(nw))
        wc, nd = np.full((4096, 3), -7, np.float32), C.c_int(-7)
        rc2 = L.flb_world_cloud_download(h.h, cp._p(wc), len(wc), C.byref(nd)) if rc1 == 0 else -99
        h.map_upload(mp)
        rc3 = L.flb_map_add_scan(h.h, C.byref(lprm), cp._p(R), cp._p(p), C.c_float(0.5))
        return [np.int32([rc0, rc1, rc2, rc3, nw.value, nd.value]), order, wc] + map_state(h)

    # ---- the map: flb_map_upload, flb_map_add_points
    h = flb.Handle(device=0, cell_size=cfg.cell_size)

    def map_upload(a):
        return lambda: L.flb_map_upload(h.h, cp._p(a), len(a), a.shape[1]), lambda: map_state(h)

    def map_add(a, ds=0.5):
        h.map_upload(mp)
        return lambda: L.flb_map_add_points(h.h, cp._p(a), len(a), a.shape[1], C.c_float(ds)), lambda: map_state(h)

    for s in STRIDES:
        for n in SIZES:
            step(h, f"map_upload-s{s}-n{n}", *map_upload(strided(take(mp, n), s)))
    for label, b in signed_zero(mp):
        step(h, f"map_upload-{label}", *map_upload(strided(b, 3)))
    for s in STRIDES:
        for label, b in refusals(mp):
            step(h, f"map_upload-s{s}-{label}", *map_upload(strided(b, s)))
    for s in STRIDES:
        for n in SIZES:
            step(h, f"map_add_points-s{s}-n{n}", *map_add(strided(take(mp, n) + np.float32(0.05), s)))
    for label, b in refusals(mp + np.float32(0.05)):
        step(h, f"map_add_points-{label}", *map_add(strided(b, 4)))
    far = with_bad(take(mp, NB), 5, 0, np.float32(1e6))
    step(h, "map_add_points-far", *map_add(strided(far, 3)))
    step(h, "map_add_points-far-and-nan", *map_add(strided(with_bad(far, 20, 1, np.nan), 3)))
    step(h, "map_add_points-nan-and-far", *map_add(strided(with_bad(far, 2, 1, np.nan), 3)))
    h.close()

    # ---- the scan: flb_scan_upload from pageable and page-locked memory, flb_frame_enqueue, flb_batch_set_frame
    h = flb.Handle(device=0, cell_size=cfg.cell_size)
    h.map_upload(mp)

    def scan_upload(a):
        return lambda: L.flb_scan_upload(h.h, cp._p(a), len(a), a.shape[1]), lambda: scan_state(h)

    for s in STRIDES:
        for n in SIZES:
            step(h, f"scan_upload-s{s}-n{n}", *scan_upload(strided(take(sc, n), s)))
    for s in (3, 12):
        for n in SIZES:
            step(h, f"scan_upload-pinned-s{s}-n{n}", *scan_upload(h.pinned_like(strided(take(sc, n), s))))
    for label, b in signed_zero(sc):
        step(h, f"scan_upload-{label}", *scan_upload(strided(b, 3)))
    for label, b in refusals(sc):
        step(h, f"scan_upload-{label}", *scan_upload(strided(b, 12)))
    for label, b in refusals(sc)[::5]:
        step(h, f"scan_upload-pinned-{label}", *scan_upload(h.pinned_like(strided(b, 3))))

    def frame(a):
        fi = h.frame_inputs(a, state(), state())

        def result():
            xo, lr, vr = cp.State18(), cp.LioReport(), cp.VioReport()
            return [np.int32(L.flb_state_download_wait(h.h, 0, C.byref(xo), C.byref(lr), C.byref(vr))), xo, lr]
        return lambda: L.flb_frame_enqueue(h.h, C.byref(fi), C.byref(lprm), None, 0), result

    h.map_upload(mp)
    for s in STRIDES:
        for n in FEW:
            step(h, f"frame_enqueue-s{s}-n{n}", *frame(strided(take(sc, n), s)))
    for label, b in refusals(sc)[::7]:
        step(h, f"frame_enqueue-{label}", *frame(strided(b, 4)))

    def scan_order():
        order = np.full(4096, -7, np.int32)
        return [np.int32(L.flb_debug_scan_order(h.h, cp._p(order), len(order))), order]

    def batch(a):
        x, xp = state(), state()
        return lambda: L.flb_batch_set_frame(h.h, 0, cp._p(a), len(a), a.shape[1], C.byref(x), C.byref(xp)), scan_order

    h.batch_begin(1, 4096)
    for s in STRIDES:
        for n in FEW:
            step(h, f"batch_set_frame-s{s}-n{n}", *batch(strided(take(sc, n), s)))
    for label, b in refusals(sc)[::7]:
        step(h, f"batch_set_frame-{label}", *batch(strided(b, 4)))
    h.close()

    # ---- flb_voxel_grid, flb_visual_candidates
    h = flb.Handle(device=0, cell_size=cfg.cell_size)

    def voxel(a):
        o, m = np.full((max(len(a), 1), 3), -7, np.float32), C.c_int(-7)
        return (lambda: L.flb_voxel_grid(h.h, cp._p(a), len(a), a.shape[1], C.c_float(0.5), cp._p(o), len(a), C.byref(m)),
                lambda: [np.int32(m.value), o])

    for s in STRIDES:
        for n in SIZES:
            step(h, f"voxel_grid-s{s}-n{n}", *voxel(strided(take(sc, n), s)))
    for label, b in signed_zero(sc):
        step(h, f"voxel_grid-{label}", *voxel(strided(b, 3)))
    for label, b in refusals(sc):
        step(h, f"voxel_grid-{label}", *voxel(strided(b, 4)))

    h.camera_set(f["cam"])
    h.image_upload(f["image"])
    ncell = (f["cam"]["width"] // 40) * (f["cam"]["height"] // 40)

    def candidates(a):
        mv, win = np.linspace(0, 50, ncell).astype(np.float32), np.full(ncell, -7, np.int32)
        return (lambda: L.flb_visual_candidates(h.h, cp._p(R), cp._p(p), cp._p(a), len(a), a.shape[1], 40, 40, cp._p(mv), cp._p(win)),
                lambda: [mv, win])

    for s in STRIDES:
        for n in SIZES:
            step(h, f"visual_candidates-s{s}-n{n}", *candidates(strided(take(mp, n), s)))
    h.close()

    # ---- the visual map: flb_vmap_select, flb_vmap_grow, flb_colorize
    seq = flb.synth.make_visual_sequence("T0", 3)
    fr0 = seq["frames"][0]
    R0, P0 = np.ascontiguousarray(fr0["Rcw"], np.float64), np.ascontiguousarray(fr0["Pcw"], np.float64)
    pg = np.ascontiguousarray(fr0["pg"], np.float32)
    h = flb.Handle(device=0)
    h.camera_set(seq["cam"])
    h.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
    h.image_upload(fr0["image"])
    W, H = seq["cam"]["width"], seq["cam"]["height"]
    bgr = np.random.default_rng(5).integers(0, 256, (H, W, 3), dtype=np.uint8)
    limits = []
    for ax in (0, 1, 2):
        for name, v in (("+lim", LIM), ("-lim", -LIM), ("+beyond", BEYOND), ("-beyond", -BEYOND)):
            limits.append((f"{name}-{'xyz'[ax]}", with_bad(take(pg, NB), 9, ax, v)))
    limits.append(("beyond-then-nan", with_bad(with_bad(take(pg, NB), 4, 2, -BEYOND), 21, 0, np.nan)))
    limits.append(("nan-then-beyond", with_bad(with_bad(take(pg, NB), 4, 2, np.nan), 21, 0, BEYOND)))

    def select(a):
        m = C.c_int(-7)

        def selected():
            sel = h.vmap_selected()
            return [np.int32(m.value)] + [sel[k] for k in sorted(sel)]
        return lambda: L.flb_vmap_select(h.h, cp._p(R0), cp._p(P0), cp._p(a), len(a), a.shape[1], C.byref(m)), selected

    for s in STRIDES:
        for n in SIZES:
            step(h, f"vmap_select-s{s}-n{n}", *select(strided(take(pg, n), s)))
    for label, b in refusals(pg) + limits:
        step(h, f"vmap_select-{label}", *select(strided(b, 4)))

    def grow(a, fid):
        return (lambda: L.flb_vmap_grow(h.h, cp._p(R0), cp._p(P0), cp._p(a), len(a), a.shape[1], fid),)

    fid = 0
    for s in STRIDES:
        for n in FEW:
            step(h, f"vmap_grow-s{s}-n{n}", *grow(strided(take(pg, n), s), fid))
            fid += 1
    for label, b in refusals(pg)[::7] + limits[:4]:
        step(h, f"vmap_grow-{label}", *grow(strided(b, 3), fid))
    step(h, "vmap_grow-after", *select(strided(pg, 3)))

    def colorize(a):
        rgb, val = np.full((len(a), 3), 7, np.uint8), np.full(len(a), 7, np.uint8)
        return (lambda: L.flb_colorize(h.h, cp._p(R0), cp._p(P0), cp._p(bgr), 3 * W, cp._p(a), len(a), a.shape[1], cp._p(rgb), cp._p(val)),
                lambda: [rgb, val])

    for s in STRIDES:
        for n in FEW:
            step(h, f"colorize-s{s}-n{n}", *colorize(strided(take(pg, n), s)))
    for label, b in refusals(pg)[::7] + limits[:4]:
        step(h, f"colorize-{label}", *colorize(strided(b, 12)))
    h.close()
    return out


DEVICE = ('NVIDIA H100 80GB HBM3', 132)         # name and SM count of the card EXPECTED was recorded on
EXPECTED = [    # (label, rc, error text or None, launches, digest of the outputs) after every call
    ('map_upload-s3-n0', -1, 'flb_map_upload: bad arguments (M=0 stride=3)', 0, 'd7c7dce3572ab8b3'),
    ('map_upload-s3-n1', 0, None, 7, '008eb841414dcc4e'),
    ('map_upload-s3-n7', 0, None, 7, '8d7990f0f8a422e9'),
    ('map_upload-s3-n8', 0, None, 7, '3fd35d75e0ceb9a7'),
    ('map_upload-s3-n9', 0, None, 7, 'edfcc27c096d2681'),
    ('map_upload-s3-n23', 0, None, 7, '5f8f499ba8edc558'),
    ('map_upload-s3-n24', 0, None, 7, '9860b27081489021'),
    ('map_upload-s3-n25', 0, None, 7, '723dbb33add3518e'),
    ('map_upload-s3-n3000', 0, None, 7, '0579101a21008ed8'),
    ('map_upload-s4-n0', -1, 'flb_map_upload: bad arguments (M=0 stride=4)', 0, '0579101a21008ed8'),
    ('map_upload-s4-n1', 0, None, 7, '008eb841414dcc4e'),
    ('map_upload-s4-n7', 0, None, 7, '8d7990f0f8a422e9'),
    ('map_upload-s4-n8', 0, None, 7, '3fd35d75e0ceb9a7'),
    ('map_upload-s4-n9', 0, None, 7, 'edfcc27c096d2681'),
    ('map_upload-s4-n23', 0, None, 7, '5f8f499ba8edc558'),
    ('map_upload-s4-n24', 0, None, 7, '9860b27081489021'),
    ('map_upload-s4-n25', 0, None, 7, '723dbb33add3518e'),
    ('map_upload-s4-n3000', 0, None, 7, '0579101a21008ed8'),
    ('map_upload-s12-n0', -1, 'flb_map_upload: bad arguments (M=0 stride=12)', 0, '0579101a21008ed8'),
    ('map_upload-s12-n1', 0, None, 7, '008eb841414dcc4e'),
    ('map_upload-s12-n7', 0, None, 7, '8d7990f0f8a422e9'),
    ('map_upload-s12-n8', 0, None, 7, '3fd35d75e0ceb9a7'),
    ('map_upload-s12-n9', 0, None, 7, 'edfcc27c096d2681'),
    ('map_upload-s12-n23', 0, None, 7, '5f8f499ba8edc558'),
    ('map_upload-s12-n24', 0, None, 7, '9860b27081489021'),
    ('map_upload-s12-n25', 0, None, 7, '723dbb33add3518e'),
    ('map_upload-s12-n3000', 0, None, 7, '0579101a21008ed8'),
    ('map_upload-signed-zero-neg-first', 0, None, 7, '2dc6d182fee348fb'),
    ('map_upload-signed-zero-pos-first', 0, None, 7, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-nan-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-+inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s3--inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s3-two-bad-3-17', -1, 'flb_map_upload: non-finite coordinate at point 3', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-nan-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-+inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s4--inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s4-two-bad-3-17', -1, 'flb_map_upload: non-finite coordinate at point 3', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-nan-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-+inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-x-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-x-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-x-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-x-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-y-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-y-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-y-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-y-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-z-first', -1, 'flb_map_upload: non-finite coordinate at point 0', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-z-middle', -1, 'flb_map_upload: non-finite coordinate at point 11', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-z-tail', -1, 'flb_map_upload: non-finite coordinate at point 25', 0, 'b7994c1f2489e128'),
    ('map_upload-s12--inf-z-last', -1, 'flb_map_upload: non-finite coordinate at point 29', 0, 'b7994c1f2489e128'),
    ('map_upload-s12-two-bad-3-17', -1, 'flb_map_upload: non-finite coordinate at point 3', 0, 'b7994c1f2489e128'),
    ('map_add_points-s3-n0', 0, None, 0, '5f22d40d5b64310c'),
    ('map_add_points-s3-n1', 0, None, 14, '5f9f704301587115'),
    ('map_add_points-s3-n7', 0, None, 14, 'd65d43cc004b74d1'),
    ('map_add_points-s3-n8', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s3-n9', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s3-n23', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s3-n24', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s3-n25', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s3-n3000', 0, None, 14, 'cbfce8044d2117e3'),
    ('map_add_points-s4-n0', 0, None, 0, '5f22d40d5b64310c'),
    ('map_add_points-s4-n1', 0, None, 14, '5f9f704301587115'),
    ('map_add_points-s4-n7', 0, None, 14, 'd65d43cc004b74d1'),
    ('map_add_points-s4-n8', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s4-n9', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s4-n23', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s4-n24', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s4-n25', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s4-n3000', 0, None, 14, 'cbfce8044d2117e3'),
    ('map_add_points-s12-n0', 0, None, 0, '5f22d40d5b64310c'),
    ('map_add_points-s12-n1', 0, None, 14, '5f9f704301587115'),
    ('map_add_points-s12-n7', 0, None, 14, 'd65d43cc004b74d1'),
    ('map_add_points-s12-n8', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s12-n9', 0, None, 14, 'c0b6ceee2ec2ac57'),
    ('map_add_points-s12-n23', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s12-n24', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s12-n25', 0, None, 14, '2fd34fed628cd783'),
    ('map_add_points-s12-n3000', 0, None, 14, 'cbfce8044d2117e3'),
    ('map_add_points-nan-x-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-x-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-x-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-x-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-y-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-y-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-y-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-y-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-z-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-z-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-z-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-z-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-x-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-x-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-x-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-x-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-y-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-y-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-y-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-y-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-z-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-z-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-z-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-+inf-z-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-x-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-x-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-x-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-x-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-y-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-y-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-y-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-y-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-z-first', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-z-middle', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-z-tail', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points--inf-z-last', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-two-bad-3-17', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-far', -1, 'flb_map_add_points: coordinate / downsample_size exceeds 2^20 voxels', 0, '5f22d40d5b64310c'),
    ('map_add_points-far-and-nan', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('map_add_points-nan-and-far', -1, 'flb_map_add_points: non-finite coordinate', 0, '5f22d40d5b64310c'),
    ('scan_upload-s3-n0', 0, None, 0, '062432175762eb56'),
    ('scan_upload-s3-n1', 0, None, 1, 'aa42372971933981'),
    ('scan_upload-s3-n7', 0, None, 1, 'bd4660c390038c4a'),
    ('scan_upload-s3-n8', 0, None, 1, '803aee46d09d11ff'),
    ('scan_upload-s3-n9', 0, None, 1, 'a0ac51f1e43be543'),
    ('scan_upload-s3-n23', 0, None, 1, 'be644c3a9ac8b74b'),
    ('scan_upload-s3-n24', 0, None, 1, '6e7685cc2dc71efa'),
    ('scan_upload-s3-n25', 0, None, 1, 'cec05d6dbed4b783'),
    ('scan_upload-s3-n3000', 0, None, 1, 'deead6d928c9d7bb'),
    ('scan_upload-s4-n0', 0, None, 0, '062432175762eb56'),
    ('scan_upload-s4-n1', 0, None, 1, 'aa42372971933981'),
    ('scan_upload-s4-n7', 0, None, 1, 'bd4660c390038c4a'),
    ('scan_upload-s4-n8', 0, None, 1, '803aee46d09d11ff'),
    ('scan_upload-s4-n9', 0, None, 1, 'a0ac51f1e43be543'),
    ('scan_upload-s4-n23', 0, None, 1, 'be644c3a9ac8b74b'),
    ('scan_upload-s4-n24', 0, None, 1, '6e7685cc2dc71efa'),
    ('scan_upload-s4-n25', 0, None, 1, 'cec05d6dbed4b783'),
    ('scan_upload-s4-n3000', 0, None, 1, 'deead6d928c9d7bb'),
    ('scan_upload-s12-n0', 0, None, 0, '062432175762eb56'),
    ('scan_upload-s12-n1', 0, None, 1, 'aa42372971933981'),
    ('scan_upload-s12-n7', 0, None, 1, 'bd4660c390038c4a'),
    ('scan_upload-s12-n8', 0, None, 1, '803aee46d09d11ff'),
    ('scan_upload-s12-n9', 0, None, 1, 'a0ac51f1e43be543'),
    ('scan_upload-s12-n23', 0, None, 1, 'be644c3a9ac8b74b'),
    ('scan_upload-s12-n24', 0, None, 1, '6e7685cc2dc71efa'),
    ('scan_upload-s12-n25', 0, None, 1, 'cec05d6dbed4b783'),
    ('scan_upload-s12-n3000', 0, None, 1, 'deead6d928c9d7bb'),
    ('scan_upload-pinned-s3-n0', 0, None, 0, '062432175762eb56'),
    ('scan_upload-pinned-s3-n1', 0, None, 1, 'aa42372971933981'),
    ('scan_upload-pinned-s3-n7', 0, None, 1, 'bd4660c390038c4a'),
    ('scan_upload-pinned-s3-n8', 0, None, 1, '803aee46d09d11ff'),
    ('scan_upload-pinned-s3-n9', 0, None, 1, 'a0ac51f1e43be543'),
    ('scan_upload-pinned-s3-n23', 0, None, 1, 'be644c3a9ac8b74b'),
    ('scan_upload-pinned-s3-n24', 0, None, 1, '6e7685cc2dc71efa'),
    ('scan_upload-pinned-s3-n25', 0, None, 1, 'cec05d6dbed4b783'),
    ('scan_upload-pinned-s3-n3000', 0, None, 1, 'deead6d928c9d7bb'),
    ('scan_upload-pinned-s12-n0', 0, None, 0, '062432175762eb56'),
    ('scan_upload-pinned-s12-n1', 0, None, 1, 'aa42372971933981'),
    ('scan_upload-pinned-s12-n7', 0, None, 1, 'bd4660c390038c4a'),
    ('scan_upload-pinned-s12-n8', 0, None, 1, '803aee46d09d11ff'),
    ('scan_upload-pinned-s12-n9', 0, None, 1, 'a0ac51f1e43be543'),
    ('scan_upload-pinned-s12-n23', 0, None, 1, 'be644c3a9ac8b74b'),
    ('scan_upload-pinned-s12-n24', 0, None, 1, '6e7685cc2dc71efa'),
    ('scan_upload-pinned-s12-n25', 0, None, 1, 'cec05d6dbed4b783'),
    ('scan_upload-pinned-s12-n3000', 0, None, 1, 'deead6d928c9d7bb'),
    ('scan_upload-signed-zero-neg-first', 0, None, 1, '3594116d8f57b858'),
    ('scan_upload-signed-zero-pos-first', 0, None, 1, '3594116d8f57b858'),
    ('scan_upload-nan-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-x-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-x-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-x-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-y-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-y-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-y-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-y-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-z-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-z-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-z-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-nan-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-x-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-x-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-x-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-y-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-y-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-y-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-y-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-z-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-z-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-z-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-+inf-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-x-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-x-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-x-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-y-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-y-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-y-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-y-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-z-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-z-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-z-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload--inf-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-two-bad-3-17', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned-nan-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned-nan-y-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned-nan-z-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned-+inf-x-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned-+inf-z-first', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned--inf-x-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned--inf-y-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('scan_upload-pinned--inf-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, '3594116d8f57b858'),
    ('frame_enqueue-s3-n1', 0, None, 4, '779f64d9d5b7c896'),
    ('frame_enqueue-s3-n9', 0, None, 4, '3e7747dff327af26'),
    ('frame_enqueue-s3-n25', 0, None, 4, 'd33006e37ec6139d'),
    ('frame_enqueue-s3-n3000', 0, None, 4, 'c1019cf9d5669a0c'),
    ('frame_enqueue-s4-n1', 0, None, 4, '779f64d9d5b7c896'),
    ('frame_enqueue-s4-n9', 0, None, 4, '3e7747dff327af26'),
    ('frame_enqueue-s4-n25', 0, None, 4, 'd33006e37ec6139d'),
    ('frame_enqueue-s4-n3000', 0, None, 4, 'c1019cf9d5669a0c'),
    ('frame_enqueue-s12-n1', 0, None, 4, '779f64d9d5b7c896'),
    ('frame_enqueue-s12-n9', 0, None, 4, '3e7747dff327af26'),
    ('frame_enqueue-s12-n25', 0, None, 4, 'd33006e37ec6139d'),
    ('frame_enqueue-s12-n3000', 0, None, 4, 'c1019cf9d5669a0c'),
    ('frame_enqueue-nan-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('frame_enqueue-nan-y-last', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('frame_enqueue-+inf-x-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('frame_enqueue-+inf-z-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('frame_enqueue--inf-y-first', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('frame_enqueue--inf-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, 'e593acbab72418cb'),
    ('batch_set_frame-s3-n1', 0, None, 2, '5f7a68b5792d61f9'),
    ('batch_set_frame-s3-n9', 0, None, 2, '5e120359f9cd5256'),
    ('batch_set_frame-s3-n25', 0, None, 2, '5d9c531f82278eb6'),
    ('batch_set_frame-s3-n3000', 0, None, 2, 'c1008f08773a61d4'),
    ('batch_set_frame-s4-n1', 0, None, 2, '5f7a68b5792d61f9'),
    ('batch_set_frame-s4-n9', 0, None, 2, '5e120359f9cd5256'),
    ('batch_set_frame-s4-n25', 0, None, 2, '5d9c531f82278eb6'),
    ('batch_set_frame-s4-n3000', 0, None, 2, 'c1008f08773a61d4'),
    ('batch_set_frame-s12-n1', 0, None, 2, '5f7a68b5792d61f9'),
    ('batch_set_frame-s12-n9', 0, None, 2, '5e120359f9cd5256'),
    ('batch_set_frame-s12-n25', 0, None, 2, '5d9c531f82278eb6'),
    ('batch_set_frame-s12-n3000', 0, None, 2, 'c1008f08773a61d4'),
    ('batch_set_frame-nan-x-first', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('batch_set_frame-nan-y-last', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('batch_set_frame-+inf-x-tail', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('batch_set_frame-+inf-z-middle', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('batch_set_frame--inf-y-first', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('batch_set_frame--inf-z-last', -1, 'flb_scan_upload: non-finite coordinate', 0, 'c1008f08773a61d4'),
    ('voxel_grid-s3-n0', 0, None, 0, '7b2a54d3d7e98d39'),
    ('voxel_grid-s3-n1', 0, None, 11, '16b7749193615425'),
    ('voxel_grid-s3-n7', 0, None, 11, '4a84229821b15da7'),
    ('voxel_grid-s3-n8', 0, None, 11, 'a68bec9eff6ddcca'),
    ('voxel_grid-s3-n9', 0, None, 11, 'aa2d1ed6deb4be3f'),
    ('voxel_grid-s3-n23', 0, None, 11, '8daeefe9175a02f4'),
    ('voxel_grid-s3-n24', 0, None, 11, 'db5a34ac7c8dd8d2'),
    ('voxel_grid-s3-n25', 0, None, 11, '6919003ec46d2ecf'),
    ('voxel_grid-s3-n3000', 0, None, 11, '326fbf2eae562314'),
    ('voxel_grid-s4-n0', 0, None, 0, '7b2a54d3d7e98d39'),
    ('voxel_grid-s4-n1', 0, None, 11, '16b7749193615425'),
    ('voxel_grid-s4-n7', 0, None, 11, '4a84229821b15da7'),
    ('voxel_grid-s4-n8', 0, None, 11, 'a68bec9eff6ddcca'),
    ('voxel_grid-s4-n9', 0, None, 11, 'aa2d1ed6deb4be3f'),
    ('voxel_grid-s4-n23', 0, None, 11, '8daeefe9175a02f4'),
    ('voxel_grid-s4-n24', 0, None, 11, 'db5a34ac7c8dd8d2'),
    ('voxel_grid-s4-n25', 0, None, 11, '6919003ec46d2ecf'),
    ('voxel_grid-s4-n3000', 0, None, 11, '326fbf2eae562314'),
    ('voxel_grid-s12-n0', 0, None, 0, '7b2a54d3d7e98d39'),
    ('voxel_grid-s12-n1', 0, None, 11, '16b7749193615425'),
    ('voxel_grid-s12-n7', 0, None, 11, '4a84229821b15da7'),
    ('voxel_grid-s12-n8', 0, None, 11, 'a68bec9eff6ddcca'),
    ('voxel_grid-s12-n9', 0, None, 11, 'aa2d1ed6deb4be3f'),
    ('voxel_grid-s12-n23', 0, None, 11, '8daeefe9175a02f4'),
    ('voxel_grid-s12-n24', 0, None, 11, 'db5a34ac7c8dd8d2'),
    ('voxel_grid-s12-n25', 0, None, 11, '6919003ec46d2ecf'),
    ('voxel_grid-s12-n3000', 0, None, 11, '326fbf2eae562314'),
    ('voxel_grid-signed-zero-neg-first', 0, None, 11, '4d6289b4c90faa7b'),
    ('voxel_grid-signed-zero-pos-first', 0, None, 11, '4d6289b4c90faa7b'),
    ('voxel_grid-nan-x-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-x-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-x-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-x-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-y-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-y-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-y-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-y-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-z-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-z-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-z-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-nan-z-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-x-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-x-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-x-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-x-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-y-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-y-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-y-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-y-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-z-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-z-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-z-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid-+inf-z-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-x-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-x-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-x-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-x-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-y-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-y-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-y-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-y-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-z-first', -1, 'flb_voxel_grid: non-finite coordinate at point 0', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-z-middle', -1, 'flb_voxel_grid: non-finite coordinate at point 11', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-z-tail', -1, 'flb_voxel_grid: non-finite coordinate at point 25', 0, '214959afb4f146d6'),
    ('voxel_grid--inf-z-last', -1, 'flb_voxel_grid: non-finite coordinate at point 29', 0, '214959afb4f146d6'),
    ('voxel_grid-two-bad-3-17', -1, 'flb_voxel_grid: non-finite coordinate at point 3', 0, '214959afb4f146d6'),
    ('visual_candidates-s3-n0', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n1', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n7', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n8', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n9', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n23', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n24', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n25', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s3-n3000', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n0', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n1', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n7', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n8', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n9', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n23', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n24', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n25', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s4-n3000', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n0', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n1', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n7', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n8', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n9', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n23', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n24', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n25', 0, None, 3, 'ea218265c8508654'),
    ('visual_candidates-s12-n3000', 0, None, 3, 'ea218265c8508654'),
    ('vmap_select-s3-n0', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n1', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n7', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n8', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n9', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n23', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n24', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n25', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s3-n3000', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n0', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n1', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n7', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n8', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n9', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n23', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n24', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n25', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s4-n3000', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n0', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n1', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n7', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n8', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n9', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n23', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n24', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n25', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-s12-n3000', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-nan-x-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-x-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-x-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-x-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-y-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-y-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-y-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-y-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-z-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-z-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-z-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-z-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-x-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-x-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-x-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-x-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-y-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-y-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-y-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-y-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-z-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-z-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-z-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+inf-z-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-x-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-x-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-x-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-x-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-y-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-y-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-y-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-y-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-z-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-z-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-z-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--inf-z-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-two-bad-3-17', -1, 'visual map: coordinate 3 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+lim-x', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select--lim-x', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-+beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+lim-y', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select--lim-y', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-+beyond-y', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--beyond-y', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-+lim-z', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select--lim-z', 0, None, 6, 'df3f619804a92fdb'),
    ('vmap_select-+beyond-z', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select--beyond-z', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-beyond-then-nan', -1, 'visual map: coordinate 4 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_select-nan-then-beyond', -1, 'visual map: coordinate 4 non-finite or beyond 2^20 voxels', 0, 'dd834710f8167e94'),
    ('vmap_grow-s3-n1', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s3-n9', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s3-n25', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s3-n3000', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s4-n1', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s4-n9', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s4-n25', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s4-n3000', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s12-n1', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s12-n9', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s12-n25', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-s12-n3000', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-nan-x-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow-nan-y-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow-+inf-x-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow-+inf-z-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow--inf-y-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow--inf-z-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow-+lim-x', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow--lim-x', 0, None, 5, 'e3b0c44298fc1c14'),
    ('vmap_grow-+beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow--beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, 'e3b0c44298fc1c14'),
    ('vmap_grow-after', 0, None, 6, '994b65f23f87b96d'),
    ('colorize-s3-n1', 0, None, 1, '982c5dd61df76ddf'),
    ('colorize-s3-n9', 0, None, 1, 'ff718baaf3fd2f91'),
    ('colorize-s3-n25', 0, None, 1, '20af711d4e02421d'),
    ('colorize-s3-n3000', 0, None, 1, '3c095ddcc5e60c7a'),
    ('colorize-s4-n1', 0, None, 1, '982c5dd61df76ddf'),
    ('colorize-s4-n9', 0, None, 1, 'ff718baaf3fd2f91'),
    ('colorize-s4-n25', 0, None, 1, '20af711d4e02421d'),
    ('colorize-s4-n3000', 0, None, 1, '3c095ddcc5e60c7a'),
    ('colorize-s12-n1', 0, None, 1, '982c5dd61df76ddf'),
    ('colorize-s12-n9', 0, None, 1, 'ff718baaf3fd2f91'),
    ('colorize-s12-n25', 0, None, 1, '20af711d4e02421d'),
    ('colorize-s12-n3000', 0, None, 1, '3c095ddcc5e60c7a'),
    ('colorize-nan-x-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize-nan-y-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize-+inf-x-tail', -1, 'visual map: coordinate 25 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize-+inf-z-middle', -1, 'visual map: coordinate 11 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize--inf-y-first', -1, 'visual map: coordinate 0 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize--inf-z-last', -1, 'visual map: coordinate 29 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize-+lim-x', 0, None, 1, '4b67a473be61fd7f'),
    ('colorize--lim-x', 0, None, 1, '4b67a473be61fd7f'),
    ('colorize-+beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
    ('colorize--beyond-x', -1, 'visual map: coordinate 9 non-finite or beyond 2^20 voxels', 0, '96a7c72dd059118d'),
]


def test_point_uploads_pinned(flb):
    assert device() == DEVICE, "recorded on %s with %d SMs: these values hold for that card only" % DEVICE
    got = run_sequence(flb)
    assert [g[0] for g in got] == [e[0] for e in EXPECTED]
    for g, e in zip(got, EXPECTED):
        assert g == e, g[0]
