import os

import numpy as np

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "T0_golden.npz")


class _Cfg:
    def __init__(self, a):
        self.laser_point_cov, self.img_point_cov, self.cell_size = float(a[0]), float(a[1]), float(a[2])


REF_GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ikdtree_ref.npz")


def load_ref_golden():
    """What the reference's own ikd-Tree returned on the tests' inputs (tests/golden/make_golden_ref.py)."""
    return dict(np.load(REF_GOLD))


def digest(*arrays):
    """SHA-256 of the arrays' exact bytes (shape and dtype included): bit equality with a stored result."""
    import hashlib
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(f"{a.dtype.str}{a.shape}".encode())
        h.update(a.tobytes())
    return h.hexdigest()


def assert_digest(g, key, *arrays, expected=None):
    """Bit equality of `arrays` with the stored result g[key].  On a mismatch the message gives the shapes and, where the
    caller can recompute the expected arrays on the CPU (`expected()` returns them), the first differing row."""
    if digest(*arrays) == str(g[key]):
        return
    msg = [f"{key}: result differs from the stored reference result (shapes {[np.shape(a) for a in arrays]})"]
    if expected is not None:
        exp = expected()
        if digest(*exp) != str(g[key]):
            msg.append("the CPU recomputation does not match the stored result either")
        for a, e in zip(arrays, exp):
            a, e = np.asarray(a), np.asarray(e)
            if a.shape != e.shape:
                msg.append(f"shape {a.shape}, expected {e.shape}")
                continue
            bad = np.nonzero((a != e).reshape(len(a), -1).any(1))[0]
            if len(bad):
                msg.append(f"{len(bad)} of {len(a)} rows differ, first row {bad[0]}: {a[bad[0]]!r}, expected {e[bad[0]]!r}")
    raise AssertionError("; ".join(msg))


def rows(a):
    """Sorted view of an (n,3) float32 array as rows, for exact set comparison."""
    a = np.ascontiguousarray(a, np.float32)
    return np.sort(a.view(np.dtype((np.void, 12))).ravel())


def world_scan(f):
    return ((f["R_true"] @ (f["R_LI"] @ f["scan_body"].T.astype(np.float64) + f["t_LI"][:, None])).T + f["p_true"]).astype(np.float32)


ADD_POINTS_CASES = [("T0", 0.3), ("T1", 0.3), ("T1", 0.5), ("C2", 0.3)]


def DELETE_BOXES(f):
    lo, hi = f["map_xyz"].min(0), f["map_xyz"].max(0)
    return np.array([[lo[0], lo[1], lo[2], lo[0] + 6, lo[1] + 40, hi[2] + 1],      # a slab along one wall
                     [0.0, 0.0, -1.0, 4.0, 4.0, 3.0],                              # a chunk in the middle
                     [hi[0] - 0.01, lo[1], lo[2], hi[0] + 1, hi[1] + 1, hi[2] + 1]], np.float32)


def lattice_fixture():
    """A map on a 0.25 m integer lattice and queries on lattice points and cell centres: exact float distance ties."""
    g = np.arange(-8, 9, dtype=np.float32) * 0.25
    lat = np.stack(np.meshgrid(g, g, g[:5], indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    rng = np.random.default_rng(3)
    lat = lat[rng.permutation(len(lat))]
    q = np.concatenate([lat[:400], lat[400:800] + np.float32(0.125), lat[800:1000] + np.array([0.125, 0, 0], np.float32)]).astype(np.float32)
    return lat, q


def load_golden():
    g = dict(np.load(GOLD))
    c = g["cam"]
    frame = {k: g[k] for k in ("map_xyz", "scan_body", "R_prop", "p_prop", "cov", "vel", "bg", "ba", "grav", "R_LI", "t_LI",
                               "Rcl", "Pcl", "image", "patch_pos", "patch_ref", "patch_level")}
    frame["cam"] = dict(width=int(c[0]), height=int(c[1]), fx=c[2], fy=c[3], cx=c[4], cy=c[5], d=tuple(c[6:11]))
    frame["cfg"] = _Cfg(g["cfg"])
    return frame, g
