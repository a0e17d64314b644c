"""Edge fixtures of the VIO photometric update, shared by its CPU and GPU tiers.

The update reads an 8x8 patch through a lattice of taps `scale` pixels apart around an integer anchor
(src/lidar_selection.cpp:809-837).  The reference reads those pixels unchecked; the oracle and the device skip and count
a patch that is behind the camera, projects to |pc| >= 1e6, or whose taps leave the image (DESIGN, "Deliberate,
documented deviations").  The fixtures here put patches exactly on that guard: the last anchor cell whose taps still
fit and the first one past it on every side and at every scale, anchors where `floorf((float)(pc / scale))` rounds up,
depths at and behind the camera, and a projection that folds back into the image.  `expected_valid` states the guard
again from the reference's own read offsets, so the tests do not take the product's constant 5 on trust.

numpy and synth only: nothing here needs a GPU, the oracle or the product library.  The pose and
projection arithmetic follows the oracle's operation order (oracle/flo_oracle.cpp mat3_mul / mat3_vec / flo_world2cam),
so the pc computed here is the pc the oracle and the device compute, to the last bit."""
import functools

import numpy as np

SIZES = [(320, 256), (321, 257), (333, 251)]   # 321 x 257: W-1 and H-1 are multiples of 16
CAMERAS = ["pinhole", "radtan", "k1"]
SCALES = (1, 2, 4, 8, 16)
FRACTIONS = (0.0, 0.37, 1.0 - 2.0 ** -20)
SIDES = ("left", "right", "top", "bottom")
K1_CAMERA_D = (-0.35, 0.0, 0.0, 0.0, 0.0)      # x (1 - 0.35 r^2) is not monotonic past r = 0.976


# ------------------------------------------------------------------------- pose / projection in the oracle's order
def _mm(A, B):
    return np.array([[A[i, 0] * B[0, j] + A[i, 1] * B[1, j] + A[i, 2] * B[2, j] for j in range(3)] for i in range(3)])


def _mv(A, v):
    """A (3, 3) times each row of v (..., 3), summed left to right like mat3_vec."""
    v = np.asarray(v, np.float64)
    return np.stack([A[i, 0] * v[..., 0] + A[i, 1] * v[..., 1] + A[i, 2] * v[..., 2] for i in range(3)], axis=-1)


def extrinsics(R_LI, t_LI, Rcl, Pcl):
    """(Rci, Pci) as LidarSelector::init forms them (src/lidar_selection.cpp:41-52; oracle vio_constants)."""
    Rli = np.asarray(R_LI, np.float64).T.copy()
    Pli = -_mv(Rli, t_LI)
    Rci = _mm(np.asarray(Rcl, np.float64), Rli)
    Pci = _mv(np.asarray(Rcl, np.float64), Pli) + np.asarray(Pcl, np.float64)
    return Rci, Pci


def synth_extrinsics():
    from fastlivo_loader import load
    s = load().synth
    return extrinsics(s.AVIA_EXTRINSIC_R, s.AVIA_EXTRINSIC_T, s.AVIA_RCL, s.AVIA_PCL)


def to_camera(Rci, Pci, R, p, pos):
    """pf = Rcw * pos + Pcw with Rcw = Rci * R^T, Pcw = -Rci R^T p + Pci (src/lidar_selection.cpp:780-781, :800)."""
    Rcw = _mm(Rci, np.asarray(R, np.float64).T.copy())
    Pcw = -_mv(Rcw, p) + Pci
    return _mv(Rcw, pos) + Pcw


def project(cam, pf):
    """vikit PinholeCamera::world2cam (flo_world2cam), vectorised with the same operation order."""
    pf = np.asarray(pf, np.float64)
    with np.errstate(all="ignore"):
        x, y = pf[..., 0] / pf[..., 2], pf[..., 1] / pf[..., 2]
        d = cam["d"]
        if not abs(d[0]) > 0.0000001:
            return np.stack([cam["fx"] * x + cam["cx"], cam["fy"] * y + cam["cy"]], axis=-1)
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        a1, a2, a3 = 2 * x * y, r2 + 2 * x * x, r2 + 2 * y * y
        cdist = 1 + d[0] * r2 + d[1] * r4 + d[4] * r6
        xd = x * cdist + d[2] * a1 + d[3] * a2
        yd = y * cdist + d[2] * a3 + d[3] * a1
        return np.stack([xd * cam["fx"] + cam["cx"], yd * cam["fy"] + cam["cy"]], axis=-1)


def anchor(pc, scale):
    """The integer anchor of src/lidar_selection.cpp:809: floorf of the FLOAT quotient, so a quotient just below an
    integer rounds up to it.  pc must be finite and below 1e6 in magnitude."""
    q = np.float32(np.asarray(pc, np.float64) / scale)
    return (np.floor(q) * np.float32(scale)).astype(np.int64)


# Read offsets of one pixel, in units of scale, from its base img_ptr (src/lidar_selection.cpp:818-837): the gradient and
# the residual read img_ptr[{-s, 0, s, 2s}] along a row and img_ptr[{-s, 0, s, 2s} * width] across rows, and pixel
# (x, y) of the 8x8 patch has its base at row v_i + (x - 4) s, column u_i + (y - 4) s.
_READ = np.array([-1, 0, 1, 2])
_BASE = np.arange(8) - 4
_FOOT_LO = int((_BASE[:, None] + _READ[None, :]).min())
_FOOT_HI = int((_BASE[:, None] + _READ[None, :]).max())


def expected_valid(cam, R, p, pos, search_level, level, ext=None):
    """Which patches the update reads at pose (R, p): in front of the camera, |pc| < 1e6, and the union of the
    reference's reads inside [0, W-1] x [0, H-1].  Returns (valid, box, scale, pf, pc); box = (col_lo, col_hi, row_lo,
    row_hi) of the reads (meaningful where the first two conditions hold)."""
    Rci, Pci = synth_extrinsics() if ext is None else ext
    pf = to_camera(Rci, Pci, R, p, pos)
    pc = project(cam, pf)
    scale = 1 << (level + np.asarray(search_level, np.int64))
    front = pf[:, 2] > 0.0
    with np.errstate(invalid="ignore"):
        near = front & (np.abs(pc[:, 0]) < 1e6) & (np.abs(pc[:, 1]) < 1e6)
    safe = np.where(near[:, None], pc, 0.0)
    u_i, v_i = anchor(safe[:, 0], scale), anchor(safe[:, 1], scale)
    box = np.stack([u_i + _FOOT_LO * scale, u_i + _FOOT_HI * scale, v_i + _FOOT_LO * scale, v_i + _FOOT_HI * scale], axis=1)
    inside = (box[:, 0] >= 0) & (box[:, 1] <= cam["width"] - 1) & (box[:, 2] >= 0) & (box[:, 3] <= cam["height"] - 1)
    return near & inside, box, scale, pf, pc


# ------------------------------------------------------------------------- placement
def _from_camera(Rci, Pci, R, p, pf):
    """The world point whose camera coordinates at pose (R, p) are pf: to_camera inverted by a solve (the configured Rcl
    is orthonormal only to about 1e-6) and one refinement step."""
    Rcw = _mm(Rci, np.asarray(R, np.float64).T.copy())
    pf = np.asarray(pf, np.float64)
    pos = np.linalg.solve(Rcw, (pf - to_camera(Rci, Pci, R, p, np.zeros(3))).T).T
    return pos + np.linalg.solve(Rcw, (pf - to_camera(Rci, Pci, R, p, pos)).T).T


def _ref_patches(ref_image, uv, search_level):
    """patch[64 pyr + 8 row + col] = bilinear(ref, uv + (col-4, row-4) * 2^(search_level + pyr)), clamped into the image."""
    from fastlivo_loader import load
    bilinear_u8 = load().synth.bilinear_u8
    H, W = ref_image.shape
    n = len(uv)
    rr, cc = np.meshgrid(np.arange(8) - 4, np.arange(8) - 4, indexing="ij")
    out = np.empty((n, 3, 64), np.float32)
    uv = np.clip(np.nan_to_num(uv, nan=0.0), -1e6, 1e6)
    for pyr in range(3):
        s = (1 << np.asarray(search_level))[:, None, None] * (1 << pyr)
        su = np.clip(uv[:, 0, None, None] + cc[None] * s, 0, W - 1.001).reshape(n, 64)
        sv = np.clip(uv[:, 1, None, None] + rr[None] * s, 0, H - 1.001).reshape(n, 64)
        out[:, pyr, :] = bilinear_u8(ref_image, su, sv)
    return out


def place(frame, R, p, targets, depth, search_level):
    """World points whose projection at pose (R, p) through frame["cam"] lands on `targets` (n, 2) pixels at camera
    depth `depth`.  The camera ray times the depth is the start; Newton steps on the projection (radtan or not) then
    bring every point within 1e-9 px of its target.  Returns dict(pos, pc, pf, patch_ref) with pc / pf recomputed from
    the returned pos: patches are classified by what was achieved, never by the request."""
    cam = frame["cam"]
    ext = extrinsics(frame["R_LI"], frame["t_LI"], frame["Rcl"], frame["Pcl"])
    t = np.asarray(targets, np.float64).reshape(-1, 2)
    d = np.broadcast_to(np.asarray(depth, np.float64), (len(t),))
    sl = np.broadcast_to(np.asarray(search_level, np.int32), (len(t),)).copy()

    def fwd(xy):
        pf = np.stack([xy[:, 0] * d, xy[:, 1] * d, d], axis=1)
        pos = _from_camera(*ext, R, p, pf)
        pf2 = to_camera(*ext, R, p, pos)
        return pos, pf2, project(cam, pf2)

    xy = np.stack([(t[:, 0] - cam["cx"]) / cam["fx"], (t[:, 1] - cam["cy"]) / cam["fy"]], axis=1)
    for _ in range(60):
        pos, pf, pc = fwd(xy)
        r = t - pc
        if np.abs(r).max() < 1e-9:
            break
        h = 1e-7
        J = np.empty((len(t), 2, 2))
        for k in range(2):
            e = np.zeros(2)
            e[k] = h
            J[:, :, k] = (fwd(xy + e)[2] - fwd(xy - e)[2]) / (2 * h)
        xy = xy + np.linalg.solve(J, r[:, :, None])[:, :, 0]
    assert np.abs(t - pc).max() < 1e-9, np.abs(t - pc).max()
    return dict(pos=pos, pc=pc, pf=pf, patch_ref=_ref_patches(frame["ref_image"], t, sl), level=sl)


def place_camera_points(frame, R, p, pf, uv_ref):
    """World points at given camera coordinates pf (no projection target: depths at or behind the camera, far off-axis
    points).  Reference patches are sampled around uv_ref."""
    ext = extrinsics(frame["R_LI"], frame["t_LI"], frame["Rcl"], frame["Pcl"])
    pos = _from_camera(*ext, R, p, pf)
    pf2 = to_camera(*ext, R, p, pos)
    pc = project(frame["cam"], pf2)
    sl = np.zeros(len(pos), np.int32)
    return dict(pos=pos, pc=pc, pf=pf2, patch_ref=_ref_patches(frame["ref_image"], np.asarray(uv_ref, np.float64), sl), level=sl)


# ------------------------------------------------------------------------- targets
def edge_targets(W, H, rng):
    """(targets (n, 2), search_level (n,)) of the anchor-cell edges.  For every search level sl and run level L
    (scale s = 2^(sl + L), every s in SCALES), on every side: the last anchor cell whose taps fit and the first one past
    it, at the sub-pixel fractions FRACTIONS of a cell, and the quotient pc / s a quarter float ulp below the integer
    between them, which floorf((float)...) rounds up.  The other coordinate sits near the image centre."""
    tg, sls = [], []
    for sl in range(3):
        for L in range(3):
            s = 1 << (sl + L)
            for side in SIDES:
                n = W if side in ("left", "right") else H
                if side in ("left", "top"):
                    cells = (5, 4)                                   # first cell that fits, the one before it
                    k_round = 5                                      # (k - ulp/4) rounds up to k: fits only in float
                else:
                    k_fit = (n - 1 - 5 * s) // s
                    cells = (k_fit, k_fit + 1)
                    k_round = k_fit + 1                              # rounds up past the last fitting cell
                q = [k + f for k in cells for f in FRACTIONS]
                q.append(k_round - float(np.spacing(np.float32(k_round))) / 4)
                a = np.array(q) * s
                m = (W if side in ("top", "bottom") else H)
                b = m / 2 + rng.uniform(-8, 8, len(a))
                tg.append(np.stack([a, b], 1) if side in ("left", "right") else np.stack([b, a], 1))
                sls.append(np.full(len(a), sl, np.int32))
    return np.concatenate(tg), np.concatenate(sls)


@functools.lru_cache(maxsize=None)
def base_frame(W, H):
    """A rendered synthetic frame (scene, image, reference image, poses) at W x H, pinhole camera."""
    if W < 160 or H < 160:        # too small for synth's patch border: the centre of a 320 x 256 frame
        f = dict(base_frame(320, 256))
        x0, y0 = (320 - W) // 2, (256 - H) // 2
        f["image"] = np.ascontiguousarray(f["image"][y0:y0 + H, x0:x0 + W])
        f["ref_image"] = np.ascontiguousarray(f["ref_image"][y0:y0 + H, x0:x0 + W])
        f["cam"] = dict(f["cam"], width=W, height=H, cx=f["cam"]["cx"] - x0, cy=f["cam"]["cy"] - y0)
        return f
    from fastlivo_loader import load
    synth = load().synth
    cfg = synth.FrameConfig(f"E{W}x{H}", n_scan=600, n_map=6000, pitch=0.3, img_w=W, img_h=H, n_patch=8, seed=20261017)
    return synth.make_frame(cfg)


def camera(frame, which):
    cam = dict(frame["cam"])
    if which == "radtan":
        from fastlivo_loader import load
        cam["d"] = tuple(load().synth.PINHOLE["d"])              # the T1 camera's distortion
    elif which == "k1":
        cam["fx"], cam["fy"] = 2 * cam["fx"], 2 * cam["fy"]      # narrower view: the image edges stay below r = 0.976
        cam["d"] = K1_CAMERA_D
    return cam


@functools.lru_cache(maxsize=None)
def scenario(W, H, which, depth_points=False, search_level=None, n_interior=48):
    """One frame with interior, edge, depth and fold-back patches, all placed at the true pose (where they are
    photometrically consistent, so the update from the prior converges).  The depth and fold-back patches come only with
    depth_points: a patch a micrometre in front of the camera has Jacobians of 1 / pf[2] and would dominate an update.  search_level forces every patch's level.
    Returns a frame dict (the keys synth.make_frame returns) plus "kind" per patch."""
    f = dict(base_frame(W, H))
    f["cam"] = camera(f, which)
    rng = np.random.default_rng(7 + 31 * W + H + CAMERAS.index(which))
    R, p = f["R_true"], f["p_true"]
    parts, kinds = [], []
    border = 64 if search_level is None else 24
    uv = np.stack([rng.uniform(border, W - 1 - border, n_interior), rng.uniform(border, H - 1 - border, n_interior)], 1)
    sl = (rng.uniform(size=n_interior) < 0.1).astype(np.int32) if search_level is None else np.full(n_interior, search_level, np.int32)
    parts.append(place(f, R, p, uv, rng.uniform(2.5, 6.0, n_interior), sl))
    kinds += ["interior"] * n_interior
    if search_level is None:
        tg, sl = edge_targets(W, H, rng)
        parts.append(place(f, R, p, tg, rng.uniform(2.5, 6.0, len(tg)), sl))
        kinds += ["edge"] * len(tg)
    if depth_points:
        c = np.array([W / 2 + 3.3, H / 2 - 2.7])
        xy = (c - [f["cam"]["cx"], f["cam"]["cy"]]) / [f["cam"]["fx"], f["cam"]["fy"]]
        zs = np.array([-1.0, 1e-12, -1e-12, 1e-3])
        pf = np.concatenate([np.stack([xy[0] * zs, xy[1] * zs, zs], 1),
                             [[1e-3, 5e-4, 1e-7]],                                     # |pc| ~ 1e10
                             [np.r_[np.tan(np.deg2rad(60)) * np.array([np.cos(0.3), np.sin(0.3)]), 1.0] * 4.0]])   # fold-back
        d = place_camera_points(f, R, p, pf, np.tile(c, (len(pf), 1)))
        d["patch_ref"][-1] = _ref_patches(f["ref_image"], np.clip(d["pc"][-1:], 0, [W - 1, H - 1]), np.zeros(1, np.int32))[0]
        parts.append(d)
        kinds += ["depth"] * 5 + ["fold"]
    f["patch_pos"] = np.ascontiguousarray(np.concatenate([q["pos"] for q in parts]))
    f["patch_ref"] = np.ascontiguousarray(np.concatenate([q["patch_ref"] for q in parts]))
    f["patch_level"] = np.ascontiguousarray(np.concatenate([q["level"] for q in parts]).astype(np.int32))
    f["kind"] = np.array(kinds)
    f["scenario"] = f"{W}x{H}-{which}"
    return f


def skip_set(H_sub, Pn):
    """Patches whose 64 exported rows are all zero: the ones the pass did not read."""
    return ~np.any(np.asarray(H_sub).reshape(Pn, 64 * 6) != 0.0, axis=1)
