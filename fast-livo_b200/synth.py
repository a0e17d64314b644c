"""Deterministic synthetic frames for the FAST-LIVO hot path (SURVEY.md §8d).

One *frame* = everything the per-frame measurement assembly + iterated ESKF update
consumes: a point map (M x 3 float32), an already-downsampled scan in the LiDAR body
frame (N x 3 float32, the role of ``feats_down_body``, reference
src/laserMapping.cpp:1398-1399), a propagated prior (``state_propagat`` + 18x18
covariance, reference src/laserMapping.cpp:1292), a gray image (uint8, the ``cv::Mat``
handed to ``LidarSelector::detect``, reference src/lidar_selection.cpp:1027) and a
patch list (positions, 3-level 8x8 reference patches, search levels: the role of
``SubSparseMap``, reference include/common_lib.h:263-292).

numpy only; no dependency on the reference tree or on the oracle.  Everything is
seeded: the same (config, seed) gives bit-identical arrays on every machine.

Scene: an axis-aligned room with interior box obstacles.  Surfaces carry a
band-limited 3-D sinusoid texture, so the rendered image has smooth, non-zero
gradients everywhere (the photometric Jacobian needs them).
"""
from __future__ import annotations

import dataclasses
import numpy as np

# Reference parameter values (config/avia.yaml, config/camera_pinhole.yaml).
AVIA_EXTRINSIC_T = np.array([0.04165, 0.02326, -0.0284])            # avia.yaml:32
AVIA_EXTRINSIC_R = np.eye(3)                                          # avia.yaml:33-35
AVIA_RCL = np.array([[0.00162756, -0.999991, 0.00390957],            # avia.yaml:42-44
                     [-0.0126748, -0.00392989, -0.999912],
                     [0.999918, 0.00157786, -0.012681]])
AVIA_PCL = np.array([0.0409257, 0.0318424, -0.0927219])              # avia.yaml:45
PINHOLE = dict(width=640, height=512, fx=431.795259219, fy=431.550090267,
               cx=310.833037316, cy=266.985989326,
               d=(-0.0944205499243979, 0.0946727677776504, -0.00807970960613932,
                  8.07461209775283e-05, 0.0))                          # camera_pinhole.yaml:2-11


@dataclasses.dataclass
class FrameConfig:
    name: str
    n_scan: int
    n_map: int
    pitch: float              # filter_size_map: lattice pitch of the map
    img_w: int = 640
    img_h: int = 512
    n_patch: int = 2000
    lio_passes: int = 3       # K passes  => max_iteration = K-1 (SURVEY.md §8d)
    vio_passes: int = 3       # per level
    distortion: bool = False
    room_h: float = 8.0
    laser_point_cov: float = 0.001
    img_point_cov: float = 100.0
    seed: int = 20260922

    @property
    def cell_size(self) -> float:
        return 2.0 * self.pitch


# BASELINE.json configs (BASELINE.md "Configs -> concrete workloads").
CONFIGS = {
    "C1": FrameConfig("C1", n_scan=1000, n_map=20000, pitch=0.3, n_patch=0, lio_passes=1, vio_passes=0, seed=20260923),
    "C2": FrameConfig("C2", n_scan=24000, n_map=240000, pitch=0.3, n_patch=2000, lio_passes=3, vio_passes=3, seed=20260924),
    "C3": FrameConfig("C3", n_scan=100000, n_map=1000000, pitch=0.15, n_patch=5000, lio_passes=5, vio_passes=5, seed=20260925),
    "C4": FrameConfig("C4", n_scan=8000, n_map=80000, pitch=0.3, img_w=1280, img_h=1024, n_patch=10000,
                      lio_passes=3, vio_passes=3, seed=20260926),
    # small cases for fast parity tests
    "T0": FrameConfig("T0", n_scan=600, n_map=6000, pitch=0.3, img_w=320, img_h=256, n_patch=96,
                      lio_passes=3, vio_passes=3, seed=20260930),
    "T1": FrameConfig("T1", n_scan=3000, n_map=30000, pitch=0.3, n_patch=300, lio_passes=4, vio_passes=3,
                      distortion=True, seed=20260931),
}


# --------------------------------------------------------------------------- scene
class Scene:
    """Room [-L/2,L/2]^2 x [0,H] with axis-aligned interior boxes."""

    def __init__(self, rng: np.random.Generator, room_l: float, room_h: float, n_boxes: int = 8):
        self.L, self.H = float(room_l), float(room_h)
        self.room_lo = np.array([-room_l / 2, -room_l / 2, 0.0])
        self.room_hi = np.array([room_l / 2, room_l / 2, room_h])
        lo, hi = [], []
        for _ in range(n_boxes):
            size = rng.uniform([0.06 * room_l, 0.06 * room_l, 0.25 * room_h], [0.16 * room_l, 0.16 * room_l, 0.7 * room_h])
            # keep the centre region (sensor location) free
            while True:
                c = rng.uniform([-0.42 * room_l, -0.42 * room_l], [0.42 * room_l, 0.42 * room_l])
                if np.max(np.abs(c)) > 0.18 * room_l:
                    break
            lo.append([c[0] - size[0] / 2, c[1] - size[1] / 2, 0.0])
            hi.append([c[0] + size[0] / 2, c[1] + size[1] / 2, size[2]])
        self.box_lo = np.array(lo).reshape(-1, 3)
        self.box_hi = np.array(hi).reshape(-1, 3)
        # band-limited texture: sum of 64 3-D sinusoids, world periods 0.8..8 m
        k = 64
        dirs = rng.normal(size=(k, 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        period = np.exp(rng.uniform(np.log(0.8), np.log(8.0), size=k))
        self.tex_f = dirs / period[:, None]
        self.tex_phase = rng.uniform(0, 2 * np.pi, size=k)
        amp = rng.uniform(0.5, 1.0, size=k)
        self.tex_amp = amp * (40.0 / np.sqrt(0.5 * np.sum(amp ** 2)))   # std ~ 40 grey levels

    def rectangles(self):
        """(axis, value, lo2, hi2) for every surface (room faces + box faces)."""
        rects = []
        for ax in range(3):
            o = [a for a in range(3) if a != ax]
            for val in (self.room_lo[ax], self.room_hi[ax]):
                rects.append((ax, float(val), self.room_lo[o], self.room_hi[o]))
        for blo, bhi in zip(self.box_lo, self.box_hi):
            for ax in range(3):
                o = [a for a in range(3) if a != ax]
                for val in (blo[ax], bhi[ax]):
                    if ax == 2 and val == 0.0:
                        continue  # box bottoms coincide with the floor
                    rects.append((ax, float(val), blo[o], bhi[o]))
        return rects

    def area(self) -> float:
        return float(sum(np.prod(hi2 - lo2) for _, _, lo2, hi2 in self.rectangles()))

    def raycast(self, origin: np.ndarray, dirs: np.ndarray) -> np.ndarray:
        """Distance along each unit ray from `origin` (inside the room) to the first surface."""
        d = np.where(np.abs(dirs) < 1e-12, 1e-12, dirs)
        inv = 1.0 / d
        # leaving the room
        t_hi = (self.room_hi - origin) * inv
        t_lo = (self.room_lo - origin) * inv
        t = np.min(np.maximum(t_hi, t_lo), axis=1)
        # entering a box (slab method)
        for blo, bhi in zip(self.box_lo, self.box_hi):
            t1 = (blo - origin) * inv
            t2 = (bhi - origin) * inv
            tn = np.max(np.minimum(t1, t2), axis=1)
            tf = np.min(np.maximum(t1, t2), axis=1)
            hit = (tn > 1e-6) & (tn <= tf)
            t = np.where(hit & (tn < t), tn, t)
        return t

    def texture(self, pts: np.ndarray) -> np.ndarray:
        """Grey level (float, roughly 128 +- 40) of surface points, evaluated in chunks."""
        out = np.empty(len(pts))
        step = 1 << 16
        for s in range(0, len(pts), step):
            ph = 2 * np.pi * (pts[s:s + step] @ self.tex_f.T) + self.tex_phase
            out[s:s + step] = 128.0 + np.sin(ph) @ self.tex_amp
        return out


def _room_for(n_map: int, pitch: float, room_h: float) -> float:
    """Room side such that the surface lattice at `pitch` holds a little over n_map points."""
    area = 1.12 * n_map * pitch * pitch
    # 2 L^2 + 4 L H = area (boxes add a bit more)
    l = (-4 * room_h + np.sqrt(16 * room_h ** 2 + 8 * area)) / 4
    return max(float(l), 6.0)


def sample_map(rng: np.random.Generator, scene: Scene, pitch: float, n_map: int) -> np.ndarray:
    """Jittered lattice of pitch `pitch` on every surface (+-20 % in-plane jitter, sigma = 5 mm
    along the normal: no exact distance ties, SURVEY.md §7 H3), trimmed to exactly n_map points."""
    chunks = []
    for ax, val, lo2, hi2 in scene.rectangles():
        n0 = max(int(np.floor((hi2[0] - lo2[0]) / pitch)), 1)
        n1 = max(int(np.floor((hi2[1] - lo2[1]) / pitch)), 1)
        g0, g1 = np.meshgrid(lo2[0] + (np.arange(n0) + 0.5) * pitch, lo2[1] + (np.arange(n1) + 0.5) * pitch, indexing="ij")
        uv = np.stack([g0.ravel(), g1.ravel()], axis=1)
        uv += rng.uniform(-0.2 * pitch, 0.2 * pitch, size=uv.shape)
        nrm = val + rng.normal(0.0, 0.005, size=len(uv))
        p = np.empty((len(uv), 3))
        o = [a for a in range(3) if a != ax]
        p[:, ax] = nrm
        p[:, o[0]] = uv[:, 0]
        p[:, o[1]] = uv[:, 1]
        chunks.append(p)
    pts = np.concatenate(chunks)
    if len(pts) < n_map:
        raise ValueError(f"scene too small: {len(pts)} lattice points < n_map={n_map}")
    keep = np.sort(rng.choice(len(pts), size=n_map, replace=False))
    return pts[keep].astype(np.float32)


# --------------------------------------------------------------------------- math
def exp_so3(v: np.ndarray) -> np.ndarray:
    th = np.linalg.norm(v)
    if th < 1e-12:
        return np.eye(3)
    k = v / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _undistort_normalized(xd, yd, d, iters=12):
    """Invert vikit's radtan model (SURVEY.md Appendix C) by fixed-point iteration."""
    x, y = xd.copy(), yd.copy()
    for _ in range(iters):
        r2 = x * x + y * y
        cd = 1 + d[0] * r2 + d[1] * r2 * r2 + d[4] * r2 ** 3
        dx = d[2] * 2 * x * y + d[3] * (r2 + 2 * x * x)
        dy = d[2] * (r2 + 2 * y * y) + d[3] * 2 * x * y
        x = (xd - dx) / cd
        y = (yd - dy) / cd
    return x, y


def pixel_rays(cam: dict, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """Unit ray directions in the camera frame through pixel centres (u, v)."""
    xd = (u - cam["cx"]) / cam["fx"]
    yd = (v - cam["cy"]) / cam["fy"]
    if abs(cam["d"][0]) > 1e-7:
        x, y = _undistort_normalized(xd, yd, cam["d"])
    else:
        x, y = xd, yd
    r = np.stack([x, y, np.ones_like(x)], axis=-1)
    return r / np.linalg.norm(r, axis=-1, keepdims=True)


def bilinear_u8(img: np.ndarray, u: np.ndarray, v: np.ndarray) -> np.ndarray:
    """Plain bilinear sample of a uint8 image at float pixel coords (float32 arithmetic)."""
    u = u.astype(np.float32)
    v = v.astype(np.float32)
    x = np.floor(u).astype(np.int64)
    y = np.floor(v).astype(np.int64)
    su = (u - x).astype(np.float32)
    sv = (v - y).astype(np.float32)
    i00 = img[y, x].astype(np.float32)
    i01 = img[y, x + 1].astype(np.float32)
    i10 = img[y + 1, x].astype(np.float32)
    i11 = img[y + 1, x + 1].astype(np.float32)
    one = np.float32(1.0)
    return ((one - su) * (one - sv) * i00 + su * (one - sv) * i01 + (one - su) * sv * i10 + su * sv * i11).astype(np.float32)


# --------------------------------------------------------------------------- frame
def make_frame(cfg: FrameConfig | str, seed: int | None = None) -> dict:
    """Build one synthetic frame.  Returns a dict of numpy arrays + scalars."""
    if isinstance(cfg, str):
        cfg = CONFIGS[cfg]
    seed = cfg.seed if seed is None else seed
    rng = np.random.default_rng(np.random.PCG64(seed))

    room_l = _room_for(cfg.n_map, cfg.pitch, cfg.room_h)
    scene = Scene(rng, room_l, cfg.room_h)
    map_xyz = sample_map(rng, scene, cfg.pitch, cfg.n_map)

    # true pose T* (IMU frame in world)
    yaw = rng.uniform(-np.pi, np.pi)
    rp = rng.uniform(-np.deg2rad(3), np.deg2rad(3), size=2)
    R_true = exp_so3(np.array([0, 0, yaw])) @ exp_so3(np.array([rp[0], rp[1], 0]))
    p_true = np.array([rng.uniform(-0.06, 0.06) * room_l, rng.uniform(-0.06, 0.06) * room_l,
                       rng.uniform(1.2, 1.8)])
    R_LI, t_LI = AVIA_EXTRINSIC_R.copy(), AVIA_EXTRINSIC_T.copy()

    # scan: N rays in an Avia-like 70.4 x 77.2 deg FoV, sigma = 1 cm range noise
    az = rng.uniform(-np.deg2rad(35.2), np.deg2rad(35.2), size=cfg.n_scan)
    el = rng.uniform(-np.deg2rad(38.6), np.deg2rad(38.6), size=cfg.n_scan)
    d_l = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], axis=1)
    R_wl = R_true @ R_LI
    o_w = R_true @ t_LI + p_true
    rng_t = scene.raycast(o_w, d_l @ R_wl.T) + rng.normal(0.0, 0.01, size=cfg.n_scan)
    scan_body = (d_l * rng_t[:, None]).astype(np.float32)          # points in the LiDAR body frame

    # prior: x_prop = T* [+] delta0, P = diag(...)
    d_rot = rng.normal(0.0, np.deg2rad(0.5), size=3)
    d_pos = rng.normal(0.0, 0.03, size=3)
    R_prop = R_true @ exp_so3(d_rot)
    p_prop = p_true + d_pos
    cov = np.diag(np.repeat([1e-4, 1e-3, 1e-2, 1e-4, 1e-3, 1e-4], 3)).astype(np.float64)

    frame = dict(
        name=cfg.name, seed=seed, cfg=cfg,
        map_xyz=map_xyz, scan_body=scan_body,
        R_true=R_true, p_true=p_true, R_prop=R_prop, p_prop=p_prop, cov=cov,
        vel=np.zeros(3), bg=np.zeros(3), ba=np.zeros(3), grav=np.array([0.0, 0.0, -9.81]),
        R_LI=R_LI, t_LI=t_LI, Rcl=AVIA_RCL.copy(), Pcl=AVIA_PCL.copy(),
        room_l=room_l,
    )

    # ---- camera -------------------------------------------------------------
    sx = cfg.img_w / PINHOLE["width"]
    sy = cfg.img_h / PINHOLE["height"]
    cam = dict(width=cfg.img_w, height=cfg.img_h, fx=PINHOLE["fx"] * sx, fy=PINHOLE["fy"] * sy,
               cx=PINHOLE["cx"] * sx, cy=PINHOLE["cy"] * sy,
               d=tuple(PINHOLE["d"]) if cfg.distortion else (0.0, 0.0, 0.0, 0.0, 0.0))
    frame["cam"] = cam
    if cfg.n_patch == 0:
        frame.update(image=np.zeros((cfg.img_h, cfg.img_w), np.uint8),
                     patch_pos=np.zeros((0, 3)), patch_ref=np.zeros((0, 3, 64), np.float32),
                     patch_level=np.zeros(0, np.int32))
        return frame

    # camera pose at T*: p_c = Rci * R^T (p_w - p) + Pci   (lidar_selection.cpp:41-52, :780-781)
    Rli = R_LI.T
    Pli = -R_LI.T @ t_LI
    Rci = frame["Rcl"] @ Rli
    Pci = frame["Rcl"] @ Pli + frame["Pcl"]
    R_wc = R_true @ Rci.T                      # camera -> world rotation
    c_w = p_true - R_true @ (Rci.T @ Pci)      # camera centre in world

    vv, uu = np.meshgrid(np.arange(cfg.img_h, dtype=np.float64), np.arange(cfg.img_w, dtype=np.float64), indexing="ij")
    rays_c = pixel_rays(cam, uu.ravel(), vv.ravel())
    rays_w = rays_c @ R_wc.T
    t_px = scene.raycast(c_w, rays_w)
    clean = scene.texture(c_w + rays_w * t_px[:, None]).reshape(cfg.img_h, cfg.img_w)
    ref_img = np.clip(np.rint(clean), 0, 255).astype(np.uint8)                        # earlier observation
    image = np.clip(np.rint(clean + rng.normal(0.0, 2.0, size=clean.shape)), 0, 255).astype(np.uint8)

    # patches: visible surface points through random pixels >= 64 px from the border
    border = 64
    pu = rng.uniform(border, cfg.img_w - 1 - border, size=cfg.n_patch)
    pv = rng.uniform(border, cfg.img_h - 1 - border, size=cfg.n_patch)
    pr_w = pixel_rays(cam, pu, pv) @ R_wc.T
    pt = scene.raycast(c_w, pr_w)
    patch_pos = c_w + pr_w * pt[:, None]
    level = (rng.uniform(size=cfg.n_patch) < 0.1).astype(np.int32)       # search_level 0 (90 %) / 1 (10 %)
    # reference patch: warpAffine with A = I (lidar_selection.cpp:279-295):
    #   patch[64*pyr + 8*row + col] = bilinear(ref, px + (col-4, row-4) * (1<<search_level) * (1<<pyr))
    patch_ref = np.empty((cfg.n_patch, 3, 64), np.float32)
    rr, cc = np.meshgrid(np.arange(8) - 4, np.arange(8) - 4, indexing="ij")
    for pyr in range(3):
        s = (1 << level)[:, None, None] * (1 << pyr)
        su = pu[:, None, None] + cc[None] * s
        sv = pv[:, None, None] + rr[None] * s
        patch_ref[:, pyr, :] = bilinear_u8(ref_img, su.reshape(cfg.n_patch, 64), sv.reshape(cfg.n_patch, 64))
    frame.update(image=image, ref_image=ref_img, patch_pos=patch_pos.astype(np.float64),
                 patch_ref=patch_ref, patch_level=level, patch_px=np.stack([pu, pv], axis=1))
    return frame


# ---------------------------------------------------------------------------------------------------------
# IMU propagation / undistortion inputs (SURVEY.md section 8 row f3)
# ---------------------------------------------------------------------------------------------------------
def make_imu_frame(seed=1, n_points=24000, imu_hz=200.0, scan_s=0.1, variant="nominal"):
    """One LidarMeasureGroup worth of inputs for ImuProcess::UndistortPcl (reference src/IMU_Processing.cpp:611):
    v_imu (last_imu_ + meas.imu) as (K,7) [t, gyr xyz, acc xyz], time-ordered lidar points with their offset in ms,
    the incoming state and the ImuProcess members that carry over.  `variant` moves the time stamps into the
    corner cases of the reference's branches."""
    rng = np.random.default_rng(seed)
    t0 = 1000.0 + 0.1 * seed
    pcl_beg = t0
    pcl_end = t0 + scan_s
    dt_imu = 1.0 / imu_hz
    k = int(round(scan_s * imu_hz)) + 2
    times = t0 - 0.6 * dt_imu + dt_imu * np.arange(k)            # last_imu_ lies before the scan start
    last_end = t0                                                # last_lidar_end_time_
    if variant == "late_imu":            # IMU stops before the scan ends   -> note = +1 (:745)
        times = times[times < pcl_end - 2.5 * dt_imu]
    elif variant == "imu_past_end":      # IMU runs past the scan end        -> note = -1 (:745)
        times = np.concatenate([times, [times[-1] + dt_imu, times[-1] + 2 * dt_imu]])
    elif variant == "stale_imu":         # leading samples older than last_lidar_end_time_ -> `continue` (:671), dt rule (:690)
        times = np.concatenate([t0 - dt_imu * np.arange(4, 1, -1) - 0.6 * dt_imu, times])
    elif variant == "imu_before_scan":   # every sample before pcl_beg_time -> the else branch of :743
        times = t0 - dt_imu * np.arange(6, 0, -1) - 1e-4
        last_end = times[2] + 1e-5
    w = 0.4 * np.sin(2 * np.pi * 1.3 * (times - t0))[:, None] * np.array([0.3, -0.5, 1.0]) + rng.normal(0, 0.01, (len(times), 3))
    a = np.array([0.2, -0.1, 9.81]) + 0.8 * np.cos(2 * np.pi * 0.9 * (times - t0))[:, None] * np.array([1.0, 0.4, -0.2]) \
        + rng.normal(0, 0.05, (len(times), 3))
    v_imu = np.concatenate([times[:, None], w, a], 1)
    off = np.sort(rng.uniform(0.0, scan_s * 1000.0, n_points)).astype(np.float32)
    if variant == "unsorted_points" and n_points > 64:   # local disorder + a late first point (the :807 quirk)
        idx = rng.integers(1, n_points - 1, n_points // 50)
        off[idx] = off[np.clip(idx + rng.integers(-40, 40, len(idx)), 0, n_points - 1)]
        off[0] = np.float32(3.7 * dt_imu * 1000.0)
    if variant == "early_points" and n_points > 64:      # offsets <= 0: the walk ends, those points stay (:790)
        off[:37] = np.float32(0.0)
        off[:5] = np.float32(-1.5)
    rng2 = np.random.default_rng(seed + 77)
    d = rng2.uniform(1.0, 60.0, n_points)
    az = rng2.uniform(-0.6, 0.6, n_points)
    el = rng2.uniform(-0.6, 0.6, n_points)
    pts = np.stack([d * np.cos(el) * np.cos(az), d * np.cos(el) * np.sin(az), d * np.sin(el)], 1).astype(np.float32)
    ax = rng.normal(size=3); ax /= np.linalg.norm(ax)
    R0 = exp_so3(ax * 0.3)
    cov = np.diag(np.concatenate([np.full(3, 1e-4), np.full(3, 1e-3), np.full(3, 1e-2), np.full(3, 1e-5), np.full(3, 1e-4), np.full(3, 1e-6)]))
    m = rng.normal(0, 1e-4, (18, 18))
    cov = cov + m @ m.T
    return dict(v_imu=v_imu, pcl_beg_time=pcl_beg, pcl_end_time=pcl_end, last_lidar_end_time=last_end,
                pts=pts, offset_ms=off, R=R0, p=np.array([1.5, -0.7, 0.3]), vel=np.array([0.8, -0.3, 0.05]),
                bg=np.array([0.002, -0.001, 0.0015]), ba=np.array([0.03, -0.02, 0.01]), grav=np.array([0.0, 0.0, -9.81]),
                cov=cov, acc_s_last=np.array([0.1, 0.05, -0.02]), angvel_last=np.array([0.01, -0.02, 0.03]),
                cov_gyr=np.array([0.1, 0.1, 0.1]), cov_acc=np.array([0.1, 0.1, 0.1]),
                cov_bias_gyr=np.array([1e-4, 1e-4, 1e-4]), cov_bias_acc=np.array([1e-4, 1e-4, 1e-4]),
                G_m_s2=9.81, mean_acc_norm=9.79,
                R_LI=exp_so3(np.array([0.01, -0.02, 0.015])), t_LI=np.array([0.04165, 0.02326, -0.0284]))


# ---------------------------------------------------------------------------------------------------------
# Raw driver messages (Preprocess::process, reference src/preprocess.cpp): flb_lidar_upload's input
# ---------------------------------------------------------------------------------------------------------
LIVOX_POINT = np.dtype([("offset_time", "<u4"), ("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("reflectivity", "u1"),
                        ("tag", "u1"), ("line", "u1"), ("pad", "u1")])                    # livox_ros_driver::CustomPoint, 20 bytes
OUSTER_POINT = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                         "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "u1", "<u2", "<u4"],
                         "offsets": [0, 4, 8, 16, 20, 24, 26, 28, 32], "itemsize": 48})    # ouster_ros::Point with its padding
VELODYNE_POINT = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"],
                           "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                           "offsets": [0, 4, 8, 12, 16, 20], "itemsize": 24})
XT32_POINT = np.dtype({"names": ["x", "y", "z", "intensity", "timestamp", "ring"],
                       "formats": ["<f4", "<f4", "<f4", "<f4", "<f8", "<u2"],
                       "offsets": [0, 4, 8, 12, 16, 24], "itemsize": 32})
LIDAR_KINDS = {"livox": 1, "velodyne": 2, "velodyne_notime": 2, "ouster": 3, "xt32": 4}      # FLB_LIDAR_*


def make_lidar_message(kind, seed=1, n=24000, point_filter_num=None, unsorted=None):
    """One driver message as (records, fmt): the raw records as bytes and a dict of flb_lidar_format's fields.
    kind: "livox" (six lines fired together, so times tie; tags over all four `& 0x30` values with other bits set; lines
    >= n_scans; runs of repeated points; (0, 0, 0) no-return points; points inside blind; a repeated point right after a
    record that is not taken), "ouster" (column order with staggered t, 48-byte records with padding), "velodyne",
    "velodyne_notime" (every time 0), "xt32" (f64 timestamp).  unsorted: shuffle the firing times (default: only the
    Ouster's stagger); point_filter_num: default 1 for Livox, 3 otherwise."""
    rng = np.random.default_rng(1000 * LIDAR_KINDS[kind] + seed)
    blind = {"livox": 0.5, "ouster": 0.8, "velodyne": 1.0, "velodyne_notime": 1.0, "xt32": 0.64}[kind]
    d = rng.uniform(1.2, 60.0, n)
    near = rng.random(n) < 0.03
    d[near] = rng.uniform(0.05, 0.95 * blind if kind != "xt32" else 0.75, near.sum())     # inside blind (XT32: blind is unsquared)
    az, el = rng.uniform(-np.pi, np.pi, n), rng.uniform(-0.4, 0.4, n)
    xyz = np.stack([d * np.cos(el) * np.cos(az), d * np.cos(el) * np.sin(az), d * np.sin(el)], 1).astype(np.float32)
    xyz[rng.random(n) < 0.03] = 0.0                                                      # no return
    rep = np.flatnonzero(rng.random(n) < 0.04)
    for i in rep[rep > 0]:                                                               # runs of repeated points
        xyz[i] = xyz[i - 1]
    idx = np.arange(n)
    if kind == "livox":
        a = np.zeros(n, LIVOX_POINT)
        group = idx // 6
        if unsorted:
            group = rng.permutation(max(int(group.max(initial=0)) + 1, 1))[group] if n else group
        a["offset_time"] = (group.astype(np.int64) * 25000 + 7).astype(np.uint32)         # ns; the six lines share a time
        a["line"] = idx % 6
        bad_line = rng.random(n) < 0.02
        a["line"][bad_line] = rng.integers(6, 9, bad_line.sum())
        tag = rng.choice(np.array([0x00, 0x10, 0x20, 0x30], np.uint8), n, p=[0.45, 0.4, 0.1, 0.05])
        a["tag"] = tag | (rng.integers(0, 256, n).astype(np.uint8) & 0xCF)
        a["reflectivity"] = rng.integers(0, 256, n)
        for j in range(40, n - 1, 997):          # a repeated point right after a record that is not taken: compared with zero
            xyz[j] = xyz[j - 1] = np.float32([3.0 + 0.001 * j, -2.0, 0.5])
            a["tag"][j - 1] = 0x20 | 0x03
            a["tag"][j] = 0x10 | 0x40
            a["line"][j] = 2
        fmt = dict(off_time=0, off_x=4, off_y=8, off_z=12, off_tag=17, off_line=18, n_scans=6,
                   point_filter_num=point_filter_num or 1)
    elif kind == "ouster":
        a = np.zeros(n, OUSTER_POINT)
        col, ring = idx // 64, idx % 64
        if unsorted is False:
            a["t"] = idx * 763
        else:
            a["t"] = col * 48828 + (3 - ring % 4) * 30000                                # staggered: not sorted in record order
        a["ring"] = ring
        a["intensity"] = rng.uniform(0, 255, n)
        a.view(np.uint8).reshape(n, 48)[:, 12:16] = 0xAB                                 # padding is not zero
        a.view(np.uint8).reshape(n, 48)[:, 36:48] = 0xCD
        fmt = dict(off_x=0, off_y=4, off_z=8, off_time=20, off_tag=0, off_line=0, n_scans=64,
                   point_filter_num=point_filter_num or 3)
    elif kind in ("velodyne", "velodyne_notime"):
        a = np.zeros(n, VELODYNE_POINT)
        a["ring"] = idx % 16
        if kind == "velodyne":
            t = (idx // 16) * 55.296e-6 + (idx % 16) * 2.304e-6 + 1e-6                    # seconds from the scan start
            a["time"] = rng.permutation(t) if unsorted else t
        fmt = dict(off_x=0, off_y=4, off_z=8, off_time=20, off_tag=0, off_line=0, n_scans=16,
                   point_filter_num=point_filter_num or 3)
    else:
        a = np.zeros(n, XT32_POINT)
        t = 1.7e9 + 0.25 * seed + (idx // 32) * 55.56e-6 + (idx % 32) * 1.5e-6
        a["timestamp"] = rng.permutation(t) if unsorted else t
        a["ring"] = idx % 32
        fmt = dict(off_x=0, off_y=4, off_z=8, off_time=16, off_tag=0, off_line=0, n_scans=32,
                   point_filter_num=point_filter_num or 3)
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    fmt.update(kind=LIDAR_KINDS[kind], point_step=a.dtype.itemsize, blind=blind)
    return a.tobytes(), fmt


# Velodyne PointCloud2 layouts (flb_lidar_upload_velodyne's input): XYZIRT (velodyne_pointcloud with times), a packed
# 22-byte XYZIRT with the float time at 18, and a 32-byte XYZIR (pcl::PointXYZIR's padded layout) without a time field.
VELODYNE_LAYOUTS = {
    "xyzirt": (np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                         "offsets": [0, 4, 8, 12, 16, 20], "itemsize": 24}), 20),
    "packed22": (np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                           "offsets": [0, 4, 8, 12, 16, 18], "itemsize": 22}), 18),
    "xyzir32": (np.dtype({"names": ["x", "y", "z", "intensity", "ring"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2"],
                          "offsets": [0, 4, 8, 16, 20], "itemsize": 32}), -1),
}


def make_velodyne_spin(layout="xyzirt", seed=1, n_scans=16, n_cols=1800, point_filter_num=1, timed=False, blind=1.0):
    """One spin of a rotating Velodyne as (records, fmt): the raw PointCloud2 data and a dict of flb_velodyne_format's
    fields.  Column by column, the rings fire in an interleaved order; the yaw turns clockwise from a random start through
    a little over 360 degrees, so it crosses +-180 and each ring's time_last wraps near the end; azimuth jitter makes some
    later records turn back, which the reference's walk takes for a spurious wrap.  Also: NaN no-return records (never a
    ring's first record, which would make the whole ring's times NaN), -0.0 coordinates (atan2 gives +-pi), points inside
    blind, an empty ring (ring 1 never fires) and a one-record ring (ring n_scans - 1 fires once).  layout: a key of
    VELODYNE_LAYOUTS.  timed: per-point times in seconds (a layout without a time field ignores it); otherwise every time
    is 0 and the times come from the yaw."""
    dt, off_time = VELODYNE_LAYOUTS[layout]
    rng = np.random.default_rng(7919 * seed + n_scans)
    order = np.concatenate([np.arange(0, n_scans, 2), np.arange(1, n_scans, 2)])          # interleaved firing order
    order = order[order != 1]                                                            # the empty ring
    lone = n_scans - 1
    ring = np.tile(order, n_cols)
    col = np.repeat(np.arange(n_cols), len(order))
    keep = (ring != lone) | (col == n_cols // 3)                                         # the one-record ring
    ring, col = ring[keep], col[keep]
    n = len(ring)
    pos = np.zeros(n_scans, np.int64)
    pos[order] = np.arange(len(order))
    slot = pos[ring]                                                                     # position in the firing order
    spin = 360.0 + rng.uniform(2.0, 8.0)                                                 # a little over one turn
    az = rng.uniform(-180.0, 180.0) - spin * (col + slot / len(order)) / n_cols          # clockwise
    az += rng.normal(0.0, 0.1, n)                                                        # azimuth jitter
    el = np.deg2rad(-15.0 + 30.0 * ring / max(n_scans - 1, 1))
    d = rng.uniform(1.2, 60.0, n)
    near = rng.random(n) < 0.03
    d[near] = rng.uniform(0.05, 0.95 * blind, near.sum())
    a_rad = np.deg2rad(az)
    xyz = np.stack([d * np.cos(el) * np.cos(a_rad), d * np.cos(el) * np.sin(a_rad), d * np.sin(el)], 1).astype(np.float32)
    first = np.zeros(n, bool)
    first[np.unique(ring, return_index=True)[1]] = True
    nan = (rng.random(n) < 0.03) & ~first
    xyz[nan] = np.nan
    neg = np.flatnonzero(~first & ~nan)
    z0 = rng.choice(neg, min(len(neg), 24), replace=False)
    xyz[z0[:8], 1] = -0.0                                                                # y = -0.0: atan2 gives -pi or -0
    xyz[z0[8:16], 0] = -0.0                                                              # x = -0.0: +-pi/2
    xyz[z0[16:], :2] = np.float32([-0.0, -0.0]) * rng.choice([1, -1], (len(z0[16:]), 2))   # both zero: +-0 or +-pi
    a = np.zeros(n, dt)
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    a["intensity"] = rng.uniform(0, 255, n)
    a["ring"] = ring
    if off_time >= 0 and timed:
        a["time"] = col * 55.296e-6 + slot * 2.304e-6 + 1e-6
    fmt = dict(point_step=dt.itemsize, off_x=0, off_y=4, off_z=8, off_time=off_time, off_ring=dt.fields["ring"][1], n_scans=n_scans,
               point_filter_num=point_filter_num, blind=blind)
    return a.tobytes(), fmt


def _feature_scene_range(az, el):
    """Ray-cast distance from the origin along (az, el) into a structured scene: the ground, two walls meeting at a
    right angle, a wall at a shallow angle, a pole, a thin wire and a plate that occludes the walls (range jumps).
    inf where nothing is hit within 60 m."""
    dx, dy, dz = np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)
    best = np.full(az.shape, np.inf)

    def take(t, ok):
        ok = ok & (t > 0) & (t < best)
        best[ok] = t[ok]

    with np.errstate(divide="ignore", invalid="ignore"):
        t = -1.6 / dz                                                       # ground z = -1.6
        take(t, dz < 0)
        t = 6.0 / dx                                                        # wall x = 6, y in [-8, 5]
        take(t, (dx > 0) & (np.abs(dy * t + 1.5) <= 6.5) & (dz * t < 3))
        t = 5.0 / dy                                                        # wall y = 5, x in [-3, 6]: the right-angle corner
        take(t, (dy > 0) & (dx * t >= -3) & (dx * t <= 6) & (dz * t < 3))
        nx, ny = -np.cos(np.deg2rad(8.0)), np.sin(np.deg2rad(8.0))          # shallow wall behind: n . p = 7
        t = 7.0 / (nx * dx + ny * dy)
        take(t, (nx * dx + ny * dy > 0) & (dz * t < 3))
        t = 2.5 / dx                                                        # occluding plate x = 2.5, y in [1.0, 1.6]
        take(t, (dx > 0) & (dy * t >= 1.0) & (dy * t <= 1.6) & (dz * t < 0.8))
        cx, cy, r = 3.0, -2.0, 0.08                                          # a pole
        b = dx * cx + dy * cy
        h2 = dx * dx + dy * dy
        disc = b * b - h2 * (cx * cx + cy * cy - r * r)
        t = (b - np.sqrt(np.maximum(disc, 0))) / h2
        take(t, disc >= 0)
        take(1.2 / dz,                                                      # a wire along x at y = -1, z = 1.2
             (dz > 0) & (np.abs(dy * 1.2 / dz + 1.0) < 0.02))
    best[best > 60.0] = np.inf
    return best


def make_feature_scan(kind, seed=1, n_scans=None, n_cols=None, point_filter_num=1, timed=True, blind=None, nan_returns=True):
    """One structured message for the feature branches (flb_lidar_upload_features, flb_lidar_upload_velodyne_features)
    as (records, fmt).  The sensor scans a scene of ground, walls at right and shallow angles, a pole, a wire and an
    occluding plate line by line, so planes, edges and range jumps all occur; also runs of points inside blind, empty,
    one-point and five-point lines, lines that end on a wall, and records the input filters drop.
    kind: "livox" (6 lines fired in turn, repeated coordinates, tags, lines >= n_scans), "ouster" (u8 ring at 26,
    zeros for no return, records with ring >= n_scans), "velodyne" (NaN for no return; `timed` False: no times, so they
    come from the yaw; `nan_returns` False: a ray that hits nothing returns from 59 m instead of NaN, as NaN points
    in pl_surf make the upload refuse the cloud).  fmt: flb_lidar_format's fields, with off_line the ring (Velodyne: flb_velodyne_format's)."""
    rng = np.random.default_rng(4099 * seed + LIDAR_KINDS[kind])
    if kind == "livox":
        n_scans = n_scans or 6
        n_cols = n_cols or 400
        blind = 0.5 if blind is None else blind
        col = np.repeat(np.arange(n_cols), n_scans)
        line = np.tile(np.arange(n_scans), n_cols)
        az = np.deg2rad(-35.0 + 70.0 * col / n_cols + 3.0 * np.sin(col / 37.0 + line)) + rng.normal(0, 2e-4, col.size)
        el = np.deg2rad(-12.0 + 4.0 * line + 6.0 * np.sin(col / 53.0 + 0.7 * line))
    else:
        n_scans = n_scans or (64 if kind == "ouster" else 16)
        n_cols = n_cols or (256 if kind == "ouster" else 450)
        blind = (0.8 if kind == "ouster" else 1.0) if blind is None else blind
        col = np.repeat(np.arange(n_cols), n_scans)
        line = np.tile(np.arange(n_scans), n_cols)
        az = np.pi - 2 * np.pi * (col + 0.5) / n_cols + rng.normal(0, 2e-4, col.size)
        el = np.deg2rad(-22.0 + 40.0 * line / max(n_scans - 1, 1))
    d = _feature_scene_range(az, el)
    d += rng.normal(0, 0.004, d.size) * np.isfinite(d)
    n = d.size
    near = (col % 97 < 6) & (line % 3 == 0)                                 # runs of points inside blind
    d[near] = 0.3 * blind + 0.02 * (col[near] % 97)
    miss = ~np.isfinite(d)
    if kind == "velodyne" and not nan_returns:
        d[miss] = 59.0
        miss[:] = False
    xyz = np.stack([d * np.cos(el) * np.cos(az), d * np.cos(el) * np.sin(az), d * np.sin(el)], 1).astype(np.float32)
    xyz[miss] = np.nan if kind == "velodyne" else 0.0
    ring = line.copy()
    sparse = [n_scans - 1, n_scans - 2, n_scans - 3] if n_scans >= 6 else []
    keep = np.ones(n, bool)
    for r, cnt in zip(sparse, (0, 1, 5)):                                   # empty, one-point and five-point lines
        idx = np.flatnonzero(ring == r)
        keep[idx[cnt:]] = False
    if kind != "livox" and n_scans >= 8:
        idx = np.flatnonzero(ring == n_scans - 4)                           # 14 points 2 cm apart on a wall: the plane
        keep[idx[14:]] = False                                              # group from the head reaches the line's end
        dense = np.stack([np.full(14, 6.0), 0.3 + 0.02 * np.arange(14), np.full(14, 0.4)], 1)
        xyz[idx[:14]] = dense + rng.normal(0, 1e-4, (14, 3))
    if kind == "velodyne" and n_scans >= 8:
        idx = np.flatnonzero(ring == n_scans - 5)                           # a line entirely within blind
        xyz[idx] *= np.float32(0.3 * blind) / np.maximum(np.linalg.norm(xyz[idx], axis=1, keepdims=True), 1e-6)
    if kind == "livox":
        keep[:] = True
        keep[np.flatnonzero(ring == n_scans - 1)[5:]] = False               # a five-point line
    xyz, ring, col = xyz[keep], ring[keep], col[keep]
    n = len(ring)
    if kind == "livox":
        a = np.zeros(n, LIVOX_POINT)
        a["offset_time"] = (np.arange(n, dtype=np.int64) * 4167 + 3).astype(np.uint32)
        rep = np.flatnonzero(rng.random(n) < 0.02)
        for i in rep[rep > 0]:                                              # repeated coordinates: all three, or one
            if rng.random() < 0.5:
                xyz[i] = xyz[i - 1]
            else:
                xyz[i, 2] = xyz[i - 1, 2]
        a["line"] = ring
        over = rng.random(n) < 0.01
        a["line"][over] = rng.integers(n_scans, n_scans + 3, over.sum())
        tag = rng.choice(np.array([0x10, 0x00, 0x20, 0x30], np.uint8), n, p=[0.93, 0.03, 0.02, 0.02])
        a["tag"] = tag | (rng.integers(0, 256, n).astype(np.uint8) & 0xC0)
        fmt = dict(kind=1, off_time=0, off_x=4, off_y=8, off_z=12, off_tag=17, off_line=18)
    elif kind == "ouster":
        a = np.zeros(n, OUSTER_POINT)
        a["t"] = col * 97656 + ring * 50
        a["ring"] = ring
        over = rng.random(n) < 0.005
        a["ring"][over] = n_scans
        fmt = dict(kind=3, off_x=0, off_y=4, off_z=8, off_time=20, off_tag=0, off_line=26)
    else:
        a = np.zeros(n, VELODYNE_POINT)
        a["ring"] = ring
        over = rng.random(n) < 0.005
        a["ring"][over] = n_scans + 1
        if timed:
            a["time"] = col * 55.296e-6 + ring * 2.304e-6 + 1e-6
        fmt = dict(kind=2, off_x=0, off_y=4, off_z=8, off_time=20, off_tag=0, off_line=16)
    a["x"], a["y"], a["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    fmt.update(point_step=a.dtype.itemsize, n_scans=n_scans, point_filter_num=point_filter_num, blind=blind)
    return a.tobytes(), fmt


# ---------------------------------------------------------------------------------------------------------
# Camera messages (flb_image_upload_msg): the synthetic texture as a driver in another encoding would send it
# ---------------------------------------------------------------------------------------------------------
BAYER_TILES = {"bayer_rggb8": "RGGB", "bayer_bggr8": "BGGR", "bayer_gbrg8": "GBRG", "bayer_grbg8": "GRBG"}


def texture_bgr(image: np.ndarray, width: int, height: int) -> np.ndarray:
    """A width x height BGR8 frame of a gray texture: three distinct channels, the texture repeated to cover the size
    (twice the camera's, give or take one pixel, is what a full-resolution camera sends)."""
    bgr = np.stack([image, np.roll(image, 3, 1), 255 - image], -1)
    reps = (-(-height // bgr.shape[0]), -(-width // bgr.shape[1]), 1)
    return np.ascontiguousarray(np.tile(bgr, reps)[:height, :width])


def mono_message(bgr: np.ndarray) -> np.ndarray:
    """A mono8 camera's frame of the same scene: the green channel, (h, w) uint8."""
    return np.ascontiguousarray(bgr[..., 1])


def bayer_message(bgr: np.ndarray, encoding: str = "bayer_rggb8") -> np.ndarray:
    """The (h, w) uint8 mosaic a camera with that colour-filter tile records of a BGR frame: each site keeps the
    channel of its filter colour; the tile is named from its top-left site (ROS image_encodings)."""
    tile = BAYER_TILES[encoding]
    m = np.empty(bgr.shape[:2], np.uint8)
    for k, c in enumerate(tile):
        m[k // 2::2, k % 2::2] = bgr[k // 2::2, k % 2::2, "BGR".index(c)]
    return m


# ---------------------------------------------------------------------------------------------------------
# Visual-map sequences (SURVEY.md section 8 rows f2 / f4): several frames of ONE scene along a short trajectory
# ---------------------------------------------------------------------------------------------------------
def voxel_centroids(xyz: np.ndarray, leaf: float) -> np.ndarray:
    """Stand-in for the caller's pcl::VoxelGrid (centroid per leaf-sized voxel), float32 in / out.  The selection
    takes the filtered cloud as an INPUT, so any deterministic filter serves the tests."""
    key = np.floor(xyz.astype(np.float64) / leaf).astype(np.int64)
    _, inv = np.unique(key, axis=0, return_inverse=True)
    inv = inv.ravel()
    n = inv.max() + 1
    out = np.zeros((n, 3))
    cnt = np.bincount(inv, minlength=n).astype(np.float64)
    for a in range(3):
        out[:, a] = np.bincount(inv, weights=xyz[:, a].astype(np.float64), minlength=n) / cnt
    return out.astype(np.float32)


def make_visual_sequence(cfg: FrameConfig | str = "T0", n_frames: int = 3, seed: int | None = None, step=(0.18, 0.06, 0.02),
                         yaw_step_deg: float = 2.5, with_map: bool = False) -> dict:
    """n_frames camera frames of one scene: image, camera pose T_f_w = (Rcw, Pcw) as LidarSelector::updateFrameState
    forms it (src/lidar_selection.cpp:905-911), the scan in WORLD coordinates (`pg` of LidarSelector::detect) and its
    0.2 m voxel-filtered version (`pg_down`, :7, :351-352)."""
    if isinstance(cfg, str):
        cfg = CONFIGS[cfg]
    seed = cfg.seed if seed is None else seed
    rng = np.random.default_rng(np.random.PCG64(seed + 77))
    room_l = _room_for(cfg.n_map, cfg.pitch, cfg.room_h)
    scene = Scene(rng, room_l, cfg.room_h)
    map_xyz = sample_map(np.random.default_rng(np.random.PCG64(seed + 78)), scene, cfg.pitch, cfg.n_map) if with_map else None
    yaw0 = rng.uniform(-np.pi, np.pi)
    p0 = np.array([rng.uniform(-0.04, 0.04) * room_l, rng.uniform(-0.04, 0.04) * room_l, rng.uniform(1.2, 1.8)])
    R_LI, t_LI = AVIA_EXTRINSIC_R.copy(), AVIA_EXTRINSIC_T.copy()
    sx, sy = cfg.img_w / PINHOLE["width"], cfg.img_h / PINHOLE["height"]
    cam = dict(width=cfg.img_w, height=cfg.img_h, fx=PINHOLE["fx"] * sx, fy=PINHOLE["fy"] * sy, cx=PINHOLE["cx"] * sx,
               cy=PINHOLE["cy"] * sy, d=tuple(PINHOLE["d"]) if cfg.distortion else (0.0, 0.0, 0.0, 0.0, 0.0))
    Rli, Pli = R_LI.T, -R_LI.T @ t_LI
    Rci = AVIA_RCL @ Rli
    Pci = AVIA_RCL @ Pli + AVIA_PCL
    vv, uu = np.meshgrid(np.arange(cfg.img_h, dtype=np.float64), np.arange(cfg.img_w, dtype=np.float64), indexing="ij")
    rays_c = pixel_rays(cam, uu.ravel(), vv.ravel())
    frames = []
    for k in range(n_frames):
        R = exp_so3(np.array([0, 0, yaw0 + np.deg2rad(yaw_step_deg) * k])) @ exp_so3(np.array([0.01 * k, -0.006 * k, 0]))
        fwd = R[:, 0]
        p = p0 + k * (step[0] * fwd + step[1] * R[:, 1] + np.array([0, 0, step[2]]))
        Rcw = Rci @ R.T
        Pcw = -Rci @ R.T @ p + Pci
        R_wc = Rcw.T
        c_w = -Rcw.T @ Pcw
        t_px = scene.raycast(c_w, rays_c @ R_wc.T)
        clean = scene.texture(c_w + (rays_c @ R_wc.T) * t_px[:, None]).reshape(cfg.img_h, cfg.img_w)
        image = np.clip(np.rint(clean + rng.normal(0.0, 2.0, size=clean.shape)), 0, 255).astype(np.uint8)
        az = rng.uniform(-np.deg2rad(35.2), np.deg2rad(35.2), size=cfg.n_scan)
        el = rng.uniform(-np.deg2rad(38.6), np.deg2rad(38.6), size=cfg.n_scan)
        d_l = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], axis=1)
        o_w = R @ t_LI + p
        d_w = d_l @ (R @ R_LI).T
        rng_t = scene.raycast(o_w, d_w) + rng.normal(0.0, 0.01, size=cfg.n_scan)
        pg = (o_w + d_w * rng_t[:, None]).astype(np.float32)
        prng = np.random.default_rng(np.random.PCG64(seed + 1000 + k))
        frames.append(dict(image=image, Rcw=Rcw, Pcw=Pcw, R=R, p=p, pg=pg, pg_down=voxel_centroids(pg, 0.2), frame_id=k,
                           scan_body=(d_l * rng_t[:, None]).astype(np.float32),
                           R_prop=R @ exp_so3(prng.normal(0.0, np.deg2rad(0.5), size=3)), p_prop=p + prng.normal(0.0, 0.03, size=3)))
    return dict(cfg=cfg, cam=cam, frames=frames, Rci=Rci, Pci=Pci, R_LI=R_LI, t_LI=t_LI, Rcl=AVIA_RCL.copy(), Pcl=AVIA_PCL.copy(),
                map_xyz=map_xyz, cov=np.diag(np.repeat([1e-4, 1e-3, 1e-2, 1e-4, 1e-3, 1e-4], 3)).astype(np.float64),
                grav=np.array([0.0, 0.0, -9.81]))
