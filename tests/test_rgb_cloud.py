"""CPU tier: publish_frame_world_rgb's laserCloudWorldRGB as records (flb_rgb_cloud) and the run's pcl_wait_save
(flb_rgb_save_*) from the rules the device applies, compiled for the host (tests/hostemu/rgb_cloud.cpp): the keep
flag and colour word per world point, the exclusive sum, the scatter into 32-byte pcl::PointXYZRGB records and into a
chunked save, and the save's expansion back to records.  The records must be byte-identical to the oracle's colorize
compacted and packed in numpy, over seeded T0- and C2-sized world clouds that include points behind the camera,
outside the image, in the (-1, 0) border band and on the last row and column; save slices that cross chunk boundaries
must expand to the same records."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

RGB_POINT = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("w", "<f4"), ("b", "u1"), ("g", "u1"), ("r", "u1"), ("a", "u1"),
                      ("pad", "u1", 12)])


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostemu", "rgb_cloud.cpp")
    so = str(tmp_path_factory.mktemp("rgb_emu") / "librgb_cloud.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, src])
    L = C.CDLL(so)
    L.emu_save_new.restype = C.c_void_p
    L.emu_save_free.argtypes = [C.c_void_p]
    L.emu_save_size.argtypes = [C.c_void_p]
    L.emu_save_size.restype = C.c_longlong
    L.emu_rgb_cloud.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_void_p]
    L.emu_save_download.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p]
    return L


def camv(cam):
    return np.array([cam["width"], cam["height"], cam["fx"], cam["fy"], cam["cx"], cam["cy"], *cam["d"]], np.float64)


def bgr_of(img, k):
    rng = np.random.default_rng(10 + k)
    return np.ascontiguousarray(np.stack([img, np.roll(img, 3, 1), 255 - img], -1) ^ rng.integers(0, 8, img.shape + (3,), dtype=np.uint8))


def pack_records(xyz, rgb):
    """numpy's pcl::PointXYZRGB records of the kept points: x y z, data[3] = 1, b g r, a = 255, zero padding."""
    out = np.zeros(len(xyz), RGB_POINT)
    out["x"], out["y"], out["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    out["w"] = 1.0
    out["r"], out["g"], out["b"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
    out["a"] = 255
    return out


def oracle_records(po, cam, Rcw, Pcw, bgr, xyz):
    rgb, val = po.colorize(cam, Rcw, Pcw, bgr, xyz)
    return pack_records(xyz[val], rgb[val])


def emu_cloud(L, cam, Rcw, Pcw, bgr, xyz, save=None):
    xyz = np.ascontiguousarray(xyz, np.float32)
    out = np.zeros(len(xyz), RGB_POINT)
    f64 = lambda a: np.ascontiguousarray(a, np.float64)
    m = L.emu_rgb_cloud(_p(camv(cam)), _p(f64(Rcw)), _p(f64(Pcw)), _p(np.ascontiguousarray(bgr)), _p(xyz), len(xyz), _p(out), save)
    return out[:m]


def edge_points(rng, cam, Rcw, Pcw, k):
    """World points (pinhole inverse; no distortion) at chosen pixels and depths: behind the camera, outside the image,
    in the (-1, 0) band of either axis, and on the last row and column."""
    W, H = cam["width"], cam["height"]
    u = np.concatenate([rng.uniform(0, W, k), rng.uniform(-40, -1.5, k), rng.uniform(W + 0.5, W + 40, k),
                        rng.uniform(-0.999, -0.001, k), rng.uniform(0, W, k), rng.uniform(W - 1, W - 1e-3, k), rng.uniform(0, W, k)])
    v = np.concatenate([rng.uniform(0, H, k), rng.uniform(0, H, k), rng.uniform(0, H, k),
                        rng.uniform(0, H, k), rng.uniform(-0.999, -0.001, k), rng.uniform(0, H, k), rng.uniform(H - 1, H - 1e-3, k)])
    d = rng.uniform(0.5, 20.0, len(u))
    d[:k] = -d[:k]                                                   # behind the camera
    pc = np.stack([(u - cam["cx"]) / cam["fx"] * d, (v - cam["cy"]) / cam["fy"] * d, d], 1)
    return ((pc - Pcw) @ Rcw).astype(np.float32)                     # Rcw^T (pc - Pcw), row by row


def world_cloud(flb, name, seed):
    seq = flb.synth.make_visual_sequence(name, 1)
    fr = seq["frames"][0]
    rng = np.random.default_rng(seed)
    assert not any(seq["cam"]["d"])
    xyz = np.concatenate([fr["pg"], edge_points(rng, seq["cam"], fr["Rcw"], fr["Pcw"], 40)])
    xyz = xyz[rng.permutation(len(xyz))]
    return seq["cam"], fr["Rcw"], fr["Pcw"], bgr_of(fr["image"], seed), np.ascontiguousarray(xyz, np.float32)


@pytest.mark.parametrize("name", ["T0", "C2"])
def test_records_equal_oracle(flb, po, emu, name):
    cam, Rcw, Pcw, bgr, xyz = world_cloud(flb, name, 3)
    W, H = cam["width"], cam["height"]
    got = emu_cloud(emu, cam, Rcw, Pcw, bgr, xyz)
    ref = oracle_records(po, cam, Rcw, Pcw, bgr, xyz)
    assert len(got) == len(ref) and got.tobytes() == ref.tobytes()
    # the cloud really holds every case: kept points in the band and on the last row / column, and refused ones
    pc = np.array([po.world2cam(cam, Rcw @ p + Pcw) for p in xyz.astype(np.float64)])
    pz = xyz.astype(np.float64) @ Rcw.T + Pcw
    _, val = po.colorize(cam, Rcw, Pcw, bgr, xyz)
    assert ((pz[:, 2] < 0) & ~val).sum() >= 40
    assert (((pc[:, 0] < -1) | (pc[:, 0] >= W)) & ~val).sum() >= 40
    assert ((((pc[:, 0] > -1) & (pc[:, 0] < 0)) | ((pc[:, 1] > -1) & (pc[:, 1] < 0))) & val).sum() >= 40
    assert (((pc[:, 0] >= W - 1) | (pc[:, 1] >= H - 1)) & val).sum() >= 40
    assert 0 < len(got) < len(xyz)
    assert (got["w"] == 1.0).all() and (got["a"] == 255).all() and not got["pad"].any()


def test_empty_and_none_kept(flb, po, emu):
    cam, Rcw, Pcw, bgr, xyz = world_cloud(flb, "T0", 4)
    assert len(emu_cloud(emu, cam, Rcw, Pcw, bgr, xyz[:0])) == 0
    behind = edge_points(np.random.default_rng(5), cam, Rcw, Pcw, 30)[:30]
    assert len(emu_cloud(emu, cam, Rcw, Pcw, bgr, behind)) == 0 == len(oracle_records(po, cam, Rcw, Pcw, bgr, behind))


@pytest.mark.parametrize("chunk_log2", [4, 7, 10])
def test_save_is_the_frames_concatenated(flb, po, emu, chunk_log2):
    """Frames of T0 and C2 size appended to a save with small chunks; the whole save and slices that start, end or
    cross chunk boundaries expand to the frames' records in call order."""
    save = emu.emu_save_new(chunk_log2)
    try:
        frames = []
        for k, (name, seed) in enumerate([("T0", 6), ("C2", 7), ("T0", 8), ("T0", 9)]):
            cam, Rcw, Pcw, bgr, xyz = world_cloud(flb, name, seed)
            if k == 2:
                xyz = xyz[:0]                                        # an empty frame appends nothing
            got = emu_cloud(emu, cam, Rcw, Pcw, bgr, xyz, save)
            assert got.tobytes() == oracle_records(po, cam, Rcw, Pcw, bgr, xyz).tobytes()
            frames.append(got)
        whole = np.concatenate(frames)
        n = emu.emu_save_size(save)
        assert n == len(whole) > 3 << chunk_log2
        out = np.zeros(n, RGB_POINT)
        emu.emu_save_download(save, 0, int(n), _p(out))
        assert out.tobytes() == whole.tobytes()
        c = 1 << chunk_log2
        for first, count in [(0, 1), (c - 1, 2), (c, c), (c - 3, 2 * c + 5), (n - 1, 1), (n - c - 1, c + 1), (5, 0)]:
            part = np.zeros(count, RGB_POINT)
            emu.emu_save_download(save, first, count, _p(part))
            assert part.tobytes() == whole[first:first + count].tobytes()
    finally:
        emu.emu_save_free(save)
