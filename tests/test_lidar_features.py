"""CPU tier of flb_lidar_upload_features.  The checker (tests/oracle_pre/feat_oracle.cpp, the reference's sequential
feature branches) and the product's per-point device math composed as the kernels compose it (tests/hostemu/
lidar_features.cpp: one plane_judge per candidate, the visited chain by pointer doubling, the small-plane firing by
alternation, the chunked output) must agree byte for byte on pl_surf and on every point's final type, over structured
scenes of every kind, point_filter_num 1 to 4 and disB 0 and non-zero; and the scenes must reach every branch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import feat_oracle
from feat_util import DIS_B, FILTERS, SCENES, scene

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    """tests/hostemu/lidar_features.cpp built for the host (into a temporary directory)."""
    so = str(tmp_path_factory.mktemp("lidar_features") / "liblidar_features.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
                           "-shared", "-o", so, os.path.join(HERE, "hostemu", "lidar_features.cpp")])
    L = C.CDLL(so)
    L.emu_feat_process.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                   C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return L


def emu_process(L, fmt, records, dis_b):
    rec = np.frombuffer(records, np.uint8)
    n = rec.size // fmt["point_step"]
    out = np.zeros((max(n, 1), 4), np.float32)
    ft = np.zeros(max(n, 1), np.int32)
    nft, bad = C.c_int(), C.c_int()
    m = L.emu_feat_process(feat_oracle.fmt_ints(fmt).ctypes.data, fmt["blind"], dis_b, rec.ctypes.data if n else None, n,
                           out.ctypes.data, ft.ctypes.data, C.byref(nft), C.byref(bad))
    return out[:m], ft[:nft.value], bad.value


CASES = [(k, kw, pf, db) for k, kw in SCENES for pf in FILTERS for db in DIS_B]


@pytest.mark.parametrize("kind,kw,pf,dis_b", CASES, ids=[f"{k}-{kw['seed']}-{kw.get('timed', '')}-pf{pf}-b{db}" for k, kw, pf, db in CASES])
def test_checker_and_device_math_agree(emu, kind, kw, pf, dis_b):
    records, fmt = scene(kind, point_filter_num=pf, **kw)
    ref, ref_ft, flags, _ = feat_oracle.process(fmt, records, dis_b)
    got, got_ft, bad = emu_process(emu, fmt, records, dis_b)
    assert len(ref) > 0
    assert got_ft.tobytes() == ref_ft.tobytes()
    assert bad == int(not np.isfinite(ref).all())
    if bad:     # a NaN time has no place in the sort (the upload refuses such a cloud): the same points, in any order
        ref, got = (np.sort(a.view(np.dtype((np.void, 16))).ravel()) for a in (ref, got))
    assert got.tobytes() == ref.tobytes()


def test_scenes_reach_every_branch():
    total = {}
    for kind, kw in SCENES:
        for pf in FILTERS:
            for db in DIS_B:
                records, fmt = scene(kind, point_filter_num=pf, **kw)
                _, _, flags, _ = feat_oracle.process(fmt, records, db)
                for k, v in flags.items():
                    total[k] = total.get(k, 0) + v
    missing = [k for k, v in total.items() if v == 0]
    assert not missing, (missing, total)


@pytest.mark.parametrize("kind", ["livox", "ouster", "velodyne"])
def test_empty_and_tiny_messages(emu, kind):
    records, fmt = scene(kind, seed=5)
    step = fmt["point_step"]
    for n in (0, 1, 2, 7):
        r = records[:n * step]
        ref, ref_ft, _, _ = feat_oracle.process(fmt, r)
        got, got_ft, _ = emu_process(emu, fmt, r, 0.0)
        assert got.tobytes() == ref.tobytes() and got_ft.tobytes() == ref_ft.tobytes()


def test_nan_group_position_rule():
    """The exchange sort of :855-867 leaves every NaN where it was and sorts the rest descending around it."""
    rng = np.random.default_rng(3)
    for _ in range(300):
        n = int(rng.integers(2, 30))
        d = rng.choice([0.0, 0.5, 1.0, 2.0, np.nan, 3.0], n) * rng.choice([1.0, 1.5], n)
        a = list(d)
        for j in range(n - 1):
            for k in range(j + 1, n):
                if a[j] < a[k]:
                    a[j], a[k] = a[k], a[j]
        nan = np.isnan(d)
        rest = np.sort(d[~nan])[::-1]
        want = d.copy()
        want[~nan] = rest
        np.testing.assert_array_equal(np.array(a), want)


def golden_cases():
    import json
    z = np.load(os.path.join(HERE, "golden", "lidar_features_golden.npz"))
    for name in sorted({k.split("__")[0] for k in z.files}):
        fmt = json.loads(bytes(z[name + "__fmt"]).decode())
        yield name, z[name + "__records"].tobytes(), fmt, fmt.pop("dis_b"), z[name + "__cloud"], z[name + "__ftypes"]


def test_golden(emu):
    """The committed outputs: the checker and the device math both reproduce them, and the generator still makes the
    committed messages."""
    from golden.make_golden_features import GOLDEN_SCENES, name_of
    made = {name_of(*g): scene(g[0], point_filter_num=g[2], **g[1])[0] for g in GOLDEN_SCENES}
    n = 0
    for name, rec, fmt, dis_b, cloud, ftypes in golden_cases():
        ref, ref_ft, _, _ = feat_oracle.process(fmt, rec, dis_b)
        got, got_ft, _ = emu_process(emu, fmt, rec, dis_b)
        assert ref.tobytes() == cloud.tobytes() == got.tobytes() and ref_ft.tobytes() == ftypes.tobytes() == got_ft.tobytes()
        assert made[name] == rec
        n += 1
    assert n == len(GOLDEN_SCENES)
