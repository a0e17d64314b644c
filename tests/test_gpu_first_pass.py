"""GPU tier: the L2 prefetch of the map at the start of the persistent LIO kernel changes no result: always on
(FLB_PREFETCH=1) and off (FLB_PREFETCH=0), the posterior state, covariance and both reports of whole frames (LIO update
then VIO update, the L2 flushed before every frame) are byte-identical, for the benchmark's workloads, a frame whose VIO
update has no patches and a device-built patch list.  FLB_PREFETCH is read once per process, so each setting runs in a
child process of its own."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[3])
import fastlivo_loader
flb = fastlivo_loader.load()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda:0")
out = {}

def put(key, x, lrep, vrep):
    out[key + "/state"] = x.vector()
    out[key + "/cov"] = np.array(x.cov[:])
    if lrep is not None:
        out[key + "/lio_report"] = np.frombuffer(bytes(lrep), np.uint8)
    out[key + "/vio_report"] = np.frombuffer(bytes(vrep), np.uint8)

def frames(key, f, n=3, patches=True):
    # the bench's frame: state reset to the prior, LIO update, prior := state, VIO update; L2 flushed before each
    cfg = f["cfg"]
    h = flb.Handle(device=0, cell_size=cfg.cell_size)
    h.map_upload(f["map_xyz"])
    h.scan_upload(f["scan_body"])
    h.camera_set(f["cam"])
    h.image_upload(f["image"])
    if patches:
        h.patches_upload(f["patch_pos"], f["patch_ref"], f["patch_level"])
    else:
        h.patches_upload(f["patch_pos"][:0], f["patch_ref"][:0], f["patch_level"][:0])
    x0 = flb.capi.State18.from_frame(f)
    h.state_upload(x0, x0.copy())
    lprm = flb.capi.lio_params(f, cfg.lio_passes - 1, early_stop=False)
    vprm = flb.capi.vio_params(f, cfg.vio_passes, early_stop=False, force_all_passes=True)
    for i in range(n):
        torch.cuda.synchronize()
        flush.zero_()
        torch.cuda.synchronize()
        if i:
            h.state_reset_enqueue()
        h.lio_update_enqueue(lprm)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
    x, lrep, vrep = h.state_download()
    put(key, x, lrep, vrep)
    h.close()

for name in ("C2", "C3", "C4", "T0", "T1"):
    frames(name, flb.synth.make_frame(name))
frames("T1_no_patches", flb.synth.make_frame("T1"), patches=False)

# device-built patch list (flb_vmap_select -> VIO, the count never visits the host), behind a LIO update
sys.path.insert(0, sys.argv[4])
from test_vmap_select import GpuVMap
seq = flb.synth.make_visual_sequence("T0", 3)
fr0, fr1 = seq["frames"][0], seq["frames"][1]
fv = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
t0 = flb.synth.make_frame("T0")
x0 = flb.capi.State18.make(fr1["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr1["p"] + [0.02, -0.015, 0.01],
                           cov=np.diag(np.repeat([1e-4, 1e-3, 1e-2, 1e-4, 1e-3, 1e-4], 3)))
h = flb.Handle(device=0)
g = GpuVMap(h, seq, 16, 300.0, 0, 0.0)
g.select(fr0["image"], fr0["Rcw"], fr0["Pcw"], fr0["pg_down"])
g.grow(fr0["image"], fr0["Rcw"], fr0["Pcw"], fr0["pg"], 0)
h.image_upload(fr1["image"])
h.map_upload(t0["map_xyz"])
h.scan_upload(t0["scan_body"])
h.state_upload(x0, x0.copy())
h.vmap_select(None, None, fr1["pg_down"], blocking=False)
h.vmap_grow(None, None, fr1["pg"], 1)
torch.cuda.synchronize()
flush.zero_()
torch.cuda.synchronize()
h.lio_update_enqueue(flb.capi.lio_params(t0, 2, early_stop=False))
h.state_set_prior_enqueue()
h.vio_update_enqueue(flb.capi.vio_params(fv, 4))
x, lrep, vrep = h.state_download()
put("pn_dev", x, lrep, vrep)
h.close()
np.savez(sys.argv[1], **out)
"""


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("first_pass")
    res = {}
    for mode in ("0", "1"):
        path = str(d / ("prefetch_%s.npz" % mode))
        env = dict(os.environ, FLB_PREFETCH=mode)
        r = subprocess.run([sys.executable, "-c", CHILD, path, ROOT, os.path.join(ROOT, "fast-livo_b200"),
                            os.path.join(ROOT, "tests")], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, "FLB_PREFETCH=%s child failed:\n%s\n%s" % (mode, r.stdout[-3000:], r.stderr[-3000:])
        res[mode] = dict(np.load(path))
    return res


@pytest.mark.parametrize("case", ["C2", "C3", "C4", "T0", "T1", "T1_no_patches", "pn_dev"])
def test_prefetch_on_and_off_byte_equal(runs, case):
    a, b = runs["0"], runs["1"]
    keys = sorted(k for k in a if k.startswith(case + "/"))
    assert keys and keys == sorted(k for k in b if k.startswith(case + "/"))
    for k in keys:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert a[k].tobytes() == b[k].tobytes(), "%s differs with the L2 prefetch on and off" % k
