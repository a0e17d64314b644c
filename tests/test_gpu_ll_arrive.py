"""GPU tier: the persistent kernels' two arrival paths -- worker sums as tagged lines the leader polls (default) and
the arrival counter (FLB_LL_ARRIVE=0) -- give byte-identical results: the same values summed in the same order.
FLB_LL_ARRIVE is read once per process, so each path runs in a child process of its own."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, ctypes as C
import numpy as np
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[3])
import fastlivo_loader
flb = fastlivo_loader.load()
out = {}

def put(key, h, x, lrep=None, vrep=None, errors=True):
    out[key + "/state"] = x.vector()
    out[key + "/cov"] = np.array(x.cov[:])
    if lrep is not None:
        out[key + "/lio_report"] = np.frombuffer(bytes(lrep), np.uint8)
    if vrep is not None:
        out[key + "/vio_report"] = np.frombuffer(bytes(vrep), np.uint8)
        if errors:
            out[key + "/errors"] = h.vio_errors()

def perturbed(f, s):
    x = flb.capi.State18.from_frame(f)
    return flb.capi.State18.make(x.R @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002]) * s),
                                 x.p + np.array([0.02, -0.015, 0.01]) * s, cov=x.P)

def frame_case(key, f, lT=4, vT=3, early=True, x0=None):
    h = flb.Handle(device=0, persistent=1)
    h.load_frame(f)
    x = x0.copy() if x0 is not None else flb.capi.State18.from_frame(f)
    lrep = h.lio_update(flb.capi.lio_params(f, lT, early_stop=early), x, x.copy())
    vrep = h.vio_update(flb.capi.vio_params(f, vT, early_stop=early), x, x.copy())
    put(key, h, x, lrep, vrep)
    h.close()

# full LIO + VIO frames
for name in ("C2", "C3", "C4", "T0", "T1"):
    frame_case(name, flb.synth.make_frame(name))

# early stop with many iterations from a perturbed start: levels end on a rejected step (speculation mispredicted)
for name in ("T1", "C2"):
    f = flb.synth.make_frame(name)
    frame_case(name + "_reject", f, lT=8, vT=10, early=True, x0=perturbed(f, 4.0))

# scan sizes around the H100 block counts
t1 = flb.synth.make_frame("T1")
for n in (131, 132, 133, 1047, 1048, 1049):
    f = dict(t1)
    keep = np.sort(np.random.default_rng(n).choice(len(f["scan_body"]), n, replace=False))
    f["scan_body"] = np.ascontiguousarray(f["scan_body"][keep])
    frame_case("scan%d" % n, f)

# device-built patch list (flb_vmap_select -> VIO, the count never visits the host)
sys.path.insert(0, sys.argv[4])
from test_vmap_select import GpuVMap
seq = flb.synth.make_visual_sequence("T0", 3)
fr0, fr1 = seq["frames"][0], seq["frames"][1]
fv = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
x0 = flb.capi.State18.make(fr1["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr1["p"] + [0.02, -0.015, 0.01],
                           cov=np.diag(np.repeat([1e-4, 1e-3, 1e-2, 1e-4, 1e-3, 1e-4], 3)))
h = flb.Handle(device=0)
g = GpuVMap(h, seq, 16, 300.0, 0, 0.0)
g.select(fr0["image"], fr0["Rcw"], fr0["Pcw"], fr0["pg_down"])
g.grow(fr0["image"], fr0["Rcw"], fr0["Pcw"], fr0["pg"], 0)
h.image_upload(fr1["image"])
h.state_upload(x0, x0.copy())
h.vmap_select(None, None, fr1["pg_down"], blocking=False)
h.vmap_grow(None, None, fr1["pg"], 1)
h.vio_update_enqueue(flb.capi.vio_params(fv, 4))
x, _, vrep = h.state_download()
put("pn_dev", h, x, vrep=vrep, errors=False)
h.close()

# back-to-back frames without a sync (the same frame again each time: tags of many epochs in the line buffer), and
# the same across the flag wrap-around (the line buffer is cleared there); each must equal a single frame
f = flb.synth.make_frame("C2")
lprm, vprm = flb.capi.lio_params(f, 4), flb.capi.vio_params(f, 3)
def chain(key, frames, epoch=None):
    h = flb.Handle(device=0, persistent=1)
    h.load_frame(f)
    if epoch is not None:
        fn = h.L.flb_debug_set_packet_epoch
        fn.argtypes = [C.c_void_p, C.c_uint]
        h._ck(fn(h.h, epoch))
    x0 = flb.capi.State18.from_frame(f)
    h.state_upload(x0, x0.copy())
    for i in range(frames):
        if i:
            h.state_reset_enqueue()
        h.lio_update_enqueue(lprm)
        h.state_set_prior_enqueue()
        h.vio_update_enqueue(vprm)
    x, lrep, vrep = h.state_download()
    put(key, h, x, lrep, vrep)
    h.close()
chain("chain1", 1)
chain("chain300", 300)
chain("chain_wrap", 8, epoch=0xFFFF0000 - 7 * 4096)
np.savez(sys.argv[1], **out)
"""


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("ll_arrive")
    res = {}
    for mode in ("0", "1"):
        path = str(d / ("mode%s.npz" % mode))
        env = dict(os.environ, FLB_LL_ARRIVE=mode)
        r = subprocess.run([sys.executable, "-c", CHILD, path, ROOT, os.path.join(ROOT, "fast-livo_b200"),
                            os.path.join(ROOT, "tests")], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, "FLB_LL_ARRIVE=%s child failed:\n%s\n%s" % (mode, r.stdout[-3000:], r.stderr[-3000:])
        res[mode] = dict(np.load(path))
    return res


CASES = ["C2", "C3", "C4", "T0", "T1", "T1_reject", "C2_reject", "scan131", "scan132", "scan133", "scan1047", "scan1048",
         "scan1049", "pn_dev", "chain1", "chain300", "chain_wrap"]


@pytest.mark.parametrize("case", CASES)
def test_lines_and_counter_byte_equal(runs, case):
    a, b = runs["0"], runs["1"]
    keys = sorted(k for k in a if k.startswith(case + "/"))
    assert keys and keys == sorted(k for k in b if k.startswith(case + "/"))
    for k in keys:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert a[k].tobytes() == b[k].tobytes(), "%s differs between the counter and the line arrival" % k


@pytest.mark.parametrize("case", ["chain300", "chain_wrap"])
def test_back_to_back_frames_equal_one_frame(runs, case):
    for mode in ("0", "1"):
        r = runs[mode]
        for part in ("state", "cov", "lio_report", "vio_report", "errors"):
            assert r["%s/%s" % (case, part)].tobytes() == r["chain1/%s" % part].tobytes(), (mode, case, part)
