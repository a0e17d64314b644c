"""GPU tier: the LIO and VIO update calls pinned to fixed values.  On T1 and C2, on a persistent and a kernel-per-pass
handle, one sequence runs every update entry point: flb_lio_pass at rematch 0/1 and width 6/12, flb_vio_pass at levels
0-2, the blocking flb_lio_update, flb_vio_update and flb_vio_update_level, the enqueue path with a pending reset and a
pending prior, flb_frame_enqueue into both result slots, a batch of three frames with and without VIO,
flb_lio_update_ikfom, and a device-built patch list (flb_vmap_select without a read-back, then the VIO update).  It also
runs the refusals: no state, no camera, a camera / image size mismatch at every caller, max_iteration out of range, a
batch frame not set and a wait on an empty result slot.  After every call it records the return code, the error text,
the launch count and a digest of every output.  The other update tests compare against the checker or against a
second run of the same code; this one catches any change to the launches, the messages, the order of the checks and
the bytes of the results.

EXPECTED was recorded on an NVIDIA H100 80GB HBM3 (700 W power limit, 132 SMs) with the host code that built each
kernel argument block by hand at every call site.  The persistent kernels size their grid from the SM count and their
sums are grouped by block, so the values hold for that card: the test checks the device name and SM count first."""
import ctypes as C
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

UNSET = -7.0                                 # what the outputs hold before a call: a refusal leaves them so


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


def run_sequence(flb, po, name, persistent):
    """[(label, rc, error text or None, launches, digest of the call's outputs)] after every call of the sequence."""
    cp = flb.capi
    L = cp.lib()
    f = flb.synth.make_frame(name)
    cfg = f["cfg"]
    h = flb.Handle(device=0, cell_size=cfg.cell_size, persistent=persistent)
    lprm = cp.lio_params(f, cfg.lio_passes - 1)
    vprm = cp.vio_params(f, cfg.vio_passes)
    x0 = cp.State18.from_frame(f)
    out = []

    def state(x=None):
        s = cp.State18()
        C.memmove(C.byref(s), C.byref(x0 if x is None else x), C.sizeof(s))
        return s

    def step(label, fn):
        """fn() -> (rc, outputs)."""
        l0 = h.launch_count()
        rc, outs = fn()
        launches = h.launch_count() - l0
        err = L.flb_last_error(h.h).decode() if rc else None
        out.append((label, rc, err, launches, digest(*outs)))

    def lio_pass(rematch, width):
        eq = cp.NormalEq()
        rc = L.flb_lio_pass(h.h, C.byref(lprm), cp._p(np.ascontiguousarray(f["R_prop"])), cp._p(np.ascontiguousarray(f["p_prop"])),
                            rematch, width, C.byref(eq))
        if rc:
            return rc, [eq]
        N = len(f["scan_body"])
        ex = [np.full((N, k), UNSET, dt) for k, dt in ((3, np.float32), (5, np.int32), (5, np.float32), (4, np.float32),
                                                         (1, np.float32), (1, np.uint8), (width, np.float64), (1, np.float64),
                                                         (1, np.int32))]
        n = C.c_int(-7)
        rc = L.flb_lio_export(h.h, *[cp._p(a) for a in ex], C.byref(n))
        return rc, [eq, np.int32(n.value)] + ex

    def vio_pass(level):
        eq = cp.VioEq()
        rc = L.flb_vio_pass(h.h, C.byref(vprm), cp._p(np.ascontiguousarray(f["R_prop"])), cp._p(np.ascontiguousarray(f["p_prop"])),
                            level, C.byref(eq))
        if rc:
            return rc, [eq]
        Pn = len(f["patch_pos"])
        z, H, e = np.full(Pn * 64, UNSET), np.full((Pn * 64, 6), UNSET), np.full(Pn, UNSET, np.float32)
        rc = L.flb_vio_export(h.h, cp._p(z), cp._p(H), cp._p(e))
        return rc, [eq, z, H, e]

    def lio_update(prm=lprm):
        x, xp, rep = state(), state(), cp.LioReport()
        return L.flb_lio_update(h.h, C.byref(prm), C.byref(x), C.byref(xp), C.byref(rep)), [x, rep]

    def vio_update():
        x, xp, rep = state(), state(), cp.VioReport()
        return L.flb_vio_update(h.h, C.byref(vprm), C.byref(x), C.byref(xp), C.byref(rep)), [x, rep]

    def vio_update_level(level, total_residual):
        x, xp, rep = state(), state(), cp.VioReport()
        le, G = C.c_float(UNSET), np.full((18, 6), UNSET)
        rc = L.flb_vio_update_level(h.h, C.byref(vprm), level, C.c_float(total_residual), C.byref(x), C.byref(xp), C.byref(le),
                                    cp._p(G), C.byref(rep))
        return rc, [x, rep, np.float32(le.value), G]

    def vio_errors():
        e = np.full(len(f["patch_pos"]), UNSET, np.float32)
        return L.flb_vio_errors(h.h, cp._p(e), len(e)), [e]

    def download():
        x, lr, vr = cp.State18(), cp.LioReport(), cp.VioReport()
        return L.flb_state_download(h.h, C.byref(x), C.byref(lr), C.byref(vr)), [x, lr, vr]

    def wait(slot):
        x, lr, vr = cp.State18(), cp.LioReport(), cp.VioReport()
        return L.flb_state_download_wait(h.h, slot, C.byref(x), C.byref(lr), C.byref(vr)), [x, lr, vr]

    def candidates():
        ncell = (f["cam"]["width"] // 40) * (f["cam"]["height"] // 40)
        mv, win = np.zeros(ncell, np.float32), np.full(ncell, -7, np.int32)
        pts = np.ascontiguousarray(f["map_xyz"][:256])
        rc = L.flb_visual_candidates(h.h, cp._p(np.ascontiguousarray(f["R_prop"])), cp._p(np.ascontiguousarray(f["p_prop"])),
                                     cp._p(pts), len(pts), 3, 40, 40, cp._p(mv), cp._p(win))
        return rc, [mv, win]

    def batch_frames():
        rs = []
        for b in range(3):
            x, lr, vr = h.batch_state_download(b)
            rs += [x, lr, vr]
        return rs

    def enq(fn, *a):
        return lambda: (fn(h.h, *[C.byref(v) if isinstance(v, C.Structure) else v for v in a]), [])

    def bad(prm, it):
        p = type(prm).from_buffer_copy(prm)
        p.max_iteration = it
        return p

    scans = [np.ascontiguousarray(f["scan_body"]), np.ascontiguousarray(f["scan_body"][::2]), np.ascontiguousarray(f["scan_body"][1::3])]

    # refusals on a fresh handle
    step("lio_enqueue-no-map", enq(L.flb_lio_update_enqueue, lprm))
    step("vio_enqueue-no-camera", enq(L.flb_vio_update_enqueue, vprm))
    step("vio_pass-no-camera", lambda: vio_pass(0))
    step("vio_update_level-no-camera", lambda: vio_update_level(2, 1e10))
    step("visual_candidates-no-camera", candidates)
    step("wait-empty-slot", lambda: wait(0))
    h.map_upload(f["map_xyz"])
    h.scan_upload(scans[0])
    h.patches_upload(f["patch_pos"], f["patch_ref"], f["patch_level"])
    step("lio_enqueue-no-state", enq(L.flb_lio_update_enqueue, lprm))
    step("vio_update-no-camera", vio_update)
    h.batch_begin(3, len(scans[0]))
    h.batch_set_frame(0, scans[0], state(), state())
    h.batch_set_frame(2, scans[2], state(), state())
    step("batch-frame-not-set", enq(L.flb_batch_update_enqueue, lprm, vprm))
    h.batch_set_frame(1, scans[1], state(), state())
    step("batch-no-camera", enq(L.flb_batch_update_enqueue, lprm, vprm))
    h.camera_set(f["cam"])
    step("vio_enqueue-no-image", enq(L.flb_vio_update_enqueue, vprm))

    # a camera twice the image's size: every caller that reads the image refuses
    h.image_upload(f["image"])
    h.camera_set(dict(f["cam"], width=2 * f["cam"]["width"], height=2 * f["cam"]["height"]))
    step("vio_enqueue-mismatch", enq(L.flb_vio_update_enqueue, vprm))
    step("vio_update-mismatch", vio_update)
    step("visual_candidates-mismatch", candidates)
    step("vio_pass-mismatch", lambda: vio_pass(1))
    step("vio_update_level-mismatch", lambda: vio_update_level(2, 1e10))
    step("batch-mismatch", enq(L.flb_batch_update_enqueue, lprm, vprm))
    h.camera_set(f["cam"])

    h.scan_upload(scans[0])
    h.state_upload(x0, state())
    step("lio_enqueue-max_iteration-1001", enq(L.flb_lio_update_enqueue, bad(lprm, 1001)))
    step("lio_enqueue-max_iteration-neg", enq(L.flb_lio_update_enqueue, bad(lprm, -1)))
    step("vio_enqueue-max_iteration-1001", enq(L.flb_vio_update_enqueue, bad(vprm, 1001)))

    # batched frames, without and with VIO
    step("batch-lio", enq(L.flb_batch_update_enqueue, lprm, None))
    step("batch-lio-frames", lambda: (0, batch_frames()))
    h.batch_state_reset_enqueue()
    step("batch-lio-vio", enq(L.flb_batch_update_enqueue, lprm, vprm))
    step("batch-lio-vio-frames", lambda: (0, batch_frames()))

    # single passes and their exports
    for rematch, width in ((1, 6), (0, 6), (1, 12), (0, 12)):
        step(f"lio_pass-r{rematch}-w{width}", lambda: lio_pass(rematch, width))
    for level in (0, 1, 2):
        step(f"vio_pass-l{level}", lambda: vio_pass(level))

    # blocking updates
    step("lio_update", lio_update)
    step("vio_update", vio_update)
    step("vio_errors", vio_errors)
    for level in (2, 1, 0):
        step(f"vio_update_level-l{level}", lambda: vio_update_level(level, 1e10))
    step("vio_update_level-errors", vio_errors)

    # the enqueue path: a pending reset, then a pending prior (each taken by the next kernel, or flushed)
    h.state_upload(x0, state())
    step("lio_enqueue", enq(L.flb_lio_update_enqueue, lprm))
    h.state_reset_enqueue()
    step("lio_enqueue-pending-reset", enq(L.flb_lio_update_enqueue, lprm))
    h.state_set_prior_enqueue()
    step("vio_enqueue-pending-prior", enq(L.flb_vio_update_enqueue, vprm))
    step("download-after-prior", download)
    h.state_reset_enqueue()
    step("vio_enqueue-pending-reset", enq(L.flb_vio_update_enqueue, vprm))
    step("download-after-reset", download)
    step("vio_enqueue-errors", vio_errors)

    # whole frames into both result slots
    img = np.ascontiguousarray(f["image"])
    pos, ref, lev = (np.ascontiguousarray(f["patch_pos"], np.float64), np.ascontiguousarray(f["patch_ref"], np.float32),
                     np.ascontiguousarray(f["patch_level"], np.int32))
    fi0 = h.frame_inputs(scans[0], state(), state(), img, pos, ref, lev)
    fi1 = h.frame_inputs(scans[1], state(), state())
    step("frame_enqueue-slot0", enq(L.flb_frame_enqueue, fi0, lprm, vprm, 0))
    step("frame_enqueue-slot1", enq(L.flb_frame_enqueue, fi1, lprm, vprm, 1))
    step("wait-slot1", lambda: wait(1))
    step("wait-slot0", lambda: wait(0))
    step("wait-slot0-again", lambda: wait(0))
    h.scan_upload(scans[0])

    # IKFoM
    xi = cp.StateIkfom()
    C.memmove(C.byref(xi), C.byref(po.state_ikfom_from_frame(f)), C.sizeof(xi))
    ip = cp.IkfomParams()
    ip.laser_point_cov, ip.max_iteration = cfg.laser_point_cov, 4
    ip.limit[:] = [0.001] * 23
    irep = cp.IkfomReport()
    step("lio_update_ikfom", lambda: (L.flb_lio_update_ikfom(h.h, C.byref(ip), C.byref(xi), C.byref(irep)), [xi, irep]))
    h.close()

    # the visual map: its image guard, then a patch list built on the device feeding the VIO update
    seq = flb.synth.make_visual_sequence("T0", 3)
    fr0, fr1 = seq["frames"][0], seq["frames"][1]
    fv = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
    t0 = flb.synth.make_frame("T0")
    xv = cp.State18.make(fr1["R"] @ flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])), fr1["p"] + [0.02, -0.015, 0.01],
                         cov=np.diag(np.repeat([1e-4, 1e-3, 1e-2, 1e-4, 1e-3, 1e-4], 3)))
    h = flb.Handle(device=0, persistent=persistent)
    pg0 = np.ascontiguousarray(fr0["pg"], np.float32)

    def grow(frame_id, R=None, P=None, pg=pg0):
        return lambda: (L.flb_vmap_grow(h.h, cp._p(R), cp._p(P), cp._p(pg), len(pg), 3, frame_id), [])

    R0, P0 = np.ascontiguousarray(fr0["Rcw"], np.float64), np.ascontiguousarray(fr0["Pcw"], np.float64)
    h.camera_set(seq["cam"])
    h.vmap_reset(seq, grid_size=16, outlier_threshold=300.0)
    step("vmap_grow-no-image", grow(0, R0, P0))
    h.image_upload(fr0["image"])
    h.camera_set(dict(seq["cam"], width=2 * seq["cam"]["width"], height=2 * seq["cam"]["height"]))
    step("vmap_grow-mismatch", grow(0, R0, P0))
    h.camera_set(seq["cam"])
    step("vmap_select", lambda: (0, [np.int32(h.vmap_select(R0, P0, fr0["pg_down"]))]))
    step("vmap_grow", grow(0, R0, P0))
    h.image_upload(fr1["image"])
    h.map_upload(t0["map_xyz"])
    h.scan_upload(t0["scan_body"])
    h.state_upload(xv, xv.copy())
    h.vmap_select(None, None, fr1["pg_down"], blocking=False)
    step("vmap_grow-1", grow(1, pg=np.ascontiguousarray(fr1["pg"], np.float32)))
    step("pn_dev-lio_enqueue", enq(L.flb_lio_update_enqueue, cp.lio_params(t0, 2, early_stop=False)))
    h.state_set_prior_enqueue()
    fvp = cp.vio_params(fv, 4)
    step("pn_dev-vio_enqueue", enq(L.flb_vio_update_enqueue, fvp))
    step("pn_dev-download", download)
    h.vmap_select(None, None, fr1["pg_down"], blocking=False)
    xb, xbp, vrep = state(xv), state(xv), cp.VioReport()
    step("pn_dev-vio_update", lambda: (L.flb_vio_update(h.h, C.byref(fvp), C.byref(xb), C.byref(xbp), C.byref(vrep)), [xb, vrep]))
    h.close()
    return out


DEVICE = ('NVIDIA H100 80GB HBM3', 132)         # name and SM count of the card EXPECTED was recorded on
EXPECTED = {    # (label, rc, error text or None, launches, digest of the outputs) after every call
    ('T1', 1): [
        ('lio_enqueue-no-map', -4, 'flb_lio_update: map and scan must be uploaded first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-camera', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_pass-no-camera', -4, 'flb_vio_pass: camera and image must be set first', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-no-camera', -4, 'flb_vio_update_level: camera and image must be set first', 0, 'cc09ab2d3f74eb8b'),
        ('visual_candidates-no-camera', -4, 'flb_visual_candidates: camera and image must be set first', 0, 'd6f41740202d4fcd'),
        ('wait-empty-slot', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_enqueue-no-state', -4, 'flb_lio_update: no device state (flb_state_upload)', 0, 'e3b0c44298fc1c14'),
        ('vio_update-no-camera', -4, 'flb_vio_update: camera and image must be set first', 1, '3c6c5c8854877b0f'),
        ('batch-frame-not-set', -4, 'flb_batch_update_enqueue: frame 1 not set', 0, 'e3b0c44298fc1c14'),
        ('batch-no-camera', -4, 'flb_batch_update_enqueue: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-image', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vio_update-mismatch', -4, 'camera / image size mismatch', 0, '3c6c5c8854877b0f'),
        ('visual_candidates-mismatch', -4, 'camera / image size mismatch', 0, 'd6f41740202d4fcd'),
        ('vio_pass-mismatch', -4, 'camera / image size mismatch', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-mismatch', -4, 'camera / image size mismatch', 0, 'cc09ab2d3f74eb8b'),
        ('batch-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-neg', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('batch-lio', 0, None, 9, 'e3b0c44298fc1c14'),
        ('batch-lio-frames', 0, None, 0, '443162625773e5d1'),
        ('batch-lio-vio', 0, None, 28, 'e3b0c44298fc1c14'),
        ('batch-lio-vio-frames', 0, None, 0, '5ba98bdabfe1ae09'),
        ('lio_pass-r1-w6', 0, None, 2, '48029132e48dffc2'),
        ('lio_pass-r0-w6', 0, None, 2, '48029132e48dffc2'),
        ('lio_pass-r1-w12', 0, None, 2, 'c7f6114857d94781'),
        ('lio_pass-r0-w12', 0, None, 2, 'c7f6114857d94781'),
        ('vio_pass-l0', 0, None, 2, '6c6a74420abca63a'),
        ('vio_pass-l1', 0, None, 2, '276ec44060060310'),
        ('vio_pass-l2', 0, None, 2, 'baa70d0d10dead0b'),
        ('lio_update', 0, None, 2, '73ff46c1b7bb65fc'),
        ('vio_update', 0, None, 2, '0edfc66da1ee11d3'),
        ('vio_errors', 0, None, 0, '0135396254f94bee'),
        ('vio_update_level-l2', 0, None, 9, 'ca1eb170f6d056c1'),
        ('vio_update_level-l1', 0, None, 9, '5c5cc1b3186d1aa9'),
        ('vio_update_level-l0', 0, None, 9, 'a512fef66212fcba'),
        ('vio_update_level-errors', 0, None, 0, 'bb540961da6c5075'),
        ('lio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('lio_enqueue-pending-reset', 0, None, 1, 'e3b0c44298fc1c14'),
        ('vio_enqueue-pending-prior', 0, None, 1, 'e3b0c44298fc1c14'),
        ('download-after-prior', 0, None, 0, 'd90c6f973ec3c14a'),
        ('vio_enqueue-pending-reset', 0, None, 1, 'e3b0c44298fc1c14'),
        ('download-after-reset', 0, None, 0, '01e4b006e0165354'),
        ('vio_enqueue-errors', 0, None, 0, '0135396254f94bee'),
        ('frame_enqueue-slot0', 0, None, 5, 'e3b0c44298fc1c14'),
        ('frame_enqueue-slot1', 0, None, 5, 'e3b0c44298fc1c14'),
        ('wait-slot1', 0, None, 0, '25d8a9e7437bf19f'),
        ('wait-slot0', 0, None, 0, 'd90c6f973ec3c14a'),
        ('wait-slot0-again', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_update_ikfom', 0, None, 1, 'cec3e501ac775b6e'),
        ('vmap_grow-no-image', -4, 'flb_vmap_grow: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vmap_grow-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vmap_select', 0, None, 6, 'df3f619804a92fdb'),
        ('vmap_grow', 0, None, 5, 'e3b0c44298fc1c14'),
        ('vmap_grow-1', 0, None, 6, 'e3b0c44298fc1c14'),
        ('pn_dev-lio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('pn_dev-vio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('pn_dev-download', 0, None, 0, 'dd5cc2c89644b8de'),
        ('pn_dev-vio_update', 0, None, 2, '2b102d3ad381c34f'),
    ],
    ('T1', 0): [
        ('lio_enqueue-no-map', -4, 'flb_lio_update: map and scan must be uploaded first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-camera', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_pass-no-camera', -4, 'flb_vio_pass: camera and image must be set first', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-no-camera', -4, 'flb_vio_update_level: camera and image must be set first', 0, 'cc09ab2d3f74eb8b'),
        ('visual_candidates-no-camera', -4, 'flb_visual_candidates: camera and image must be set first', 0, 'd6f41740202d4fcd'),
        ('wait-empty-slot', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_enqueue-no-state', -4, 'flb_lio_update: no device state (flb_state_upload)', 0, 'e3b0c44298fc1c14'),
        ('vio_update-no-camera', -4, 'flb_vio_update: camera and image must be set first', 1, '3c6c5c8854877b0f'),
        ('batch-frame-not-set', -4, 'flb_batch_update_enqueue: frame 1 not set', 0, 'e3b0c44298fc1c14'),
        ('batch-no-camera', -4, 'flb_batch_update_enqueue: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-image', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vio_update-mismatch', -4, 'camera / image size mismatch', 0, '3c6c5c8854877b0f'),
        ('visual_candidates-mismatch', -4, 'camera / image size mismatch', 0, 'd6f41740202d4fcd'),
        ('vio_pass-mismatch', -4, 'camera / image size mismatch', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-mismatch', -4, 'camera / image size mismatch', 0, 'cc09ab2d3f74eb8b'),
        ('batch-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-neg', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('batch-lio', 0, None, 9, 'e3b0c44298fc1c14'),
        ('batch-lio-frames', 0, None, 0, '443162625773e5d1'),
        ('batch-lio-vio', 0, None, 28, 'e3b0c44298fc1c14'),
        ('batch-lio-vio-frames', 0, None, 0, '5ba98bdabfe1ae09'),
        ('lio_pass-r1-w6', 0, None, 2, '48029132e48dffc2'),
        ('lio_pass-r0-w6', 0, None, 2, '48029132e48dffc2'),
        ('lio_pass-r1-w12', 0, None, 2, 'c7f6114857d94781'),
        ('lio_pass-r0-w12', 0, None, 2, 'c7f6114857d94781'),
        ('vio_pass-l0', 0, None, 2, '6c6a74420abca63a'),
        ('vio_pass-l1', 0, None, 2, '276ec44060060310'),
        ('vio_pass-l2', 0, None, 2, 'baa70d0d10dead0b'),
        ('lio_update', 0, None, 10, '225e82285831f276'),
        ('vio_update', 0, None, 20, '04a9db97ce9bfce7'),
        ('vio_errors', 0, None, 0, '0135396254f94bee'),
        ('vio_update_level-l2', 0, None, 9, 'ca1eb170f6d056c1'),
        ('vio_update_level-l1', 0, None, 9, '5c5cc1b3186d1aa9'),
        ('vio_update_level-l0', 0, None, 9, 'a512fef66212fcba'),
        ('vio_update_level-errors', 0, None, 0, 'bb540961da6c5075'),
        ('lio_enqueue', 0, None, 9, 'e3b0c44298fc1c14'),
        ('lio_enqueue-pending-reset', 0, None, 9, 'e3b0c44298fc1c14'),
        ('vio_enqueue-pending-prior', 0, None, 19, 'e3b0c44298fc1c14'),
        ('download-after-prior', 0, None, 0, '65cfcec593b348f5'),
        ('vio_enqueue-pending-reset', 0, None, 19, 'e3b0c44298fc1c14'),
        ('download-after-reset', 0, None, 0, '143faec0790c85fd'),
        ('vio_enqueue-errors', 0, None, 0, '0135396254f94bee'),
        ('frame_enqueue-slot0', 0, None, 31, 'e3b0c44298fc1c14'),
        ('frame_enqueue-slot1', 0, None, 31, 'e3b0c44298fc1c14'),
        ('wait-slot1', 0, None, 0, '6388d5ae9faaf300'),
        ('wait-slot0', 0, None, 0, '65cfcec593b348f5'),
        ('wait-slot0-again', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_update_ikfom', 0, None, 1, 'cec3e501ac775b6e'),
        ('vmap_grow-no-image', -4, 'flb_vmap_grow: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vmap_grow-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vmap_select', 0, None, 6, 'df3f619804a92fdb'),
        ('vmap_grow', 0, None, 5, 'e3b0c44298fc1c14'),
        ('vmap_grow-1', 0, None, 6, 'e3b0c44298fc1c14'),
        ('pn_dev-lio_enqueue', 0, None, 7, 'e3b0c44298fc1c14'),
        ('pn_dev-vio_enqueue', 0, None, 25, 'e3b0c44298fc1c14'),
        ('pn_dev-download', 0, None, 0, 'de8a584dfb264bb7'),
        ('pn_dev-vio_update', 0, None, 26, '3248239a56ef00c1'),
    ],
    ('C2', 1): [
        ('lio_enqueue-no-map', -4, 'flb_lio_update: map and scan must be uploaded first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-camera', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_pass-no-camera', -4, 'flb_vio_pass: camera and image must be set first', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-no-camera', -4, 'flb_vio_update_level: camera and image must be set first', 0, '5d65e0574e049f74'),
        ('visual_candidates-no-camera', -4, 'flb_visual_candidates: camera and image must be set first', 0, 'd6f41740202d4fcd'),
        ('wait-empty-slot', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_enqueue-no-state', -4, 'flb_lio_update: no device state (flb_state_upload)', 0, 'e3b0c44298fc1c14'),
        ('vio_update-no-camera', -4, 'flb_vio_update: camera and image must be set first', 1, '4b0670d56f046361'),
        ('batch-frame-not-set', -4, 'flb_batch_update_enqueue: frame 1 not set', 0, 'e3b0c44298fc1c14'),
        ('batch-no-camera', -4, 'flb_batch_update_enqueue: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-image', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vio_update-mismatch', -4, 'camera / image size mismatch', 0, '4b0670d56f046361'),
        ('visual_candidates-mismatch', -4, 'camera / image size mismatch', 0, 'd6f41740202d4fcd'),
        ('vio_pass-mismatch', -4, 'camera / image size mismatch', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-mismatch', -4, 'camera / image size mismatch', 0, '5d65e0574e049f74'),
        ('batch-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-neg', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('batch-lio', 0, None, 7, 'e3b0c44298fc1c14'),
        ('batch-lio-frames', 0, None, 0, 'f2799053d16fc908'),
        ('batch-lio-vio', 0, None, 26, 'e3b0c44298fc1c14'),
        ('batch-lio-vio-frames', 0, None, 0, '5fde951db62d0990'),
        ('lio_pass-r1-w6', 0, None, 2, '5e22a8406bad2673'),
        ('lio_pass-r0-w6', 0, None, 2, '5e22a8406bad2673'),
        ('lio_pass-r1-w12', 0, None, 2, 'ea93b44d38839aa0'),
        ('lio_pass-r0-w12', 0, None, 2, 'ea93b44d38839aa0'),
        ('vio_pass-l0', 0, None, 2, '65a4e86d90ad8587'),
        ('vio_pass-l1', 0, None, 2, 'f05c3b9860951c24'),
        ('vio_pass-l2', 0, None, 2, 'd8624a4074d2c19a'),
        ('lio_update', 0, None, 2, 'd311229e1950b04b'),
        ('vio_update', 0, None, 2, 'a6972f159fa9885e'),
        ('vio_errors', 0, None, 0, 'e232d38551cd0721'),
        ('vio_update_level-l2', 0, None, 9, '0c1eeaa98083f0c9'),
        ('vio_update_level-l1', 0, None, 9, '6369568a130969ef'),
        ('vio_update_level-l0', 0, None, 9, '44a2a35be8349cf1'),
        ('vio_update_level-errors', 0, None, 0, 'd46ad150d5027e0a'),
        ('lio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('lio_enqueue-pending-reset', 0, None, 1, 'e3b0c44298fc1c14'),
        ('vio_enqueue-pending-prior', 0, None, 1, 'e3b0c44298fc1c14'),
        ('download-after-prior', 0, None, 0, '9d6f5bcafadd9743'),
        ('vio_enqueue-pending-reset', 0, None, 1, 'e3b0c44298fc1c14'),
        ('download-after-reset', 0, None, 0, '9cd4c07d27c6ac8a'),
        ('vio_enqueue-errors', 0, None, 0, 'e232d38551cd0721'),
        ('frame_enqueue-slot0', 0, None, 9, 'e3b0c44298fc1c14'),
        ('frame_enqueue-slot1', 0, None, 5, 'e3b0c44298fc1c14'),
        ('wait-slot1', 0, None, 0, 'c081081e3ade871d'),
        ('wait-slot0', 0, None, 0, '9d6f5bcafadd9743'),
        ('wait-slot0-again', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_update_ikfom', 0, None, 1, 'eb4683781a805b06'),
        ('vmap_grow-no-image', -4, 'flb_vmap_grow: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vmap_grow-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vmap_select', 0, None, 6, 'df3f619804a92fdb'),
        ('vmap_grow', 0, None, 5, 'e3b0c44298fc1c14'),
        ('vmap_grow-1', 0, None, 6, 'e3b0c44298fc1c14'),
        ('pn_dev-lio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('pn_dev-vio_enqueue', 0, None, 1, 'e3b0c44298fc1c14'),
        ('pn_dev-download', 0, None, 0, 'dd5cc2c89644b8de'),
        ('pn_dev-vio_update', 0, None, 2, '2b102d3ad381c34f'),
    ],
    ('C2', 0): [
        ('lio_enqueue-no-map', -4, 'flb_lio_update: map and scan must be uploaded first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-camera', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_pass-no-camera', -4, 'flb_vio_pass: camera and image must be set first', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-no-camera', -4, 'flb_vio_update_level: camera and image must be set first', 0, '5d65e0574e049f74'),
        ('visual_candidates-no-camera', -4, 'flb_visual_candidates: camera and image must be set first', 0, 'd6f41740202d4fcd'),
        ('wait-empty-slot', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_enqueue-no-state', -4, 'flb_lio_update: no device state (flb_state_upload)', 0, 'e3b0c44298fc1c14'),
        ('vio_update-no-camera', -4, 'flb_vio_update: camera and image must be set first', 1, '4b0670d56f046361'),
        ('batch-frame-not-set', -4, 'flb_batch_update_enqueue: frame 1 not set', 0, 'e3b0c44298fc1c14'),
        ('batch-no-camera', -4, 'flb_batch_update_enqueue: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-no-image', -4, 'flb_vio_update: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vio_update-mismatch', -4, 'camera / image size mismatch', 0, '4b0670d56f046361'),
        ('visual_candidates-mismatch', -4, 'camera / image size mismatch', 0, 'd6f41740202d4fcd'),
        ('vio_pass-mismatch', -4, 'camera / image size mismatch', 0, 'd3df611a0ed2e328'),
        ('vio_update_level-mismatch', -4, 'camera / image size mismatch', 0, '5d65e0574e049f74'),
        ('batch-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('lio_enqueue-max_iteration-neg', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('vio_enqueue-max_iteration-1001', -1, 'max_iteration outside [0, 1000]', 0, 'e3b0c44298fc1c14'),
        ('batch-lio', 0, None, 7, 'e3b0c44298fc1c14'),
        ('batch-lio-frames', 0, None, 0, 'f2799053d16fc908'),
        ('batch-lio-vio', 0, None, 26, 'e3b0c44298fc1c14'),
        ('batch-lio-vio-frames', 0, None, 0, '5fde951db62d0990'),
        ('lio_pass-r1-w6', 0, None, 2, '5e22a8406bad2673'),
        ('lio_pass-r0-w6', 0, None, 2, '5e22a8406bad2673'),
        ('lio_pass-r1-w12', 0, None, 2, 'ea93b44d38839aa0'),
        ('lio_pass-r0-w12', 0, None, 2, 'ea93b44d38839aa0'),
        ('vio_pass-l0', 0, None, 2, '65a4e86d90ad8587'),
        ('vio_pass-l1', 0, None, 2, 'f05c3b9860951c24'),
        ('vio_pass-l2', 0, None, 2, 'd8624a4074d2c19a'),
        ('lio_update', 0, None, 8, '0cfe16c515fa8525'),
        ('vio_update', 0, None, 20, '865344c7b6f2227e'),
        ('vio_errors', 0, None, 0, 'e232d38551cd0721'),
        ('vio_update_level-l2', 0, None, 9, '0c1eeaa98083f0c9'),
        ('vio_update_level-l1', 0, None, 9, '6369568a130969ef'),
        ('vio_update_level-l0', 0, None, 9, '44a2a35be8349cf1'),
        ('vio_update_level-errors', 0, None, 0, 'd46ad150d5027e0a'),
        ('lio_enqueue', 0, None, 7, 'e3b0c44298fc1c14'),
        ('lio_enqueue-pending-reset', 0, None, 7, 'e3b0c44298fc1c14'),
        ('vio_enqueue-pending-prior', 0, None, 19, 'e3b0c44298fc1c14'),
        ('download-after-prior', 0, None, 0, '1450989a3a6c40e4'),
        ('vio_enqueue-pending-reset', 0, None, 19, 'e3b0c44298fc1c14'),
        ('download-after-reset', 0, None, 0, '1a00b237e5691ee7'),
        ('vio_enqueue-errors', 0, None, 0, 'e232d38551cd0721'),
        ('frame_enqueue-slot0', 0, None, 33, 'e3b0c44298fc1c14'),
        ('frame_enqueue-slot1', 0, None, 29, 'e3b0c44298fc1c14'),
        ('wait-slot1', 0, None, 0, '6010229db7dfa28f'),
        ('wait-slot0', 0, None, 0, '1450989a3a6c40e4'),
        ('wait-slot0-again', -4, 'flb_state_download_wait: nothing enqueued in this slot', 0, '19c36509388e414a'),
        ('lio_update_ikfom', 0, None, 1, 'eb4683781a805b06'),
        ('vmap_grow-no-image', -4, 'flb_vmap_grow: camera and image must be set first', 0, 'e3b0c44298fc1c14'),
        ('vmap_grow-mismatch', -4, 'camera / image size mismatch', 0, 'e3b0c44298fc1c14'),
        ('vmap_select', 0, None, 6, 'df3f619804a92fdb'),
        ('vmap_grow', 0, None, 5, 'e3b0c44298fc1c14'),
        ('vmap_grow-1', 0, None, 6, 'e3b0c44298fc1c14'),
        ('pn_dev-lio_enqueue', 0, None, 7, 'e3b0c44298fc1c14'),
        ('pn_dev-vio_enqueue', 0, None, 25, 'e3b0c44298fc1c14'),
        ('pn_dev-download', 0, None, 0, 'de8a584dfb264bb7'),
        ('pn_dev-vio_update', 0, None, 26, '3248239a56ef00c1'),
    ],
}


@pytest.mark.parametrize("persistent", [1, 0], ids=["persistent", "per_pass"])
@pytest.mark.parametrize("name", ["T1", "C2"])
def test_update_calls_pinned(flb, po, name, persistent):
    assert device() == DEVICE, "recorded on %s with %d SMs: these values hold for that card only" % DEVICE
    got = run_sequence(flb, po, name, persistent)
    exp = EXPECTED[name, persistent]
    assert [g[0] for g in got] == [e[0] for e in exp]
    for g, e in zip(got, exp):
        assert g == e, g[0]
