"""GPU tier: flb_map_fov_segment (lasermap_fov_segment + Delete_Point_Boxes with the cube on the device).  The boxes and
the cube must equal the oracle's (tests/oracle_fov) bit for bit; the pruned map must equal a second handle driven by the
oracle's boxes through flb_map_delete_boxes (same rows, same kNN answers, same LIO posterior); frames whose boxes hold
no map point must leave the map untouched.  Every case runs on the dense cell table and on the sparse index.

The map is the C2 room (every 4th point) plus four translated copies, so that the boxes cut real slabs without ever
taking the whole map: the shipped configuration (cube 20 m) cuts the 20 m cube around the start and then the copies on
the negative diagonal; the 1000 m cube, driven along +x, cuts x slabs of the copy 400 m back and of the room's edge."""
import ctypes as C

import numpy as np
import pytest

import fov_oracle
from conftest import bits

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_STATE = -1, -4
OFFS = [(0, 0, 0), (-150, -150, -150), (-300, -300, -300), (-400, 0, 0), (0, 450, 0)]
CONFIGS = {"shipped": fov_oracle.SHIPPED, "cube1000": (1000.0, 300.0, 1.5)}
INDEX = {"dense": 0, "sparse": 2}


@pytest.fixture(scope="module")
def world(frames):
    f = frames("C2")
    room = f["map_xyz"][::4]
    m = np.concatenate([room + np.array(o, np.float32) for o in OFFS]).astype(np.float32)
    return f, m


def trajectory(f, cfg, n=30, seed=0):
    rng = np.random.default_rng(seed)
    p0 = np.asarray(f["p_true"], np.float64)
    if cfg == "shipped":
        t = p0 + rng.uniform(-3.0, 3.0, (n, 3))
    else:
        t = p0 + rng.normal(0, 0.5, (n, 3))
        t[:, 0] += 15.0 * np.arange(n)
    t[0] = p0
    return t


def handle(flb, f, m, index, scan=True):
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    if INDEX[index]:
        h.debug_set_map_index(INDEX[index])
    if m is not None:
        h.map_upload(m)
    if scan:
        h.scan_upload(f["scan_body"])
    return h


def same(a, b):
    return a.shape == b.shape and (bits(a) == bits(b)).all()


def inside(m, boxes):
    c = np.zeros(len(m), bool)
    for b in boxes:
        c |= ((m >= b[:3]) & (m < b[3:])).all(1)
    return c


def sorted_rows(m):
    return m[np.lexsort((m[:, 2], m[:, 1], m[:, 0]))]


# state_op_enqueued: the pose is the uploaded state restored by flb_state_reset_enqueue after a LIO update moved x, both
# still pending when the call is made (near the room only: the LIO update needs the map around it)
MODES = [(c, m) for c in CONFIGS for m in ("state_upload", "state_op_enqueued", "explicit")
         if not (c == "cube1000" and m == "state_op_enqueued")]


@pytest.mark.parametrize("cfg,mode", MODES)
@pytest.mark.parametrize("index", list(INDEX))
def test_boxes_match_oracle(flb, world, index, cfg, mode):
    f, m = world
    prm = CONFIGS[cfg]
    lprm = flb.capi.lio_params(f, 3)
    a = handle(flb, f, m, index)
    t = fov_oracle.Tracker(*prm)
    traj = trajectory(f, cfg)
    inits = (0, 10, 20) if mode == "state_op_enqueued" else (0,)
    if mode == "state_op_enqueued":                   # the LIO update does move x away from the uploaded position
        x = flb.capi.State18.from_frame(f)
        x.pos[:] = list(traj[0])
        a.lio_update(lprm, x, x.copy())
        assert (x.p != traj[0]).all()
    cut = 0
    for k, p in enumerate(traj):
        before = a.map_download()
        if mode == "explicit":
            boxes, local, nd = a.map_fov_segment(*prm, pos=p)
        else:
            x = flb.capi.State18.from_frame(f)
            x.pos[:] = list(p)
            a.state_upload(x, x.copy())
            if mode == "state_op_enqueued":
                a.lio_update_enqueue(lprm)
                a.state_reset_enqueue()                # x := the uploaded state, deferred: no synchronise before the call
                if k in inits[1:]:
                    a.map_fov_reset()
                    t.reset()
            boxes, local, nd = a.map_fov_segment(*prm)
        wb, wl = t.step(p)
        assert same(boxes, wb) and same(local, wl), k
        assert k not in inits or len(wb) == 0
        assert cfg != "shipped" or k in inits or len(wb) == 3
        assert nd == inside(before, wb).sum() and a.M == len(before) - nd, k
        cut += nd > 0
    assert 0 < cut < len(traj) - 1                    # real cuts and empty frames both occur
    a.close()


@pytest.mark.parametrize("index", list(INDEX))
def test_pose_after_lio_update_enqueue(flb, world, index):
    """NULL pose after flb_lio_update_enqueue with no synchronise: the cube steps at the posterior's position."""
    f, m = world
    prm = fov_oracle.SHIPPED
    lprm = flb.capi.lio_params(f, 3)
    a = handle(flb, f, m, index)
    t = fov_oracle.Tracker(*prm)
    for k in range(2):
        x = flb.capi.State18.from_frame(f)
        x.pos[:] = list(np.array(x.pos[:]) + k * np.array([0.2, -0.1, 0.05]))
        a.state_upload(x, x.copy())
        a.lio_update_enqueue(lprm)
        boxes, local, nd = a.map_fov_segment(*prm)
        xs, _, _ = a.state_download()
        wb, wl = t.step(xs.p)
        assert same(boxes, wb) and same(local, wl), k
    assert len(wb) == 3 and nd > 0
    a.close()


def assert_same_queries(flb, f, a, b, rng):
    ma, mb = a.map_download(), b.map_download()
    q = (ma[rng.integers(0, len(ma), 2000)] + rng.normal(0, 0.3, (2000, 3))).astype(np.float32)
    ia, da = a.knn(q)
    ib, db = b.knn(q)
    assert (bits(da) == bits(db)).all()
    assert ((ia >= 0) == (ib >= 0)).all()
    ca = np.where((ia >= 0)[..., None], ma[ia.clip(0)], 0).astype(np.float32)
    cb = np.where((ib >= 0)[..., None], mb[ib.clip(0)], 0).astype(np.float32)
    diff = (bits(ca) != bits(cb)).any(2).any(1)
    for r in np.nonzero(diff)[0]:                     # only among neighbours at the same distance may the order differ
        sa = sorted(zip(da[r].tolist(), map(tuple, ca[r].tolist())))
        sb = sorted(zip(db[r].tolist(), map(tuple, cb[r].tolist())))
        assert sa == sb, r
    lprm = flb.capi.lio_params(f, 3)
    xa, xb = flb.capi.State18.from_frame(f), flb.capi.State18.from_frame(f)
    ra = a.lio_update(lprm, xa, xa.copy())
    rb = b.lio_update(lprm, xb, xb.copy())
    assert bytes(xa) == bytes(xb) and bytes(ra) == bytes(rb)


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("index", list(INDEX))
def test_map_equals_delete_boxes(flb, world, index, cfg):
    f, m = world
    prm = CONFIGS[cfg]
    a, b = handle(flb, f, m, index), handle(flb, f, m, index)
    t = fov_oracle.Tracker(*prm)
    rng = np.random.default_rng(4)
    for k, p in enumerate(trajectory(f, cfg)):
        _, _, nd = a.map_fov_segment(*prm, pos=p)
        wb, _ = t.step(p)
        if len(wb):
            b.map_delete_boxes(wb)
        ma, mb = a.map_download(), b.map_download()
        assert len(ma) == len(mb)
        assert sorted_rows(ma).tobytes() == sorted_rows(mb).tobytes(), k
        if nd > 0 or k in (0, 5):
            assert_same_queries(flb, f, a, b, rng)
    a.close()
    b.close()


@pytest.mark.parametrize("index", list(INDEX))
def test_empty_frames_leave_map_untouched(flb, world, index):
    """Boxes that hold no point: the map bytes, grid and M stay, and the next flb_map_add_scan takes the incremental
    path -- its result is byte-identical to a handle that never ran the tracker."""
    f, m = world
    prm = fov_oracle.SHIPPED
    a, b = handle(flb, f, m, index), handle(flb, f, m, index)
    t = fov_oracle.Tracker(*prm)
    far = np.asarray(f["p_true"], np.float64) + np.array([0.0, 0.0, 1000.0])   # the boxes stay far from every point
    launches = []
    for k in range(6):
        p = far + np.array([0.5 * k, -0.2 * k, 0.1 * k])
        before, info, M = a.map_download(), a.map_grid_info(), a.M
        l0 = a.launch_count()
        boxes, local, nd = a.map_fov_segment(*prm, pos=p)
        launches.append(a.launch_count() - l0)
        wb, wl = t.step(p)
        assert same(boxes, wb) and same(local, wl)
        assert len(boxes) == (0 if k == 0 else 3) and nd == 0
        assert a.M == M and a.map_grid_info() == info and a.map_download().tobytes() == before.tobytes()
    assert set(launches) == {2}                       # the cube step and the flagging kernel
    lprm = flb.capi.lio_params(f, 3)
    info = a.map_grid_info()
    for h in (a, b):
        h.map_add_scan(lprm, 0.3, f["R_true"], f["p_true"])
    assert a.map_grid_info() == b.map_grid_info()
    if index == "dense":                              # the incremental path: the same table over the same box
        assert a.map_grid_info() == info
    assert a.map_download().tobytes() == b.map_download().tobytes()
    a.close()
    b.close()


@pytest.mark.parametrize("index", list(INDEX))
def test_first_call_reset_and_empty_map(flb, world, index):
    f, m = world
    prm = fov_oracle.SHIPPED
    p0 = np.asarray(f["p_true"], np.float64)
    # M = 0: the cube moves, nothing is deleted; it survives the map upload that follows
    a = handle(flb, f, None, index, scan=False)
    t = fov_oracle.Tracker(*prm)
    for k in range(3):
        p = p0 + np.array([0.3 * k, 0.0, 0.0])
        boxes, local, nd = a.map_fov_segment(*prm, pos=p)
        wb, wl = t.step(p)
        assert same(boxes, wb) and same(local, wl) and nd == 0 and a.M == 0
    a.map_upload(m)
    boxes, local, nd = a.map_fov_segment(*prm, pos=p0)
    wb, wl = t.step(p0)
    assert same(boxes, wb) and same(local, wl) and len(wb) == 3 and nd == inside(m, wb).sum()
    # reset: the next call only places the cube, wherever the old one was
    before = a.map_download()
    a.map_fov_reset()
    p1 = p0 + np.array([7.0, -3.0, 0.5])
    boxes, local, nd = a.map_fov_segment(*prm, pos=p1)
    t.reset()
    wb, wl = t.step(p1)
    assert len(boxes) == 0 and nd == 0 and same(local, wl) and a.map_download().tobytes() == before.tobytes()
    boxes, local, nd = a.map_fov_segment(*prm, pos=p1)
    wb, wl = t.step(p1)
    assert same(boxes, wb) and same(local, wl) and len(wb) == 3
    a.close()


@pytest.mark.parametrize("index", list(INDEX))
def test_whole_map_and_argument_errors(flb, world, index):
    f, m = world
    prm = fov_oracle.SHIPPED
    p0 = np.asarray(f["p_true"], np.float64)
    small = m[(np.abs(m - p0) < 8.0).all(1)]           # inside the start cube: frame 2's boxes take all of it
    a = handle(flb, f, small, index)
    t = fov_oracle.Tracker(*prm)
    a.map_fov_segment(*prm, pos=p0)
    t.step(p0)
    before, info = a.map_download(), a.map_grid_info()
    with pytest.raises(flb.FlbError) as e:
        a.map_fov_segment(*prm, pos=p0 + 0.5)
    assert e.value.code == ERR_STATE
    assert a.M == len(small) and a.map_download().tobytes() == before.tobytes() and a.map_grid_info() == info
    # the cube did not move either: the next call (on a larger map) steps from the cube of the first call
    a.map_upload(m)
    p2 = p0 + np.array([1.0, 2.0, -0.5])
    boxes, local, nd = a.map_fov_segment(*prm, pos=p2)
    wb, wl = t.step(p2)
    assert same(boxes, wb) and same(local, wl) and nd == inside(m, wb).sum()
    # arguments
    for bad in [(0.0, 300.0, 1.5), (-20.0, 300.0, 1.5), (np.nan, 300.0, 1.5), (np.inf, 300.0, 1.5), (20.0, 0.0, 1.5),
                (20.0, np.nan, 1.5), (20.0, 300.0, -1.0), (20.0, 300.0, np.inf)]:
        with pytest.raises(flb.FlbError) as e:
            a.map_fov_segment(*bad, pos=p2)
        assert e.value.code == ERR_INVALID, bad
    n = C.c_int()
    assert a.L.flb_map_fov_segment(a.h, None, None, C.byref(n), None, None, None) == ERR_INVALID
    boxes, local, nd = a.map_fov_segment(*prm, pos=p2)     # none of the refusals moved the cube
    wb, wl = t.step(p2)
    assert same(boxes, wb) and same(local, wl)
    a.close()
    b = handle(flb, f, m, index)
    with pytest.raises(flb.FlbError) as e:
        b.map_fov_segment(*prm)                          # NULL pose, no device state
    assert e.value.code == ERR_STATE
    b.close()
