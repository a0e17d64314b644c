"""GPU tier: flb_vmap_reclaim.  The reference frees a Feature when addObservation evicts it and a keyframe image with its
last Feature (src/lidar_selection.cpp:183, :946-957); the device map restates that by compacting the feature array and
reusing keyframe slots.  Nothing may change: selections, patches, errors, map values and VIO results are byte-identical
with and without reclaim; the compacted map is the filtered uncompacted one; on a loitering run the feature array levels
off and most keyframe slots are reused."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GRID = {"T0": 16, "T1": 24}
MAPPING_FRAMES = 12        # frames whose scan feeds flb_vmap_grow; afterwards the site is mapped and frames only observe it


def loiter_sequence(flb, name, n_render=4, step=0.6):
    """A few rendered poses 0.6 m apart (> 0.5 m: every selected point gains an observation per frame, so lists reach
    20 entries and start evicting)."""
    return flb.synth.make_visual_sequence(name, n_render, step=(step, 0.0, 0.0), yaw_step_deg=1.0)


def replay(seq, k):
    """Frame k of the loiter: the rendered poses back and forth (0 1 2 3 2 1 0 1 ...), frame id k."""
    n = len(seq["frames"])
    r = k % (2 * (n - 1))
    return seq["frames"][r if r < n else 2 * (n - 1) - r]


def vio_report_tuple(r):
    return (tuple(r.passes), np.array(r.last_error[:], np.float32).tobytes(), r.rows_total, r.skipped_last, r.cov_updated, r.status)


class Run:
    """One visual-map session through the C ABI: per frame select -> grow -> in-place VIO update -> add_observations."""

    def __init__(self, flb, seq, name, vio=True, stream=None):
        self.flb, self.seq = flb, seq
        self.h = flb.Handle(device=0)
        if stream is not None:
            self.h.set_stream(stream.cuda_stream)
        self.h.camera_set(seq["cam"])
        self.h.image_upload(seq["frames"][0]["image"])
        self.grid = GRID[name]
        self.h.vmap_reset(seq, grid_size=self.grid, outlier_threshold=300.0)
        self.length = (seq["cam"]["width"] // self.grid) * (seq["cam"]["height"] // self.grid)
        f = dict(R_LI=seq["R_LI"], t_LI=seq["t_LI"], Rcl=seq["Rcl"], Pcl=seq["Pcl"], cfg=seq["cfg"])
        self.vprm = flb.capi.vio_params(f, 4) if vio else None
        self.pinned = None            # frame id of the last frame that committed a keyframe slot
        self.commits = 0

    def frame(self, k, reclaim_mid=False, record=True):
        h, fr = self.h, replay(self.seq, k)
        pg = fr["pg"] if k < MAPPING_FRAMES else np.zeros((0, 3), np.float32)
        h.image_upload(fr["image"])
        h.vmap_select(fr["Rcw"], fr["Pcw"], fr["pg_down"], blocking=False)
        out = {}
        if record:
            out["sel"] = h.vmap_selected()
            out["map_value"] = h.vmap_map_value(self.length)
        if reclaim_mid:
            h.vmap_reclaim()
        h.vmap_grow(fr["Rcw"], fr["Pcw"], pg, k)
        if record:
            self._committed(k)
        if self.vprm is not None:
            x0 = self.flb.capi.State18.make(fr["R"] @ self.flb.synth.exp_so3(np.array([0.004, -0.003, 0.002])),
                                            fr["p"] + np.array([0.02, -0.015, 0.01]), cov=self.seq["cov"])
            h.state_upload(x0, x0.copy())
            h.vio_update_enqueue(self.vprm)
        h.vmap_add_observations(fr["Rcw"], fr["Pcw"], k)
        if record:
            self._committed(k)
            if self.vprm is not None:
                x, _, vrep = h.state_download()
                out["state"] = x.vector().copy()
                out["cov"] = np.array(x.cov[:])
                out["vio"] = vio_report_tuple(vrep)
        return out

    def _committed(self, k):
        if self.h.vmap_counts()["last_added"] > 0 and self.pinned != k:
            self.pinned = k
            self.commits += 1

    def close(self):
        self.h.close()


def assert_frames_equal(a, b):
    for fa, fb in zip(a, b):
        for key in ("index", "point", "search_level"):
            assert (fa["sel"][key] == fb["sel"][key]).all()
        for key in ("error", "patch"):
            assert fa["sel"][key].tobytes() == fb["sel"][key].tobytes()
        assert fa["sel"]["pos"].tobytes() == fb["sel"]["pos"].tobytes()
        assert fa["map_value"].tobytes() == fb["map_value"].tobytes()
        assert fa["state"].tobytes() == fb["state"].tobytes() and fa["cov"].tobytes() == fb["cov"].tobytes()
        assert fa["vio"] == fb["vio"]


def filter_dump(d):
    """The dump of a never-reclaimed map as a reclaim leaves it: the features some obs list names, creation order,
    obs remapped by rank."""
    live = np.zeros(len(d["ft_score"]), bool)
    for j in range(len(d["n_obs"])):
        live[d["obs"][j, :d["n_obs"][j]]] = True
    rank = np.concatenate([[0], np.cumsum(live)]).astype(np.int32)
    obs = np.where(d["obs"] >= 0, rank[np.maximum(d["obs"], 0)], -1)
    return dict(pos=d["pos"], value=d["value"], n_obs=d["n_obs"], obs=obs, ft_geo=d["ft_geo"][live], ft_score=d["ft_score"][live],
                ft_level_id_img=d["ft_level_id_img"][live]), live


def assert_dump_is_filtered(h, seq, full, got, exact_geo=True):
    f, _ = filter_dump(full)
    assert (f["pos"] == got["pos"]).all() and f["value"].tobytes() == got["value"].tobytes()
    assert (f["n_obs"] == got["n_obs"]).all() and (f["obs"] == got["obs"]).all()
    assert f["ft_score"].tobytes() == got["ft_score"].tobytes()
    assert (f["ft_level_id_img"][:, :2] == got["ft_level_id_img"][:, :2]).all()
    if exact_geo:
        assert f["ft_geo"].tobytes() == got["ft_geo"].tobytes()
    else:
        np.testing.assert_allclose(got["ft_geo"], f["ft_geo"], rtol=1e-13, atol=1e-13)
    # every surviving feature's slot holds its frame's image, byte for byte
    slot_of = {}
    for fid, slot in got["ft_level_id_img"][:, 1:]:
        assert slot_of.setdefault(int(fid), int(slot)) == int(slot)
    assert len(set(slot_of.values())) == len(slot_of)
    for fid, slot in slot_of.items():
        assert (h.vmap_keyframe(slot) == replay(seq, fid)["image"]).all()
    return slot_of


@pytest.mark.parametrize("name", ["T0", "T1"])
def test_reclaim_changes_nothing(flb, po, name):
    seq = loiter_sequence(flb, name)
    n = 120 if name == "T0" else 60
    A, B, Cr = Run(flb, seq, name), Run(flb, seq, name), Run(flb, seq, name)
    ra, rb, rc = [], [], []
    dead_seen, tails = 0, []
    for k in range(n):
        ra.append(A.frame(k))
        rb.append(B.frame(k))
        dead_seen = max(dead_seen, B.h.vmap_usage()["dead_features"])
        B.h.vmap_reclaim()
        u = B.h.vmap_usage()
        assert u["dead_features"] == 0
        tails.append(u["slots_in_use"] + u["free_slots"])
        rc.append(Cr.frame(k, reclaim_mid=(k == 31)))
        if k % 7 == 6:
            Cr.h.vmap_reclaim()
    assert_frames_equal(ra, rb)
    assert_frames_equal(ra, rc)
    da, db = A.h.vmap_dump(), B.h.vmap_dump()
    # the run exercised the new path: lists full and evicting, dead features reclaimed, slots freed and reused
    assert da["n_obs"].max() == 20 and dead_seen > 0
    ua, ub = A.h.vmap_usage(), B.h.vmap_usage()
    assert ua["dead_features"] > 0 and ub["features"] == ua["features"] - ua["dead_features"]
    if name == "T0":                                               # long enough for whole frames to die
        assert tails[-1] < B.commits                               # fewer slots handed out than frames committed: reuse
        assert ub["slots_in_use"] < ua["slots_in_use"]
    assert_dump_is_filtered(B.h, seq, da, db)
    Cr.h.vmap_reclaim()                                            # C holds the features evicted since its last reclaim
    assert_dump_is_filtered(Cr.h, seq, da, Cr.h.vmap_dump())
    if name == "T0":
        # once against the oracle's restatement (po.VMap: the reference's map, nothing ever freed), same filter
        ovm = po.VMap(seq["cam"], grid_size=GRID[name], outlier_threshold=300.0)
        for k in range(n):
            fr = replay(seq, k)
            ovm.select(fr["image"], fr["Rcw"], fr["Pcw"], fr["pg_down"])
            ovm.grow(fr["image"], fr["Rcw"], fr["Pcw"], fr["pg"] if k < MAPPING_FRAMES else np.zeros((0, 3), np.float32), k)
            ovm.add_observations(fr["image"], fr["Rcw"], fr["Pcw"], k)
        assert_dump_is_filtered(B.h, seq, ovm.dump(), db, exact_geo=False)
    for r in (A, B, Cr):
        r.close()


def test_memory_is_bounded(flb):
    """300 loitering frames: with reclaim every frame the slots in use are exactly the live features' frames plus the
    pinned current one, the feature array stops growing and the slots grow ever more slowly; without reclaim the pool
    grows with every frame."""
    seq = loiter_sequence(flb, "T0")
    n = 300
    R, N = Run(flb, seq, "T0", vio=False), Run(flb, seq, "T0", vio=False)
    caps, in_use = [], []
    for k in range(n):
        R.frame(k)
        N.frame(k)
        R.h.vmap_reclaim()
        d = R.h.vmap_dump()
        u = R.h.vmap_usage()
        frames = set(d["ft_level_id_img"][:, 1].tolist()) | ({R.pinned} if R.pinned is not None else set())
        assert u["slots_in_use"] == len(frames) and u["dead_features"] == 0
        caps.append((u["pool_slots"], u["feature_capacity"]))
        in_use.append(u["slots_in_use"])
        if k > 0 and caps[-1][0] > caps[-2][0]:
            assert prev_free == 0                                    # the pool grows only with no free slot left
        prev_free = u["free_slots"]
    un = N.h.vmap_usage()
    print(f"\nslots in use with reclaim: {in_use[::20]}; capacities {caps[::20]}; without: {un}")
    assert caps[n // 3][1] == caps[-1][1]                              # the feature array levelled off
    assert in_use[-1] - in_use[n // 2] < (n // 2) / 3                  # slots: most frames now reuse a freed one
    assert un["slots_in_use"] >= 0.9 * N.commits and N.commits > 0.9 * n      # without reclaim: one slot per frame
    assert un["slots_in_use"] > 1.5 * in_use[-1] and un["pool_slots"] > caps[-1][0] and un["feature_capacity"] > 2 * caps[-1][1]
    assert R.h.vmap_usage()["device_bytes"] < un["device_bytes"]
    R.close()
    N.close()


def test_reclaim_edge_cases(flb):
    seq = loiter_sequence(flb, "T0")
    r = Run(flb, seq, "T0", vio=False)
    h = r.h
    h.vmap_reclaim()                                                 # empty map
    u = h.vmap_usage()
    assert (u["points"], u["features"], u["dead_features"], u["slots_in_use"], u["free_slots"]) == (0, 0, 0, 0, 0)
    for k in range(300):                                             # until a reclaim leaves free slots
        r.frame(k, record=False)
        h.vmap_reclaim()
        if h.vmap_usage()["free_slots"] > 0:
            break
    d1, u1 = h.vmap_dump(), h.vmap_usage()
    assert u1["free_slots"] > 0
    h.vmap_reclaim()                                                 # a second reclaim in a row is a no-op
    d2, u2 = h.vmap_dump(), h.vmap_usage()
    assert u1 == u2 and all(d1[k].tobytes() == d2[k].tobytes() for k in d1)
    h.vmap_reset(seq, grid_size=GRID["T0"], outlier_threshold=300.0)  # reset clears the free-slot stack
    h.vmap_reclaim()
    u = h.vmap_usage()
    assert (u["points"], u["features"], u["slots_in_use"], u["free_slots"]) == (0, 0, 0, 0)
    assert u["pool_slots"] == u1["pool_slots"]
    c = h.vmap_counts()
    assert (c["points"], c["features"], c["images"]) == (0, 0, 0)
    with pytest.raises(flb.FlbError):
        h.vmap_keyframe(0)                                           # no slot handed out since the reset
    r.close()


def test_reclaim_is_enqueue_only(flb):
    """Reclaim with frames in flight: a fixed number of launches, no host synchronisation (the stream is still busy
    behind a sleeping kernel when it returns), and the same map as the same frames without it."""
    import torch
    seq = loiter_sequence(flb, "T0")
    s = torch.cuda.Stream()
    r, ref = Run(flb, seq, "T0", vio=False, stream=s), Run(flb, seq, "T0", vio=False)
    launches = []
    for k in range(30):
        r.frame(k, record=False)
        ref.frame(k, record=False)
        n0 = r.h.launch_count()
        r.h.vmap_reclaim()
        launches.append(r.h.launch_count() - n0)
    assert len(set(launches)) == 1 and launches[0] == 6
    with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000_000)                              # about a second of device time
    r.h.vmap_reclaim()
    r.h.vmap_reclaim()
    assert not s.query()                                              # neither call waited for the stream
    s.synchronize()
    for k in range(30, 45):                                           # frames keep flowing through the refilled slots
        r.frame(k, record=False)
        r.h.vmap_reclaim()
        ref.frame(k, record=False)
    full = ref.h.vmap_dump()
    assert_dump_is_filtered(r.h, seq, full, r.h.vmap_dump())
    r.close()
    ref.close()


def test_refresh_fills_freed_slots_before_growing(flb):
    """Enqueue-only frames (the host's slot bound runs ahead of the device until it hits the pool's capacity): once a
    reclaim has freed slots, the capacity refresh counts them as room and the pool does not grow."""
    seq = loiter_sequence(flb, "T0")
    r = Run(flb, seq, "T0", vio=False)
    k = 0
    while True:                                                      # until every slot is handed out and some are free again
        r.frame(k, record=False)
        k += 1
        r.h.vmap_reclaim()
        u = r.h.vmap_usage()
        if (u["free_slots"] >= 1 and u["slots_in_use"] + u["free_slots"] == u["pool_slots"]) or k > 400:
            break
    pool0, free0, tail0 = u["pool_slots"], u["free_slots"], u["slots_in_use"] + u["free_slots"]
    assert free0 >= 1 and tail0 == pool0, u
    # enqueue-only: no blocking call until the free slots are used up (the host's bound reaches the capacity on the way)
    for j in range(free0):
        r.frame(k + j, record=False)
    u = r.h.vmap_usage()
    assert u["pool_slots"] == pool0
    assert u["slots_in_use"] + u["free_slots"] == tail0                # every new keyframe went into a freed slot
    r.close()
