"""GPU tier: the device map's maintenance chain pinned to fixed values.  On the dense cell table and on the sparse index,
a seeded sequence -- map upload, Add_Points inside the grid box, flb_map_add_scan at an explicit pose, a local-map cube
trajectory that deletes part of the map, Add_Points again, and a batch outside the dense grid box (the full path there)
-- must give, after every step, the launch count, the grid description, the map bytes (flb_map_download's order) and
the kNN answers recorded here.  The other map tests compare two handles running the same code or compare row sets;
this one catches any change to the order or the launches of the merge itself.

The map is the frame's room (every 4th point) plus the translated copies of test_gpu_fov_segment, so that the shipped
cube cuts real slabs without ever taking the whole map."""
import hashlib

import numpy as np
import pytest

import fov_oracle
from golden_util import world_scan
from test_gpu_fov_segment import OFFS, trajectory

pytestmark = pytest.mark.gpu


def digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).hexdigest()[:16]


def run_chain(flb, name, index):
    """[(step, launches, n_deleted or None, grid info, map digest, kNN digest)] after every step of the sequence."""
    f = flb.synth.make_frame(name)
    m = np.concatenate([f["map_xyz"][::4] + np.array(o, np.float32) for o in OFFS]).astype(np.float32)
    rng = np.random.default_rng(11)
    q = (m[rng.integers(0, len(m), 2000)] + rng.normal(0, 0.3, (2000, 3))).astype(np.float32)
    new = world_scan(f)
    lprm = flb.capi.lio_params(f, 3)
    h = flb.Handle(device=0, cell_size=f["cfg"].cell_size)
    h.debug_set_map_index(index)
    out = []

    def step(label, fn):
        l0 = h.launch_count()
        r = fn()
        launches = h.launch_count() - l0
        info = h.map_grid_info()
        idx, d2 = h.knn(q)
        out.append((label, launches, r, (info["cell_size"], info["sparse"], info["cells"], info["index_bytes"]),
                    digest(h.map_download()), digest(idx, d2)))

    step("upload", lambda: h.map_upload(m))
    h.scan_upload(f["scan_body"])
    step("add_points", lambda: h.map_add_points(new + rng.normal(0, 0.02, new.shape).astype(np.float32), 0.3))
    step("add_scan", lambda: h.map_add_scan(lprm, 0.3, f["R_true"], f["p_true"] + np.array([0.05, -0.03, 0.02])))
    for k, p in enumerate(trajectory(f, "shipped", n=8)):
        step(f"fov{k}", lambda: h.map_fov_segment(*fov_oracle.SHIPPED, pos=p)[2])
    step("add_points_2", lambda: h.map_add_points(
        rng.uniform(f["map_xyz"].min(0), f["map_xyz"].max(0), (len(new) // 4, 3)).astype(np.float32), 0.3))
    step("add_points_far", lambda: h.map_add_points(new + np.array([2000.0, 0.0, 0.0], np.float32), 0.3))
    h.close()
    return out


EXPECTED = {    # recorded on an H100 80GB HBM3; (step, launches, n_deleted, (cell_size, sparse, cells, index_bytes), map, kNN)
    ('T1', 1): [
        ('upload', 7, None, (1.9054781198501587, 0, 20227000, 80908004), '0693720d885b8ca0', 'ade032af06ea852c'),
        ('add_points', 14, None, (1.9054781198501587, 0, 20227000, 80908004), '866dae3d4ba32ab3', '2803310ab6155ad3'),
        ('add_scan', 15, None, (1.9054781198501587, 0, 20227000, 80908004), 'f13cf81161eca89b', '839a558704e09476'),
        ('fov0', 2, 0, (1.9054781198501587, 0, 20227000, 80908004), 'f13cf81161eca89b', '839a558704e09476'),
        ('fov1', 8, 5410, (1.9054781198501587, 0, 20227000, 80908004), 'cf858a42decf3b1d', 'afd4864136318dcb'),
        ('fov2', 8, 4551, (1.9054781198501587, 0, 20227000, 80908004), 'd21db15ea605dde5', '835e6e3274551a32'),
        ('fov3', 8, 4551, (1.9054781198501587, 0, 20227000, 80908004), 'c8d4318e63a0edbb', 'e7fb438976a8ea28'),
        ('fov4', 2, 0, (1.9054781198501587, 0, 20227000, 80908004), 'c8d4318e63a0edbb', 'e7fb438976a8ea28'),
        ('fov5', 2, 0, (1.9054781198501587, 0, 20227000, 80908004), 'c8d4318e63a0edbb', 'e7fb438976a8ea28'),
        ('fov6', 2, 0, (1.9054781198501587, 0, 20227000, 80908004), 'c8d4318e63a0edbb', 'e7fb438976a8ea28'),
        ('fov7', 2, 0, (1.9054781198501587, 0, 20227000, 80908004), 'c8d4318e63a0edbb', 'e7fb438976a8ea28'),
        ('add_points_2', 14, None, (1.9054781198501587, 0, 20227000, 80908004), '8f9b2f15475b629f', '9813d61efa42e6d9'),
        ('add_points_far', 17, None, (3.025137186050415, 0, 28501425, 114005704), '8d520ee32544c741', '0e726ffa42bf1a04'),
    ],
    ('T1', 2): [
        ('upload', 9, None, (0.6000000238418579, 1, 29120, 1048576), '0693720d885b8ca0', 'ade032af06ea852c'),
        ('add_points', 16, None, (0.6000000238418579, 1, 29589, 1048576), '24aaa0cdda183567', 'cfad3fb0451a0f53'),
        ('add_scan', 17, None, (0.6000000238418579, 1, 29615, 1048576), '9a40022de93194bc', '11a3ef7f9d03f1b5'),
        ('fov0', 2, 0, (0.6000000238418579, 1, 29615, 1048576), '9a40022de93194bc', '11a3ef7f9d03f1b5'),
        ('fov1', 10, 5410, (0.6000000238418579, 1, 25908, 1048576), '7cfc2064b4be5af5', '54a4bf094979e898'),
        ('fov2', 10, 4551, (0.6000000238418579, 1, 22387, 1048576), 'fd40628598f456b8', 'ec4d5d926d67b2d1'),
        ('fov3', 10, 4551, (0.6000000238418579, 1, 18866, 1048576), '95421e84ec1e0238', 'ce57914dcdeb7fab'),
        ('fov4', 2, 0, (0.6000000238418579, 1, 18866, 1048576), '95421e84ec1e0238', 'ce57914dcdeb7fab'),
        ('fov5', 2, 0, (0.6000000238418579, 1, 18866, 1048576), '95421e84ec1e0238', 'ce57914dcdeb7fab'),
        ('fov6', 2, 0, (0.6000000238418579, 1, 18866, 1048576), '95421e84ec1e0238', 'ce57914dcdeb7fab'),
        ('fov7', 2, 0, (0.6000000238418579, 1, 18866, 1048576), '95421e84ec1e0238', 'ce57914dcdeb7fab'),
        ('add_points_2', 16, None, (0.6000000238418579, 1, 19588, 1048576), 'ef7c78f0a94526a2', '2877d01237337ae9'),
        ('add_points_far', 16, None, (0.6000000238418579, 1, 20553, 1048576), '74c2fab3c6ce86d5', '4536ed5da2ddcbff'),
    ],
    ('C2', 1): [
        ('upload', 7, None, (1.9054781198501587, 0, 25679877, 102719512), '25ac04631ef4cec0', '444e7b8a09b2a05e'),
        ('add_points', 14, None, (1.9054781198501587, 0, 25679877, 102719512), 'e39b2cbd4dc79893', '8657a66eb35837f5'),
        ('add_scan', 15, None, (1.9054781198501587, 0, 25679877, 102719512), 'f0bd7e174c0135f2', 'e28d44cda4cbd265'),
        ('fov0', 2, 0, (1.9054781198501587, 0, 25679877, 102719512), 'f0bd7e174c0135f2', 'e28d44cda4cbd265'),
        ('fov1', 8, 14292, (1.9054781198501587, 0, 25679877, 102719512), 'b3db8be97da4d9d1', '0b46fd53b265b5c9'),
        ('fov2', 8, 9938, (1.9054781198501587, 0, 25679877, 102719512), 'd75aec0175c8db59', '7c6c2e798fef2caa'),
        ('fov3', 8, 9938, (1.9054781198501587, 0, 25679877, 102719512), '09cf85f5b8e8c4ad', 'bc74638ffe2cbf3d'),
        ('fov4', 2, 0, (1.9054781198501587, 0, 25679877, 102719512), '09cf85f5b8e8c4ad', 'bc74638ffe2cbf3d'),
        ('fov5', 2, 0, (1.9054781198501587, 0, 25679877, 102719512), '09cf85f5b8e8c4ad', 'bc74638ffe2cbf3d'),
        ('fov6', 2, 0, (1.9054781198501587, 0, 25679877, 102719512), '09cf85f5b8e8c4ad', 'bc74638ffe2cbf3d'),
        ('fov7', 2, 0, (1.9054781198501587, 0, 25679877, 102719512), '09cf85f5b8e8c4ad', 'bc74638ffe2cbf3d'),
        ('add_points_2', 14, None, (1.9054781198501587, 0, 25679877, 102719512), '05ff447b32670c9a', 'e41916b373a23ae6'),
        ('add_points_far', 17, None, (3.025137186050415, 0, 31277270, 125109084), 'b422a810ac732677', 'c2ccc3540e2f442c'),
    ],
    ('C2', 2): [
        ('upload', 9, None, (0.6000000238418579, 1, 231724, 8388608), '25ac04631ef4cec0', '444e7b8a09b2a05e'),
        ('add_points', 16, None, (0.6000000238418579, 1, 233969, 8388608), '7edc1667de2cbfb9', '141e13c57244d832'),
        ('add_scan', 17, None, (0.6000000238418579, 1, 234035, 8388608), 'c3a645863e9b2ec9', '6b911830703afc3e'),
        ('fov0', 2, 0, (0.6000000238418579, 1, 234035, 8388608), 'c3a645863e9b2ec9', '6b911830703afc3e'),
        ('fov1', 10, 14292, (0.6000000238418579, 1, 225632, 8388608), '3d7ba605f7bd94b0', 'b1a53aa735e03c14'),
        ('fov2', 10, 9938, (0.6000000238418579, 1, 218012, 8388608), '0d0276857b951f3e', 'c37a4e8cd5de8323'),
        ('fov3', 10, 9938, (0.6000000238418579, 1, 210393, 8388608), '36b26ac2df3c6f9e', '43d23a22a0ac2b27'),
        ('fov4', 2, 0, (0.6000000238418579, 1, 210393, 8388608), '36b26ac2df3c6f9e', '43d23a22a0ac2b27'),
        ('fov5', 2, 0, (0.6000000238418579, 1, 210393, 8388608), '36b26ac2df3c6f9e', '43d23a22a0ac2b27'),
        ('fov6', 2, 0, (0.6000000238418579, 1, 210393, 8388608), '36b26ac2df3c6f9e', '43d23a22a0ac2b27'),
        ('fov7', 2, 0, (0.6000000238418579, 1, 210393, 8388608), '36b26ac2df3c6f9e', '43d23a22a0ac2b27'),
        ('add_points_2', 16, None, (0.6000000238418579, 1, 215892, 8388608), '441f8f83c76d4f24', '3ba6f7c3f7defc81'),
        ('add_points_far', 16, None, (0.6000000238418579, 1, 221231, 8388608), 'fb39cf6c89642b2b', '052248b346881b3b'),
    ],
}


@pytest.mark.parametrize("index", [1, 2], ids=["dense", "sparse"])
@pytest.mark.parametrize("name", ["T1", "C2"])
def test_map_chain_pinned(flb, name, index):
    got = run_chain(flb, name, index)
    exp = EXPECTED[name, index]
    assert len(got) == len(exp)
    for g, e in zip(got, exp):
        assert g == e, g[0]
