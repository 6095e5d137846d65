"""CPU: the label-map contract of DESIGN.md §25 in oracle/label_map_oracle.py on analytic scenes of fronto-parallel
squares, its compositing against the reference's own `get_mask_of_all_objects` (tests/golden/ref_label_map.npz),
the host-side pose conversion of `pvnet_b200.render.occlusion_poses`, and the argument errors of `MeshSet` and of
`pvnet_render_label_map`'s host checks."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import label_map_oracle as lo
from oracle import render_oracle as ro
from tests import label_map_cases as lc
from tests.helpers import GOLDEN

H, W = 24, 32
K = np.array([[40.0, 0, 16.0], [0, 40.0, 12.0], [0, 0, 1]], np.float32)


def square(half):
    v = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def poses_at(*zs, x=()):
    """one image, a fronto-parallel pose per slot at depth zs[m] (and x offset x[m])"""
    P = np.zeros((1, len(zs), 3, 4), np.float32)
    for m, z in enumerate(zs):
        P[0, m, :, :3] = np.eye(3)
        P[0, m, :, 3] = (x[m] if x else 0.0, 0.0, z)
    return P


def covered(z, half=100.0):
    """the pixels a square of half-width `half` at depth z covers, from the oracle's single-mesh render"""
    v, f = square(half)
    d = ro.render(v, f, K, poses_at(z)[0], H, W, 10, 20000)[0][0]
    return d > 0


def test_nearer_object_wins_in_either_slot_order():
    big, small = square(200.0), square(60.0)
    for order in ((big, small, 900.0, 700.0, 3, 5), (small, big, 700.0, 900.0, 5, 3)):
        m0, m1, z0, z1, l0, l1 = order
        label, depth = lo.label_map([m0, m1], [l0, l1], poses_at(z0, z1), K, H, W, 10, 20000)
        near = covered(700.0, 60.0)
        assert near.any() and (label[0][near] == 5).all() and (depth[0][near] == np.float32(700.0)).all()
        rest = covered(900.0, 200.0) & ~near
        assert rest.any() and (label[0][rest] == 3).all() and (depth[0][rest] == np.float32(900.0)).all()
        assert (label[0][~(near | rest)] == 0).all() and np.isinf(depth[0][~(near | rest)]).all()


def test_equal_depth_goes_to_the_earlier_slot():
    v, f = square(100.0)
    for labels in ([7, 2], [2, 7]):
        label, _ = lo.label_map([(v, f), (v, f)], labels, poses_at(800.0, 800.0), K, H, W, 10, 20000)
        cov = covered(800.0)
        assert cov.any() and (label[0][cov] == labels[0]).all()


def ulp_pair_equal_after_division(divisor=np.float32(1000.0)):
    """two fp32 depths near 1 m, one ulp apart, whose quotients by 1000 are the same fp32 value"""
    z = np.float32(1001.0)
    while True:
        z2 = np.nextafter(z, np.float32(np.inf))
        if z / divisor == z2 / divisor:
            return z, z2
        z = z2


def test_depths_that_differ_in_z_but_divide_to_the_same_value_go_to_the_earlier_slot():
    z, z2 = ulp_pair_equal_after_division()
    assert z != z2
    v, f = square(100.0)
    for zs in ((z, z2), (z2, z)):                                   # the earlier slot wins, nearer in Z or not
        label, depth = lo.label_map([(v, f), (v, f)], [4, 9], poses_at(*zs), K, H, W, 10, 20000,
                                    depth_divisor=1000.0)
        cov = covered(z)
        assert cov.any() and (label[0][cov] == 4).all() and (depth[0][cov] == z / np.float32(1000)).all()
    # divided by 1 the nearer one wins
    label, _ = lo.label_map([(v, f), (v, f)], [4, 9], poses_at(z2, z), K, H, W, 10, 20000)
    assert (label[0][covered(z)] == 9).all()


def test_an_object_exactly_at_max_depth_after_division_is_excluded():
    v, f = square(2000.0)
    for z, want in ((np.float32(10000.0), 0), (np.nextafter(np.float32(10000.0), np.float32(0)), 6)):
        label, depth = lo.label_map([(v, f)], [6], poses_at(z), K, H, W, 10, 20000, depth_divisor=1000.0,
                                    max_depth=10.0)
        cov = covered(z, 2000.0)
        assert cov.any() and (label[0][cov] == want).all()
        assert (depth[0][cov] == (np.float32(10) if want == 0 else z / np.float32(1000))).all()
        assert (depth[0][~cov] == np.float32(10)).all()


def test_absent_slots_and_empty_meshes_draw_nothing():
    v, f = square(100.0)
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    P = np.concatenate([poses_at(600.0, 700.0, 800.0)] * 2)
    present = np.array([[0, 1, 1], [1, 1, 0]], np.uint8)
    label, _ = lo.label_map([(v, f), empty, (v, f)], [1, 2, 3], P, K, H, W, 10, 20000, present=present)
    assert covered(800.0).any() and (label[0][covered(800.0)] == 3).all() and (label[1][covered(600.0)] == 1).all()
    assert (label[0][~covered(800.0)] == 0).all() and (label[1][~covered(600.0)] == 0).all()
    assert not (label == 2).any()


def test_one_mesh_gives_the_single_mesh_render():
    rng = np.random.default_rng(3)
    from tests import render_cases as rc
    v, f = rc.icosphere(1, 60.0)
    P = rc.poses(3, rng)
    label, depth = lo.label_map([(v, f)], [200], P[:, None], K, H, W, 100, 2000)
    for i in range(3):
        d = ro.render(v, f, K, P[i:i + 1], H, W, 100, 2000)[0][0]
        assert d.max() > 0
        assert np.array_equal(label[i] == 200, d > 0) and not ((label[i] != 0) & (label[i] != 200)).any()
        assert np.array_equal(depth[i][d > 0].view(np.int32), d[d > 0].view(np.int32))
        assert np.isinf(depth[i][d == 0]).all()


def test_compositing_matches_the_reference_method_on_recorded_cases():
    z = np.load(os.path.join(GOLDEN, "ref_label_map.npz"))
    labels = [int(n) for _, n in lc.OCCLUSION_CLASSES]
    ties = 0
    for case in range(lc.GOLDEN_CASES):
        maps = lc.golden_depth_maps(case)
        depths = np.stack([np.zeros((lc.H, lc.W), np.float32) if d is None else d for _, d in maps])
        label, depth = lo.composite(depths, labels, max_depth=10.0)
        assert np.array_equal(label, z[f"case{case}"]), case
        assert ((depth < 10) == (label != 0)).all()
        # the recipe exercises what it is for: equal depths of two objects at one pixel, and missing poses
        d = np.where(depths > 0, depths, np.nan)
        ties += int(sum(((d[i] == d[j]) & (d[i] < 10)).sum() for i in range(9) for j in range(i)))
    assert ties > 1000
    assert sum(d is None for case in range(lc.GOLDEN_CASES) for _, d in lc.golden_depth_maps(case)) > 3


class PoseDB:
    class_type_to_number = dict(lc.OCCLUSION_CLASSES)

    def __init__(self, poses):
        self.poses = poses
        self.class_type = None
        self.seen = []

    def read_blender_pose(self, index):
        self.seen.append((self.class_type, index))
        return self.poses.get((self.class_type, index), np.array([]))


def test_pose_conversion_follows_the_renderer_in_the_poses_own_dtype():
    from pvnet_b200.render import occlusion_poses
    rng = np.random.default_rng(9)
    poses = {}
    for index in (4, 11):
        for k, (name, _) in enumerate(lc.OCCLUSION_CLASSES):
            if (k + index) % 4 == 0:
                continue
            t = rng.normal(0, 0.3, (3, 1)) + [[0], [0], [0.8]]
            p = np.concatenate([np.linalg.qr(rng.normal(size=(3, 3)))[0], t], 1)
            poses[(name, index)] = p.astype(np.float32) if name == "benchvise" else p
    db = PoseDB(poses)
    P, present = occlusion_poses(db, [4, 11])
    assert P.dtype == np.float32 and P.shape == (2, 9, 3, 4) and present.shape == (2, 9)
    assert db.seen == [(n, i) for i in (4, 11) for n, _ in lc.OCCLUSION_CLASSES]
    assert db.class_type == "benchvise"
    for j, index in enumerate((4, 11)):
        for k, (name, _) in enumerate(lc.OCCLUSION_CLASSES):
            p = poses.get((name, index))
            assert present[j, k] == (p is not None)
            if p is None:
                assert not P[j, k].any()
                continue
            t = p[:, 3:] * 1000.                                     # float32 stays float32, float64 stays float64
            assert t.dtype == p.dtype
            assert np.array_equal(P[j, k, :, :3], p[:, :3].astype(np.float32))
            assert np.array_equal(P[j, k, :, 3:], t.astype(np.float32))


def test_mesh_set_argument_errors():
    from pvnet_b200.render import MeshSet
    v, f = square(10.0)
    dev = "cuda:0"                                                  # every check below runs before the device is used
    bad = [([], []), ([(v, f)] * 256, [1] * 256), ([(v, f)], [0]), ([(v, f)], [256]), ([(v, f)] * 2, [1]),
           ([(v[:, :2], f)], [1]), ([(v, f[:, :2])], [1]), ([(v, f.astype(np.float32))], [1])]
    for meshes, labels in bad:
        with pytest.raises(ValueError):
            MeshSet(meshes, labels, device=dev)
    with pytest.raises(RuntimeError):
        MeshSet([(v, f)], [1], device="cpu")


def test_native_host_checks_reject_bad_arguments():
    from pvnet_b200 import _native
    L = _native.lib()
    dummy = ctypes.c_void_p(16)                                     # never dereferenced: every call below is refused

    def call(M=2, labels=(1, 2), nf=4, near=10.0, far=100.0, div=1000.0, maxd=10.0, table=dummy, poses=dummy,
             label=dummy, ws_bytes=1 << 20, b=1, h=8, w=8):
        lab = (ctypes.c_uint8 * max(len(labels), 1))(*labels)
        return L.pvnet_render_label_map(dummy, dummy, table, lab, M, nf, poses, None, dummy, 0, b, h, w, near, far,
                                        div, maxd, label, None, dummy, ws_bytes, None)

    cases = [dict(M=0), dict(M=256, labels=(1,) * 256), dict(labels=(1, 0)), dict(div=0.0), dict(div=-1.0),
             dict(div=math.inf), dict(div=math.nan), dict(maxd=0.0), dict(maxd=-1.0), dict(maxd=math.nan),
             dict(near=1e-30, div=1e30), dict(near=0.0), dict(near=200.0), dict(table=None), dict(poses=None),
             dict(label=None), dict(ws_bytes=8 * 64 - 1), dict(nf=-1), dict(b=0), dict(b=2 ** 20, nf=2 ** 12)]
    for kw in cases:
        assert call(**kw) == -1, kw
        assert L.pvnet_last_error()
