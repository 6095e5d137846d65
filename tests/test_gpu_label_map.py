"""GPU: `pvnet_b200.render.render_label_map` (csrc/render.cu, `pvnet_render_label_map`) bit-identical to
oracle/label_map_oracle.py and to single-mesh `render_mesh` depth maps composited in slot order; the
`get_mask_of_all_objects` drop-in against the reference's loop on the `opengl_render_backend` drop-in; run-to-run
identity without host synchronisation; argument errors."""
import math

import numpy as np
import pytest
import torch

from oracle import label_map_oracle as lo
from tests import label_map_cases as lc
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a, dt=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)


def square(half):
    v = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def fronto(b, zs, rng=None):
    P = np.zeros((b, len(zs), 3, 4), np.float32)
    P[:, :, :3, :3] = np.eye(3)
    P[:, :, 2, 3] = zs
    if rng is not None:
        P[:, :, :2, 3] = rng.normal(0, 15, (b, len(zs), 2))
    return P


def small_scene(name):
    """-> meshes, labels, poses [b,M,3,4], K, h, w, near, far, present or None, depth_divisor, max_depth"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "mixed_b3_48x64":
        cube, ico, soup = rc.cube(40.0), rc.icosphere(1, 50.0), rc.soup(30, rng, spread=40.0, size=20.0)
        empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
        meshes = [cube, ico, soup, cube, empty, ico]                       # slots 0 and 3 tie wherever posed alike
        P = np.zeros((3, 6, 3, 4), np.float32)
        for i in range(3):
            for m in range(6):
                P[i, m, :, :3] = rc.rotation(rng)
                P[i, m, :, 3] = (rng.normal(0, 30), rng.normal(0, 30), rng.uniform(600, 900))
            P[i, 3] = P[i, 0]
        Ks = np.stack([rc.camera_for(48, 64, float(rng.uniform(60, 90))) for _ in range(3)])
        present = (rng.random((3, 6)) > 0.2).astype(np.uint8)
        present[:, 0] = present[:, 3] = 1
        return meshes, [9, 4, 200, 17, 1, 255], P, Ks, 48, 64, 10, 10000, present, 1000.0, 10.0
    if name == "ulp_ties_b2_32x40":
        z = np.float32(1001.0)
        while not z / np.float32(1000) == np.nextafter(z, np.float32(np.inf)) / np.float32(1000):
            z = np.nextafter(z, np.float32(np.inf))
        z2 = np.nextafter(z, np.float32(np.inf))
        meshes = [square(200.0), square(200.0), square(100.0)]
        P = fronto(2, [z2, z, 1002.0])
        P[1] = fronto(1, [z, z2, 999.0])[0]
        return meshes, [3, 8, 5], P, rc.camera_for(32, 40, 60.0), 32, 40, 10, 10000, None, 1000.0, 10.0
    if name == "max_depth_edge_b2_24x32":
        z = np.float32(10000.0)
        meshes = [square(3000.0), square(1500.0)]
        P = fronto(2, [z, np.nextafter(z, np.float32(0))])
        P[1, 1, 2, 3] = np.float32(12000.0)
        return meshes, [1, 2], P, rc.camera_for(24, 32, 40.0), 24, 32, 10, 20000, None, 1000.0, 10.0
    if name == "soups_b4_40x52_unit_divisor":
        meshes = [rc.soup(25, rng, spread=50.0, size=30.0) for _ in range(4)]
        P = fronto(4, [700.0, 720.0, 740.0, 760.0], rng)
        for i in range(4):
            for m in range(4):
                P[i, m, :, :3] = rc.rotation(rng)
        return meshes, [10, 20, 30, 40], P, rc.camera_for(40, 52, 70.0), 40, 52, 100, 2000, None, 1.0, math.inf
    raise KeyError(name)


SMALL = ["mixed_b3_48x64", "ulp_ties_b2_32x40", "max_depth_edge_b2_24x32", "soups_b4_40x52_unit_divisor"]


@pytest.mark.parametrize("name", SMALL)
def test_bit_identical_to_oracle(name):
    from pvnet_b200.render import MeshSet, render_label_map
    meshes, labels, P, K, h, w, near, far, present, div, maxd = small_scene(name)
    ms = MeshSet(meshes, labels, device=DEV)
    label, depth = render_label_map(ms, dev(P), dev(K), h, w, near, far,
                                    present=None if present is None else dev(present, torch.uint8),
                                    depth_divisor=div, max_depth=maxd)
    torch.cuda.synchronize()
    ol, od = lo.label_map(meshes, labels, P, K, h, w, near, far, present=present, depth_divisor=div, max_depth=maxd)
    assert np.array_equal(label.cpu().numpy(), ol), name
    assert np.array_equal(depth.cpu().numpy().view(np.int32), od.view(np.int32)), name
    assert (ol != 0).any()
    if name == "ulp_ties_b2_32x40":
        assert (ol[0] == 3).any() and (ol[1] == 3).any()                # the earlier slot keeps the tie both ways
    if name == "max_depth_edge_b2_24x32":
        assert not (ol == 1).any() and (ol[0] == 2).any() and not (ol[1] != 0).any()


def composited_render_mesh(meshes, labels, P, K, present, h, w, near, far, div, maxd):
    """Each slot's depth from render_mesh alone, divided in numpy fp32 (the reference's `render(...) / 1000.`) and
    composited slot by slot as the reference's get_mask_of_all_objects does."""
    from pvnet_b200.render import render_mesh
    b, M = P.shape[:2]
    label = np.zeros((b, h, w), np.uint8)
    depth = np.full((b, h, w), np.float32(maxd), np.float32)
    for m, (v, f) in enumerate(meshes):
        d = render_mesh(dev(v), dev(f, torch.int32), dev(K), dev(P[:, m]), h, w, near, far).cpu().numpy()
        d = d / np.float32(div)
        take = (d != 0) & (d < depth) & (present[:, m] != 0)[:, None, None]
        label[take] = labels[m]
        depth[take] = d[take]
    return label, depth


@pytest.mark.parametrize("b", [1, 13, 64])
def test_bit_identical_to_composited_render_mesh_at_linemod_sizes(b):
    from pvnet_b200.render import MeshSet, render_label_map
    rng = np.random.default_rng(100 + b)
    meshes, labels, P, K, present = lc.scene(b, rng)
    assert all(len(f) == 20480 for _, f in meshes)
    ms = MeshSet(meshes, labels, device=DEV)
    label, depth = render_label_map(ms, dev(P), dev(K), 480, 640, 10, 10000, present=dev(present, torch.uint8),
                                    depth_divisor=1000.0, max_depth=10.0)
    label, depth = label.cpu().numpy(), depth.cpu().numpy()
    wl, wd = composited_render_mesh(meshes, labels, P, K, present, 480, 640, 10, 10000, 1000.0, 10.0)
    assert np.array_equal(label, wl)
    assert np.array_equal(depth.view(np.int32), wd.view(np.int32))
    assert all(len(np.unique(label[i])) >= 3 for i in range(b))         # the objects overlap in every image


def test_get_mask_of_all_objects_dropin_equals_the_reference_loop():
    from pvnet_b200 import render as pr
    indices = list(range(6))
    db = lc.fake_db(indices, np.random.default_rng(5))
    ref_db = lc.fake_db(indices, np.random.default_rng(5))
    type(db).get_mask_of_all_objects = pr.get_mask_of_all_objects
    try:
        for index in indices:
            got = db.get_mask_of_all_objects(index)
            want = lc.reference_loop(ref_db, index)
            assert got.dtype == np.uint8 and got.shape == (480, 640)
            assert np.array_equal(got, want), index
            assert db.class_type == ref_db.class_type == "benchvise"
            assert len(np.unique(got)) >= 4
    finally:
        del type(db).get_mask_of_all_objects
    # colours divided in place once, as the drop-in render does for the models it draws
    for name, _ in lc.OCCLUSION_CLASSES:
        assert np.array_equal(db.opengl_renderer.models[name]["colors"], ref_db.opengl_renderer.models[name]["colors"])
        assert db.opengl_renderer.models[name]["colors"].max() <= 1.0
    # a batch gives the per-index maps, in one device call per chunk, and reuses the uploaded meshes
    cached = pr._mesh_cache[0][3]
    batch = pr.masks_of_all_objects(db, indices, chunk=4)
    assert pr._mesh_cache[0][3] is cached
    assert batch.shape == (6, 480, 640) and batch.dtype == np.uint8
    assert np.array_equal(batch, np.stack([lc.reference_loop(ref_db, i) for i in indices]))


def test_same_output_twice_and_no_host_synchronisation():
    from pvnet_b200.render import MeshSet, render_label_map
    rng = np.random.default_rng(8)
    meshes, labels, P, K, present = lc.scene(16, rng, subdiv=4)
    ms = MeshSet(meshes, labels, device=DEV)
    Pd, Kd, pd = dev(P), dev(K), dev(present, torch.uint8)
    render_label_map(ms, Pd, Kd, 480, 640, 10, 10000, present=pd, depth_divisor=1000.0, max_depth=10.0)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = render_label_map(ms, Pd, Kd, 480, 640, 10, 10000, present=pd, depth_divisor=1000.0, max_depth=10.0)
        b = render_label_map(ms, Pd, Kd, 480, 640, 10, 10000, present=pd, depth_divisor=1000.0, max_depth=10.0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert (a[0] > 0).float().mean() > 0.02


def test_argument_errors():
    from pvnet_b200.render import MeshSet, render_label_map
    v, f = rc.cube(50.0)
    ms = MeshSet([(v, f), (v, f)], [1, 2], device=DEV)
    P = dev(fronto(3, [600.0, 700.0]))
    K = dev(rc.camera_for(48, 64))
    ok = dict(mesh_set=ms, poses=P, K=K, h=48, w=64, near=10, far=10000)
    bad = [dict(mesh_set=[(v, f)]), dict(poses=P[:, :1]), dict(poses=P[:, :, :, :3]), dict(poses=P[:0]),
           dict(K=torch.stack([K] * 2)), dict(h=0), dict(near=0), dict(near=20000), dict(depth_divisor=0.0),
           dict(depth_divisor=math.inf), dict(depth_divisor=-2.0), dict(max_depth=0.0), dict(max_depth=math.nan),
           dict(near=1e-30, depth_divisor=1e30), dict(present=torch.ones(3, 3, dtype=torch.uint8, device=DEV)),
           dict(poses=P.cpu().numpy())]
    for kw in bad:
        with pytest.raises(ValueError):
            render_label_map(**{**ok, **kw})
    with pytest.raises(RuntimeError):
        render_label_map(**{**ok, "poses": P.cpu()})
    with pytest.raises(RuntimeError):
        render_label_map(**{**ok, "present": torch.ones(3, 2, dtype=torch.bool)})
    label, depth = render_label_map(**ok, present=torch.ones(3, 2, dtype=torch.bool, device=DEV))
    assert label.shape == depth.shape == (3, 48, 64) and label.dtype == torch.uint8
