"""GPU: `pvnet_b200.render.render_mesh` (csrc/render.cu) bit-identical to oracle/render_oracle.py in depth, RGB and
coverage, run to run, without host synchronisation; the `lib.utils.opengl_render_backend` drop-in against it."""
import numpy as np
import pytest
import torch

from oracle import render_oracle as ro
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def colors_for(nv, seed):
    return np.random.default_rng(seed).uniform(0, 1, (nv, 3)).astype(np.float32)


def scene(name):
    """-> verts, faces, K ([3,3] or [b,3,3]), poses [b,3,4], h, w, near, far, colors, images the oracle checks"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "icosphere_b1_480x640":
        v, f = rc.icosphere(2, 90.0)
        return v, f, rc.K_LINEMOD, rc.poses(1, rng), 480, 640, 100, 2000, colors_for(len(v), 1), None
    if name == "icosphere_b64_480x640":
        v, f = rc.icosphere(1, 70.0)
        return v, f, rc.K_LINEMOD, rc.poses(64, rng), 480, 640, 100, 2000, colors_for(len(v), 2), [0, 31, 63]
    if name == "cube_b13_per_image_k_61x47":
        v, f = rc.cube(50.0)
        Ks = np.stack([rc.camera_for(61, 47, float(rng.uniform(40, 90))) for _ in range(13)])
        Ks[:, 0, 1] = rng.normal(0, 2, 13)                                  # skew
        Ks[:, :2, 2] += rng.normal(0, 3, (13, 2))
        return v, f, Ks.astype(np.float32), rc.poses(13, rng), 61, 47, 100, 2000, colors_for(8, 3), None
    if name == "soup_b13_96x128":
        v, f = rc.soup(200, rng)
        return v, f, rc.camera_for(96, 128, 150.0), rc.poses(13, rng), 96, 128, 100, 2000, colors_for(len(v), 4), None
    if name == "cube_b64_tiny_sizes":
        v, f = rc.cube(50.0)
        return v, f, rc.camera_for(1, 1, 2.0), rc.poses(64, rng), 1, 1, 100, 2000, None, None
    if name == "cube_b64_1x7":
        v, f = rc.cube(50.0)
        return v, f, rc.camera_for(1, 7, 8.0), rc.poses(64, rng), 1, 7, 100, 2000, colors_for(8, 5), None
    if name == "cube_b13_7x1":
        v, f = rc.cube(50.0)
        return v, f, rc.camera_for(7, 1, 8.0), rc.poses(13, rng), 7, 1, 100, 2000, colors_for(8, 6), None
    if name == "quad_fills_frame_480x640":
        v = np.array([[-2000, -2000, 0], [2000, -2000, 0], [2000, 2000, 0], [-2000, 2000, 0]], np.float32)
        f = np.array([[0, 1, 2], [2, 3, 0]], np.int32)
        P = np.zeros((1, 3, 4), np.float32)
        P[0, :, :3] = np.eye(3)
        P[0, :, 3] = (10.0, -5.0, 700.0)
        return v, f, rc.K_LINEMOD, P, 480, 640, 100, 2000, colors_for(4, 7), None
    if name == "subpixel_faces_b13_480x640":
        v, f = rc.icosphere(2, 1.5)
        sv, sf = rc.soup(60, rng, spread=40.0, size=0.3)
        verts = np.concatenate([v, sv])
        faces = np.concatenate([f, sf + len(v)])
        return verts, faces, rc.K_LINEMOD, rc.poses(13, rng), 480, 640, 100, 2000, colors_for(len(verts), 8), [5]
    if name == "behind_and_crossing_camera_60x80":
        v, f = rc.soup(60, rng, spread=150.0, size=120.0)
        P = np.zeros((5, 3, 4), np.float32)
        for i in range(5):
            P[i, :, :3] = rc.rotation(rng)
            P[i, :, 3] = (0, 0, 60.0 * i - 60.0)                           # the soup straddles Z = 0 and near
        return v, f, rc.camera_for(60, 80, 50.0), P, 60, 80, 10, 400, colors_for(len(v), 9), None
    raise KeyError(name)


SCENES = ["icosphere_b1_480x640", "icosphere_b64_480x640", "cube_b13_per_image_k_61x47", "soup_b13_96x128",
          "cube_b64_tiny_sizes", "cube_b64_1x7", "cube_b13_7x1", "quad_fills_frame_480x640",
          "subpixel_faces_b13_480x640", "behind_and_crossing_camera_60x80"]


def device_inputs(v, f, K, P, colors):
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt)  # noqa: E731
    return (t(v, torch.float32), t(f, torch.int32), t(K, torch.float32), t(P, torch.float32),
            None if colors is None else t(colors, torch.float32))


@pytest.mark.parametrize("name", SCENES)
def test_bit_identical_to_oracle(name):
    v, f, K, P, h, w, near, far, colors, check = scene(name)
    vd, fd, Kd, Pd, cd = device_inputs(v, f, K, P, colors)
    amb, bg = 0.35, (0.1, 0.25, 0.9)
    rgb, depth = render_mesh_call(vd, fd, Kd, Pd, h, w, near, far, cd, "rgb+depth", amb, bg)
    depth_only = render_mesh_call(vd, fd, Kd, Pd, h, w, near, far, cd, "depth", amb, bg)
    rgb_only = render_mesh_call(vd, fd, Kd, Pd, h, w, near, far, cd, "rgb", amb, bg)
    torch.cuda.synchronize()
    depth, rgb = depth.cpu().numpy(), rgb.cpu().numpy()
    assert np.array_equal(depth_only.cpu().numpy().view(np.int32), depth.view(np.int32))
    assert np.array_equal(rgb_only.cpu().numpy(), rgb)
    b = P.shape[0]
    for i in (range(b) if check is None else check):
        Ki = K if K.ndim == 2 else K[i]
        od, orgb, win = ro.render(v, f, Ki, P[i:i + 1], h, w, near, far, colors=colors, ambient=amb, bg=bg)
        assert np.array_equal(depth[i] > 0, win[0] >= 0), (name, i)
        assert np.array_equal(depth[i].view(np.int32), od[0].view(np.int32)), (name, i)
        assert np.array_equal(rgb[i], orgb[0]), (name, i)
    if name not in ("cube_b64_tiny_sizes", "behind_and_crossing_camera_60x80"):
        assert (depth > 0).any()


def render_mesh_call(*args):
    from pvnet_b200.render import render_mesh
    return render_mesh(*args[:8], colors=args[8], mode=args[9], ambient_weight=args[10], bg_color=args[11])


def test_same_output_twice_and_no_host_synchronisation():
    from pvnet_b200.render import render_mesh
    rng = np.random.default_rng(21)
    v, f = rc.icosphere(4, 90.0)
    vd, fd, Kd, Pd, cd = device_inputs(v, f, np.stack([rc.K_LINEMOD] * 16), rc.poses(16, rng), colors_for(len(v), 1))
    render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, colors=cd, mode="rgb+depth")      # warm the allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, colors=cd, mode="rgb+depth")
        b = render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, colors=cd, mode="rgb+depth")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert (a[1] > 0).float().mean() > 0.05


def test_dropin_equals_render_mesh_with_in_place_colour_division():
    from lib.utils import opengl_render_backend as ob
    from pvnet_b200.render import render_mesh
    rng = np.random.default_rng(4)
    v, f = rc.icosphere(2, 80.0)
    cols255 = rng.uniform(0, 255, (len(v), 3))
    model = {"pts": v, "faces": f, "colors": cols255.copy()}
    P = rc.poses(1, rng)
    R, t = P[0, :, :3], P[0, :, 3:].astype(np.float64)                      # t as [3,1]
    K = rc.K_LINEMOD.astype(np.float64)
    rgb1, d1 = ob.render(model, [640, 480], K, R, t, ambient_weight=0.4)
    assert np.array_equal(model["colors"], cols255 / 255.0)                 # divided in place
    rgb2, d2 = ob.render(model, [640, 480], K, R, t, ambient_weight=0.4)   # max <= 1 now: not divided again
    assert np.array_equal(model["colors"], cols255 / 255.0)
    assert np.array_equal(rgb1, rgb2) and np.array_equal(d1.view(np.int32), d2.view(np.int32))
    vd, fd, Kd, Pd, cd = device_inputs(v, f, rc.K_LINEMOD, P, (cols255 / 255.0).astype(np.float32))
    rgb, depth = render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, colors=cd, mode="rgb+depth", ambient_weight=0.4)
    assert rgb1.dtype == np.uint8 and rgb1.shape == (480, 640, 3) and d1.dtype == np.float32 and d1.shape == (480, 640)
    assert np.array_equal(rgb1, rgb[0].cpu().numpy())
    assert np.array_equal(d1.view(np.int32), depth[0].cpu().numpy().view(np.int32))
    # the depth mode divides as well
    model = {"pts": v, "faces": f, "colors": cols255.copy()}
    d3 = ob.render(model, [640, 480], K, R, t[:, 0], mode="depth")
    assert np.array_equal(model["colors"], cols255 / 255.0) and np.array_equal(d3, d1)
    # surf_color and bg_color; no colours gives 0.5 grey
    model = {"pts": v, "faces": f}
    rgb_s = ob.render(model, [640, 480], K, R, t, surf_color=(0.2, 0.7, 0.1), bg_color=(0.3, 0.0, 1.0, 1.0),
                      mode="rgb")
    want = render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, mode="rgb", bg_color=(0.3, 0.0, 1.0),
                       colors=torch.tensor([[0.2, 0.7, 0.1]], device=DEV).expand(len(v), 3).contiguous())
    assert np.array_equal(rgb_s, want[0].cpu().numpy())
    assert (rgb_s[depth[0].cpu().numpy() == 0] == ro.to_u8(np.float32([0.3, 0.0, 1.0]))).all()
    grey = ob.render(model, [640, 480], K, R, t, mode="rgb")
    want = render_mesh(vd, fd, Kd, Pd, 480, 640, 100, 2000, mode="rgb")
    assert np.array_equal(grey, want[0].cpu().numpy())


def test_dropin_errors():
    from lib.utils import opengl_render_backend as ob
    v, f = rc.cube(50.0)
    model = {"pts": v, "faces": f}
    args = (model, [64, 48], rc.camera_for(48, 64), np.eye(3), np.array([0, 0, 500.0]))
    with pytest.raises(ValueError):
        ob.render(*args, texture=np.ones((8, 8, 3)))
    with pytest.raises(ValueError):
        ob.render(*args, shading="phong")
    with pytest.raises(ValueError):
        ob.render(*args, mode="rgbd")


def test_render_mesh_shape_errors():
    from pvnet_b200.render import render_mesh
    v, f = rc.cube(50.0)
    vd, fd, Kd, Pd, cd = device_inputs(v, f, rc.camera_for(48, 64), rc.poses(2, np.random.default_rng(0)),
                                       colors_for(8, 0))
    ok = dict(vertices=vd, faces=fd, K=Kd, poses=Pd, h=48, w=64, near=100, far=2000)
    bad = [dict(vertices=vd[:, :2]), dict(faces=fd[:, :2]), dict(faces=fd.float()), dict(poses=Pd[:, :, :3]),
           dict(K=torch.stack([Kd] * 3)), dict(K=Kd[:2]), dict(h=0), dict(near=0), dict(near=3000)]
    for kw in bad:
        with pytest.raises(ValueError):
            render_mesh(**{**ok, **kw})
    with pytest.raises(ValueError):
        render_mesh(**ok, colors=cd[:5])
    with pytest.raises(ValueError):
        render_mesh(**ok, mode="normals")
    with pytest.raises(RuntimeError):
        render_mesh(**{**ok, "vertices": vd.cpu()})
