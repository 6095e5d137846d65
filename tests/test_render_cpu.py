"""CPU: the mesh-rendering contract of DESIGN.md §24 in oracle/render_oracle.py against analytic scenes, the
half-pixel convention against the matrices the reference's OpenGL backend builds (tests/golden/ref_render.npz), and
the `lib.utils.opengl_render_backend` drop-in's signature and argument errors."""
import inspect
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import Delaunay

from oracle import render_oracle as ro
from tests import render_cases as rc
from tests.helpers import GOLDEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = np.array([[500.0, 0, 320.0], [0, 510.0, 240.0], [0, 0, 1]], np.float32)


def pose(R=np.eye(3), t=(0, 0, 0)):
    P = np.zeros((1, 3, 4), np.float32)
    P[0, :, :3] = R
    P[0, :, 3] = t
    return P


def pixel_rays(h, w, Kf):
    """fp64 ray directions K^-1 (c + 0.5, r + 0.5, 1), scaled to Z = 1: [h,w,3]."""
    r, c = np.mgrid[0:h, 0:w]
    p = np.stack([c + 0.5, r + 0.5, np.ones_like(c, np.float64)], -1)
    return p @ np.linalg.inv(Kf.astype(np.float64)).T


def plane_hits(tri, rays):
    """Ray-plane intersections of a camera-space triangle [3,3] (fp64): points [h,w,3] and barycentrics [h,w,3]."""
    a, b, c = tri
    n = np.cross(b - a, c - a)
    s = (n @ a) / (rays @ n)
    X = rays * s[..., None]
    T = np.stack([a, b, c], 1)                                            # columns are the vertices
    lam = np.linalg.solve(np.vstack([T, np.ones(3)]).T @ np.vstack([T, np.ones(3)]),
                          (np.concatenate([X, np.ones(X.shape[:-1] + (1,))], -1) @ np.vstack([T, np.ones(3)]))[..., None])[..., 0]
    return X, lam


def test_fronto_parallel_square_covers_pixel_centres_inside_at_exact_depth():
    d = np.float32(800.3)
    v = np.array([[-50, -50, 0], [50, -50, 0], [50, 50, 0], [-50, 50, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    depth, rgb, win = ro.render(v, f, K, pose(t=(3.0, -2.0, d)), 480, 640, 100, 2000)
    x = (np.array([-50, 50]) + np.float64(np.float32(3.0))) / np.float64(d)
    y = (np.array([-50, 50]) + np.float64(np.float32(-2.0))) / np.float64(d)
    u, vv = 500.0 * x + 320.0, 510.0 * y + 240.0
    r, c = np.mgrid[0:480, 0:640]
    inside = (c + 0.5 >= u[0]) & (c + 0.5 <= u[1]) & (r + 0.5 >= vv[0]) & (r + 0.5 <= vv[1])
    assert np.array_equal(depth[0] > 0, inside)
    assert (depth[0][inside] == d).all()
    assert (depth[0][~inside] == 0).all() and (rgb[0][~inside] == 0).all()
    assert set(np.unique(win)) == {-1, 0, 1}


def test_tilted_plane_depth_within_one_ulp_of_ray_plane_intersection():
    rng = np.random.default_rng(3)
    R = rc.rotation(rng)
    R = R if abs(R[2, 2]) > 0.5 else R.T
    v = np.array([[-400, -400, 0], [400, -400, 0], [400, 400, 0], [-400, 400, 0]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    P = pose(R, (0, 0, 1000))
    Kc = rc.camera_for(120, 160)
    depth, _, _ = ro.render(v, f, Kc, P, 120, 160, 100, 5000)
    V, _ = ro.camera_vertices(v, P[0], Kc)
    n = np.cross(V[1] - V[0], V[2] - V[0])
    rays = pixel_rays(120, 160, Kc)
    Z = (n @ V[0]) / (rays @ n)
    hit = depth[0] > 0
    assert hit.mean() > 0.2
    err = np.abs(depth[0][hit].astype(np.float64) - Z[hit]) / np.spacing(depth[0][hit])
    assert err.max() <= 1.0


def test_nearer_face_wins_and_exact_tie_goes_to_lower_index():
    far_tri = np.array([[-100, -100, 900], [100, -100, 900], [0, 100, 900]], np.float32)
    near_tri = np.array([[-60, -60, 700], [60, -60, 700], [0, 60, 700]], np.float32)
    v = np.concatenate([far_tri, near_tri, far_tri])                     # face 2 duplicates face 0's geometry
    f = np.arange(9).reshape(3, 3)
    depth, _, win = ro.render(v, f, rc.camera_for(96, 128, 60.0), pose(), 96, 128, 100, 2000)
    assert (win[0] == 1).any() and (win[0] == 0).any()
    assert not (win[0] == 2).any()                                         # the tie with face 0 goes to face 0
    assert (depth[0][win[0] == 1] == np.float32(700)).all()
    assert (depth[0][win[0] == 0] == np.float32(900)).all()
    # with the order reversed the later copy loses again
    _, _, win2 = ro.render(v, f[::-1].copy(), rc.camera_for(96, 128, 60.0), pose(), 96, 128, 100, 2000)
    assert np.array_equal(win2[0] == 0, win[0] == 0)                       # face 0 of the reversed list is old face 2


@pytest.mark.parametrize("mesh", ["icosphere", "cube"])
def test_closed_mesh_has_no_hole_inside_its_silhouette(mesh):
    rng = np.random.default_rng(11)
    v, f = rc.icosphere(2, 80.0) if mesh == "icosphere" else rc.cube(60.0)
    h, w = 90, 110
    Kc = rc.camera_for(h, w, 150.0)
    for _ in range(3):
        P = rc.poses(1, rng, depth=(400.0, 600.0), shift=10.0)
        depth, _, win = ro.render(v, f, Kc, P, h, w, 10, 5000)
        V, hh = ro.camera_vertices(v, P[0], Kc)
        uv = hh[:, :2] / hh[:, 2:]
        tri = Delaunay(uv)
        r, c = np.mgrid[0:h, 0:w]
        pts = np.stack([c + 0.5, r + 0.5], -1).reshape(-1, 2)
        in_hull = tri.find_simplex(pts) >= 0
        # the silhouette is the hull of the projected vertices; keep away from its edges by more than rounding
        a, b = uv[tri.convex_hull[:, 0]], uv[tri.convex_hull[:, 1]]
        ab = b - a
        t = np.clip(np.einsum("pej,ej->pe", pts[:, None] - a, ab) / np.einsum("ej,ej->e", ab, ab), 0, 1)
        dist = np.linalg.norm(pts[:, None] - (a + t[..., None] * ab), axis=-1).min(1)
        inside = in_hull & (dist > 1e-6)
        assert inside.sum() > 500
        covered = (win[0] >= 0).reshape(-1)
        assert covered[inside].all()
        assert not covered[~in_hull].any()


def test_faces_crossing_the_near_plane_and_the_camera_plane_follow_the_per_fragment_rule():
    h, w = 60, 80
    Kc = rc.camera_for(h, w, 40.0)
    rays = pixel_rays(h, w, Kc)
    cases = [
        np.array([[-300, -200, 50], [300, -200, 50], [0, 250, 500]], np.float32),     # crosses near = 100
        np.array([[-300, -200, -80], [300, -150, 400], [-50, 300, 700]], np.float32),  # crosses Z = 0
        np.array([[-300, -200, 1500], [300, -200, 1500], [0, 250, 3000]], np.float32),  # crosses far = 2000
        np.array([[-300, -200, 2500], [300, -200, 2500], [0, 250, 3000]], np.float32),  # beyond far
        np.array([[-300, -200, -80], [300, -200, -80], [0, 250, -30]], np.float32),     # behind the camera
    ]
    for tri in cases:
        depth, _, win = ro.render(tri, np.array([[0, 1, 2]]), Kc, pose(), h, w, 100, 2000)
        X, lam = plane_hits(tri.astype(np.float64), rays)
        Z = X[..., 2]
        want = (lam >= 0).all(-1) & (Z >= 100) & (Z <= 2000)
        clear = (np.abs(lam) > 1e-9).all(-1) & (np.abs(Z - 100) > 1e-6) & (np.abs(Z - 2000) > 1e-6)
        got = win[0] >= 0
        assert np.array_equal(got[clear], want[clear]), tri
        assert (np.abs(depth[0][got] - Z[got]) <= 1e-3).all()


def test_degenerate_nan_and_out_of_range_faces_cover_nothing():
    v = np.array([[-50, -50, 800], [50, -50, 800], [0, 50, 800], [100, -50, 800], [np.nan, 0, 800],
                  [-50, -50, 800]], np.float32)
    bad = np.array([[0, 0, 1],      # repeated index
                    [0, 1, 3],      # collinear
                    [0, 1, 4],      # NaN vertex
                    [0, 1, 6],      # index == nv
                    [-1, 1, 2],     # negative index
                    [0, 5, 1]])     # two indices, one position: zero area
    depth, rgb, win = ro.render(v, bad, K, pose(), 48, 64, 100, 2000, bg=(0.2, 0.4, 1.0))
    assert (win == -1).all() and (depth == 0).all()
    assert (rgb[0] == ro.to_u8(np.float32([0.2, 0.4, 1.0]))).all()
    ok = np.concatenate([bad, [[0, 1, 2]]])
    _, _, win = ro.render(v, ok, rc.camera_for(48, 64, 600.0), pose(), 48, 64, 100, 2000)
    assert set(np.unique(win)) == {-1, len(bad)}


def test_u8_rounding_is_half_to_even_of_the_fp32_product():
    assert ro.to_u8(np.array([0.5, 1.5 / 255, 2.5 / 255, 1.0, 1.2, -0.1, np.nan])).tolist() == \
        [int(np.rint(np.float32(0.5) * np.float32(255))), 2, 2, 255, 255, 0, 0]


def test_shared_edges_are_exact_negations():
    rng = np.random.default_rng(5)
    v, f = rc.icosphere(1, 90.0)
    _, hh = ro.camera_vertices(v, rc.poses(1, rng)[0], rc.K_LINEMOD)
    c, ok, fi = ro.face_setup(f, len(v), hh)
    assert ok.all()
    edges = {}
    for k, face in enumerate(fi):
        for i in range(3):
            a, b = face[(i + 1) % 3], face[(i + 2) % 3]
            edges.setdefault((min(a, b), max(a, b)), []).append((a < b, c[k, i]))
    for (a, b), uses in edges.items():
        assert len(uses) == 2
        (s0, c0), (s1, c1) = uses
        assert s0 != s1 and np.array_equal(c0, -c1)


# ------------------------------------------------------------------------------ the reference's GL conventions
@pytest.fixture(scope="module")
def ref_render():
    z = np.load(os.path.join(GOLDEN, "ref_render.npz"))
    return {name: {k.split("/")[1]: z[k] for k in z.files if k.startswith(name + "/")}
            for name in sorted({k.split("/")[0] for k in z.files})}


def test_fixture_matrices_map_pixel_centres_to_half_pixel_points(ref_render):
    """GL's chain on the reference's own matrices -- clip = [X, 1] u_mvp, NDC = clip / w, window = (NDC + 1) / 2 *
    size, output row = h - 1 - window row -- puts OpenCV's image point (u, v) at window (u, h - v): output pixel
    (r, c) (window centre (c + 0.5, h - r - 0.5)) samples (c + 0.5, r + 0.5)."""
    assert len(ref_render) == 4
    rng = np.random.default_rng(1)
    for name, z in ref_render.items():
        w, h = (int(x) for x in z["im_size"])
        near, far = z["clip"]
        Kf = z["K"].astype(np.float32).astype(np.float64)
        R, t = z["R"].astype(np.float32).astype(np.float64), z["t"].reshape(3).astype(np.float32).astype(np.float64)
        r = rng.integers(0, h, 50)
        c = rng.integers(0, w, 50)
        Zc = rng.uniform(near, far, 50)
        ray = np.stack([c + 0.5, r + 0.5, np.ones(50)], -1) @ np.linalg.inv(Kf).T
        Xc = ray * Zc[:, None]                                              # OpenCV camera space
        X = (Xc - t) @ R                                                    # object space (R orthonormal)
        clip = np.concatenate([X, np.ones((50, 1))], 1) @ z["mvp"]
        ndc = clip[:, :3] / clip[:, 3:]
        xw, yw = (ndc[:, 0] + 1) / 2 * w, (ndc[:, 1] + 1) / 2 * h
        assert np.allclose(xw, c + 0.5, atol=1e-4), name
        assert np.allclose(h - 1 - (yw - 0.5), r, atol=1e-4), name          # the [::-1] row flip
        eye = np.concatenate([X, np.ones((50, 1))], 1) @ z["mv"]
        assert np.allclose(-eye[:, 2], Zc, rtol=1e-5), name                 # v_eye_depth is OpenCV's Z
        assert (np.abs(ndc[:, 2]) <= 1 + 1e-6).all()
        # GL's near and far clipping is NDC z = -1 at Z = near and +1 at Z = far: the per-fragment near <= Z <= far
        for zz, want in ((near, -1.0), (far, 1.0)):
            cz = np.array([0, 0, -zz, 1.0]) @ z["proj"]
            assert abs(cz[2] / cz[3] - want) < 1e-9


def test_dropin_signature_matches_reference():
    from lib.utils import opengl_render_backend as ob
    with open(os.path.join(GOLDEN, "ref_render_signature.json")) as f:
        want = json.load(f)["render"]
    parts = [p.name if p.default is inspect.Parameter.empty else f"{p.name}={p.default!r}"
             for p in inspect.signature(ob.render).parameters.values()]
    assert ", ".join(parts) == want


def test_dropin_import_loads_neither_glumpy_nor_cv2():
    code = ("import sys; from lib.utils.opengl_render_backend import render; "
            "print(sorted(m for m in ('glumpy', 'cv2') if m in sys.modules))")
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "[]", out.stdout


@pytest.mark.parametrize("kw", [dict(texture=np.zeros((4, 4, 3))), dict(shading="phong"), dict(mode="normals")])
def test_dropin_refuses_texture_phong_and_unknown_mode(kw):
    from lib.utils import opengl_render_backend as ob
    model = {"pts": np.zeros((3, 3), np.float32), "faces": np.array([[0, 1, 2]])}
    with pytest.raises(ValueError):
        ob.render(model, [8, 6], K, np.eye(3), np.array([0, 0, 500.0]), **kw)
