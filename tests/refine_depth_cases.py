"""Observed depth images for the depth-anchored refinement tests (tests/test_refine_depth_cpu.py,
tests/test_gpu_refine_depth.py) and benchmarks/refine_depth.py.  The mesh itself is the sensor: the observed depth is
its render at the true pose, then one of the variants below.  Lengths are in metres."""
import numpy as np

from oracle import refine_oracle as rfo

GATE = 0.03                                          # 3 cm: above a 1 cm / 3 degree start's largest point offset


def noisy(depth, sigma, rng):
    """Seeded Gaussian noise of `sigma` on every reading, float32; pixels without a reading keep 0."""
    d = np.asarray(depth, np.float32)
    out = d + rng.normal(0.0, sigma, d.shape).astype(np.float32)
    return np.where(d > 0, out, np.float32(0)).astype(np.float32)


def holed(depth, r0, c0, size):
    """A size x size block of zero readings (no reading) with its top-left corner at (r0, c0)."""
    out = np.array(depth, np.float32, copy=True)
    out[..., r0:r0 + size, c0:c0 + size] = 0
    return out


def occluded(depth, mask, r0, c0, size, gap=0.05):
    """An occluder: a size x size patch at (r0, c0) `gap` closer than the object's nearest reading in the image, and
    the mask cut out where it sits (the segmentation sees the occluder, not the object)."""
    d = np.array(depth, np.float32, copy=True)
    m = np.array(mask, copy=True)
    near = d[d > 0].min() if (d > 0).any() else 0.5
    d[r0:r0 + size, c0:c0 + size] = np.float32(near - gap)
    m[r0:r0 + size, c0:c0 + size] = 0
    return d, m


def as_u16_mm(depth):
    """uint16 millimetres (the LINEMOD PNG format), rounded to the nearest; read back with depth_scale = 1e-3."""
    return np.round(np.asarray(depth, np.float64) * 1000.0).clip(0, 65535).astype(np.uint16)


def along_axis(P, dist):
    """The poses P [b,3,4] moved by `dist` along the optical axis (t_z only)."""
    out = np.array(P, np.float64, copy=True)
    out[..., 2, 3] += dist
    return out


# ---- scenes at the pair predicate's edges (tests/test_refine_anchored_edges_cpu.py,
#      tests/test_gpu_refine_anchored_edges.py) ----

def square(half):
    """A square of side 2 half in the object's z = 0 plane, two triangles facing -z."""
    v = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def flat_face(h, w, f, z=0.5):
    """A square facing the camera that fills an h x w image: mesh, K (no skew), pose R = I, t = (0, 0, z).  Its
    rendered depth is z at every pixel, so every pair's observed normal is exactly (0, 0, -1): the normal equations'
    rows for dw_z, dt_x and dt_y are exactly zero."""
    K = np.array([[f, 0, w / 2.0], [0, f, h / 2.0], [0, 0, 1]], np.float32)
    return square(z * max(h, w) / f), K, np.hstack([np.eye(3), [[0.0], [0.0], [z]]])


def tilted_plane(h, w, f, z=0.5):
    """A square turned 25 and 20 degrees about the x and y axes, z away along the optical axis, filling an h x w
    image: mesh, K (no skew) and pose.  Its normals are not the optical axis, so the system is regular."""
    K = np.array([[f, 0, w / 2.0], [0, f, h / 2.0], [0, 0, 1]], np.float32)
    R = rfo.so3_exp(np.deg2rad([25.0, 20.0, 0.0]))
    return square(2.0 * z * max(h, w) / f), K, np.hstack([R, [[0.0], [0.0], [z]]])


def strip(shape, r0, c0, rows, cols):
    """A rows x cols mask rectangle with its top-left corner at (r0, c0), uint8.  With readings everywhere and the
    render covering it, a 3 x c strip has c - 2 pixels whose four 4-neighbours are all in the mask."""
    m = np.zeros(shape, np.uint8)
    m[r0:r0 + rows, c0:c0 + cols] = 1
    return m


def tiny_ray_scene(h=12, w=12):
    """fx = fy = 3e37 px and a square 4e-36 across at z = 0.5, covering the image: mesh, K, pose and the render-sized
    readings, with the four 4-neighbours of the centre pixel read as the least fp32 subnormal.  Their observed points
    differ by ~5e-83, so the centre's normal a x b (~2e-165 per entry) squares to below the least fp64 subnormal and
    |n| = 0: n = 0 / 0, a residual that is not a number, while the centre's own point lies on the surface (|d| <<
    gate).  -> (mesh, K, pose, centre pixel index, the four neighbour indices)."""
    K = np.array([[3e37, 0, w / 2.0], [0, 3e37, h / 2.0], [0, 0, 1]], np.float32)
    r, c = h // 2, w // 2
    nb = [r * w + c + 1, r * w + c - 1, (r + 1) * w + c, (r - 1) * w + c]
    return square(2e-36), K, np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]]), r * w + c, nb


def tilted_tool():
    """`refine_cases.tool_mesh` turned by a fixed rotation in its own frame, float32: at R = I and t = (0, 0, t_z)
    the rendered point of every pixel comes back exactly (R X + t = Z (xn, yn, 1) when Z and t_z are within a factor
    of two), so against its own render every residual is exactly 0, and the faces it shows are not all parallel."""
    from tests import refine_cases as rf
    v, f = rf.tool_mesh()
    R = rfo.so3_exp(np.array([0.5, -0.4, 0.3]))
    return (v.astype(np.float64) @ R.T).astype(np.float32), f


def straddles(idx, period):
    """True when two consecutive pixels p, p + 1 both appear in idx with p + 1 a multiple of `period`."""
    s = np.asarray(idx, np.int64)
    return bool(np.isin(s[(s + 1) % period == 0] + 1, s).any())


def shrinking_strip(render, h=60, w=80, f=150.0, seed=5):
    """A 3 x 9 mask strip on `refine_cases.tool_mesh` whose pairs fall below six after the first round's steps:
    seeded truths and starts 3 degrees and 1 cm away, the strip centred on a pixel that both renders cover, the
    truth's render as the readings; the first draw whose oracle run is undone at its third evaluation with fewer
    than six pairs.  render: refine_oracle's render step.  -> (mask, readings, start, K)."""
    from oracle import refine_depth_oracle as rdo
    from tests import refine_cases as rf
    from tests import render_cases as rc
    K = rc.camera_for(h, w, f)
    mesh = rf.tool_mesh()
    rng = np.random.default_rng(seed)
    for _ in range(100):
        Pt = rf.true_poses(1, rng)[0]
        P0 = rf.perturb(Pt[None], rng, 3.0, 0.01)[0]
        dt = render(*mesh, K, Pt.astype(np.float32), h, w, rf.NEAR, rf.FAR)
        d0 = render(*mesh, K, P0.astype(np.float32), h, w, rf.NEAR, rf.FAR)
        rows, cols = np.nonzero((dt > 0) & (d0 > 0))
        if not len(rows):
            continue
        k = rng.integers(len(rows))
        m = strip((h, w), rows[k] - 1, cols[k] - 4, 3, 9)
        tr = []
        rdo.refine_image(m, dt, P0, K, *mesh, rf.NEAR, rf.FAR, GATE, rounds=3, trace=tr, render=render)
        if len(tr) == 3 and tr[1]["n_pairs"] >= 6 and tr[2]["n_pairs"] < 6:
            return m, dt, P0, K
    raise AssertionError("no strip loses its pairs")
