"""Instance scenes for depth-anchored refinement per instance (tests/test_gpu_refine_depth_instances.py,
benchmarks/refine_depth_instances.py, DESIGN.md §31): lumpy meshes at seeded poses composited by depth into a label
map, with the composite's nearest depth as the sensor.  `render` is refine_oracle's render step (rfo.oracle_depth on
the CPU, refine_cases.device_depth on the device, which test_gpu_render pins bit for bit to it).  Lengths in metres.

`refine_instances` restates the per-instance contract as a loop over oracle/refine_depth_oracle.py's one-image
refinement, one row per (image, instance) mask."""
import numpy as np

from oracle import refine_depth_oracle as rdo
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc


def linemod_k(h, w, scale=1.0):
    """LINEMOD's focal lengths with the principal point at the image centre, the focal lengths times `scale`."""
    return np.array([[572.4114 * scale, 0.0, w / 2.0], [0.0, 573.57043 * scale, h / 2.0], [0.0, 0.0, 1.0]],
                    np.float32)


def poses_at(xs, zs, rng):
    """Instances at (x, y, z), y within 1 cm of the axis, with random rotations -> float64 [n,3,4]."""
    P = np.zeros((len(xs), 3, 4))
    for i, (x, z) in enumerate(zip(xs, zs)):
        P[i, :, :3] = rf.axis_angle(rng.normal(size=3) * 0.3)
        P[i, :, 3] = (x, rng.uniform(-0.01, 0.01), z)
    return P


def composite(render, mesh, K, P, h, w, noise=1e-3, hole=None, rng=None):
    """Render each pose, take the nearest surface per pixel: -> labels int64 [h,w] (1 + index of the nearest
    instance, 0 where none), the observed depth float32 [h,w] (the nearest depth, `noise` metres of Gaussian noise on
    every reading, and a hole = (r0, c0, size) block without readings)."""
    d = np.stack([render(*mesh, K, p.astype(np.float32), h, w, rf.NEAR, rf.FAR) for p in P])
    dd = np.where(d > 0, d, np.inf)
    hit = np.isfinite(dd).any(0)
    lab = np.where(hit, dd.argmin(0) + 1, 0).astype(np.int64)
    obs = np.where(hit, dd.min(0), 0).astype(np.float32)
    if noise:
        obs = rdc.noisy(obs, noise, rng if rng is not None else np.random.default_rng(0))
    if hole is not None:
        obs = rdc.holed(obs, *hole)
    return lab, obs


NO_INSTANCE = 32


def refine_instances(labels, num, depth, poses, K, verts, faces, near, far, gate, rounds=8, max_points=4096,
                     depth_scale=1.0, render=None, traces=None):
    """The contract of `pvnet_refine_poses_depth_instances` (DESIGN.md §31) as a loop over
    oracle/refine_depth_oracle.py: labels [b,h,w] integer (0 background, j+1 instance j), num [b], depth [b,h,w],
    poses [b,L,3,4], K [3,3] or [b,3,3] -> poses fp64 [b,L,3,4], info dict of [b,L] arrays.  Row (i, j) with
    j < num[i] is `rdo.refine_image` on the mask labels[i] == j+1; the others keep their pose with status NO_INSTANCE,
    0 pairs and NaN distances.  traces (a dict) receives each present row's trace under (i, j)."""
    labels = np.asarray(labels).astype(np.int64)
    poses = np.asarray(poses, np.float64)
    b, L = poses.shape[:2]
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    out = poses.copy()
    info = {key: np.zeros((b, L), dt) for key, dt in (("status", np.int32), ("pairs", np.int32),
                                                     ("dist_before", np.float64), ("dist_after", np.float64))}
    info["dist_before"][:] = np.nan
    info["dist_after"][:] = np.nan
    for i in range(b):
        for j in range(L):
            if j >= num[i]:
                info["status"][i, j] = NO_INSTANCE
                continue
            tr = [] if traces is not None else None
            out[i, j], d = rdo.refine_image(labels[i] == j + 1, depth[i], poses[i, j], Ks[i], verts, faces, near, far,
                                            gate, rounds, max_points, depth_scale, trace=tr, render=render)
            if traces is not None:
                traces[(i, j)] = tr
            for key in info:
                info[key][i, j] = d[key]
    return out, info
