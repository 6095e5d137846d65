"""Keypoints for the keypoint-anchored refinement tests (tests/test_refine_keypoints_cpu.py,
tests/test_gpu_refine_keypoints.py) and benchmarks/refine_keypoints.py: model points on tests/refine_cases.py's meshes
and keypoints as a voting layer would give them.  Lengths are in metres."""
import numpy as np

from oracle import pnp_oracle as pno
from oracle import refine_oracle as rfo


def tool_keypoints():
    """Eight model points of `refine_cases.tool_mesh`, float32 [8,3]: corners of its three boxes spread over the
    solid, so together they fix every rotation."""
    return np.array([[-0.07, -0.015, -0.01], [0.05, 0.015, 0.01], [-0.07, 0.015, 0.01], [0.03, -0.015, 0.02],
                     [0.06, 0.05, 0.02], [0.03, 0.05, -0.01], [-0.06, -0.01, 0.035], [-0.03, 0.01, 0.035]],
                    np.float32)


def keypoint_votes(P, K, pts, sigma, rng):
    """Keypoints as a voting layer would give them: the projections of `pts` at the poses P [b,3,4] (the renderer's
    pixel convention, so they vanish with the silhouette term at the truth) plus Gaussian noise of `sigma` pixels,
    float32 [b,nk,2]; cov = sigma^2 I float32 [b,nk,2,2].  K: [3,3] or [b,3,3]."""
    P = np.asarray(P, np.float64).reshape(-1, 3, 4)
    b, nk = len(P), len(pts)
    K = np.asarray(K, np.float32)
    kp = np.empty((b, nk, 2))
    for i in range(b):
        u, v = rfo.project(np.asarray(pts, np.float64), P[i], K if K.ndim == 2 else K[i])
        kp[i] = np.stack([u, v], -1) + rng.normal(0, sigma, (nk, 2))
    cov = np.broadcast_to(np.eye(2) * sigma * sigma, (b, nk, 2, 2))
    return kp.astype(np.float32), np.ascontiguousarray(cov, np.float32)


def isotropic_weights(cov):
    """pnp_oracle.covariance_to_weights of cov [..., 2, 2], rounded to float32 as the device weights are."""
    c = np.asarray(cov, np.float64)
    return pno.covariance_to_weights(c.reshape(-1, 2, 2)).astype(np.float32).reshape(c.shape[:-2] + (3,))


def singular_scene_keypoints():
    """Five model points of `refine_cases.singular_scene` off its optical-axis line, float32 [5,3]: unlike the
    silhouette, their projections move under a rotation about the optical axis."""
    return np.array([[1.0, 0.0, 2.0], [0.0, 1.0, 2.0], [-1.0, 0.0, 3.0], [0.0, -1.0, 3.0], [1.0, 1.0, 4.0]],
                    np.float32)


def spread_keypoints(nk, seed=0):
    """nk model points spread over `refine_cases.tool_mesh`, float32 [nk,3]: each drawn uniformly inside one of its
    three boxes in turn, so every count has points on all three parts."""
    boxes = [((-0.07, -0.015, -0.01), (0.05, 0.015, 0.01)), ((0.03, -0.015, -0.01), (0.06, 0.05, 0.02)),
             ((-0.06, -0.01, 0.0), (-0.03, 0.01, 0.035))]
    rng = np.random.default_rng(seed)
    return np.array([rng.uniform(*boxes[k % 3]) for k in range(nk)], np.float32)


def camera_depth(P, X):
    """Z of the model point X [3] (float32) at the fp64 pose P [3,4], in the kernel's order:
    ((R20 x + R21 y) + R22 z) + t2, each operation rounded."""
    P = np.asarray(P, np.float64).reshape(3, 4)
    x, y, z = (np.float64(v) for v in np.asarray(X, np.float32))
    return ((P[2, 0] * x + P[2, 1] * y) + P[2, 2] * z) + P[2, 3]


def point_at_zero_depth(P):
    """A float32 model point [3] whose camera depth at the fp64 pose P is exactly 0 in `camera_depth`'s operations:
    z brings R22 z to within fp32 rounding of -t2, y cancels most of what is left and x, at a far finer fp32 scale,
    the rest; the fp32 neighbours of x and y are searched for an exact zero."""
    P = np.asarray(P, np.float64).reshape(3, 4)
    r0, r1, r2, t2 = P[2]
    z = np.float32(-t2 / r2)
    y0 = np.float32((-t2 - r2 * np.float64(z)) / r1)
    for y in _neighbours(y0, 8):
        x0 = np.float32((-t2 - r2 * np.float64(z) - r1 * np.float64(y)) / r0)
        for x in _neighbours(x0, 64):
            X = np.array([x, y, z], np.float32)
            if camera_depth(P, X) == 0.0:
                return X
    raise AssertionError("no fp32 point at zero depth")


def _neighbours(v, n):
    """v and its n nearest fp32 neighbours on each side, nearest first."""
    out, lo, hi = [v], v, v
    for _ in range(n):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return out
