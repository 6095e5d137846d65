"""Seeded scenes of several posed instances of one rigid object for the per-instance pose tests and benchmark.

`instance_vote_cases.instance_scene` lays out the discs (touching or apart) and the ground-truth label map; here each
disc is an object at a known pose whose centre (model point 0,0,0) projects to the disc's centre, and the planted field
points, per pixel, at its own instance's projected model points.  The last model point is the centre, so
`vertex[..., -1, :]` is the centre field `ransac_voting_center` reads.
"""
import numpy as np

from tests import instance_vote_cases as ivc

K_LINEMOD = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]])

# model points (m), the last one the object centre
POINTS_3D = np.array([[0.045, 0.008, 0.0], [-0.036, 0.027, 0.012], [0.012, -0.05, -0.01], [-0.022, -0.03, 0.02],
                      [0.04, 0.03, -0.02], [-0.046, -0.009, -0.015], [0.018, 0.044, 0.025], [0.037, -0.021, 0.03],
                      [0.0, 0.0, 0.0]], np.float32)


def _rotation(rng, max_deg=25.0):
    """A random rotation within max_deg of the identity."""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    th = np.deg2rad(rng.uniform(0.0, max_deg))
    W = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(th) * W + (1 - np.cos(th)) * W @ W


def project(P, R, t, K):
    X = P.astype(np.float64) @ R.T + t
    uv = X @ K.T
    return uv[:, :2] / uv[:, 2:]


def pose_scene(n, seed, h=480, w=640, sigma=0.0, touching=False, K=K_LINEMOD):
    """-> dict(mask uint8 [h,w], gt int32 [h,w] (1..n), R [n,3,3], t [n,3], keypoints [n,9,2] f64 (the projected
    model points), field f32 [h,w,9,2]).  Depths are 0.9..1.1 m."""
    s = ivc.instance_scene(n, seed, h, w, k=1, touching=touching)
    rng = np.random.default_rng(10_000 + seed)
    Kinv = np.linalg.inv(K)
    R = np.stack([_rotation(rng) for _ in range(n)])
    z = rng.uniform(0.9, 1.1, n)
    t = np.stack([z[i] * Kinv @ np.array([s["centers"][i, 0], s["centers"][i, 1], 1.0]) for i in range(n)])
    kps = np.stack([project(POINTS_3D, R[i], t[i], K) for i in range(n)])
    gt = s["gt"]
    k = POINTS_3D.shape[0]
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    field = np.zeros((h, w, k, 2), np.float32)
    fg = gt > 0
    own = kps[np.maximum(gt, 1) - 1]                                              # [h,w,k,2]
    for j in range(k):
        dx, dy = own[:, :, j, 0] - xs, own[:, :, j, 1] - ys
        nrm = np.sqrt(dx * dx + dy * dy)
        nrm[nrm < 1e-3] += 1e-3
        dx, dy = dx / nrm, dy / nrm
        eps = rng.normal(0.0, sigma, size=(h, w)) if sigma > 0 else np.zeros((h, w))
        c, sn = np.cos(eps), np.sin(eps)
        field[:, :, j, 0] = (c * dx - sn * dy) * fg
        field[:, :, j, 1] = (sn * dx + c * dy) * fg
    return dict(mask=fg.astype(np.uint8), gt=gt, R=R, t=t, keypoints=kps, field=field, centers=s["centers"])


def touching_pairs(gt):
    """Pairs (a, b), a < b, of instances with 4-adjacent pixels."""
    pairs = set()
    for d in ((gt[:, 1:], gt[:, :-1]), (gt[1:, :], gt[:-1, :])):
        a, b = d
        m = (a > 0) & (b > 0) & (a != b)
        pairs |= {(min(x, y), max(x, y)) for x, y in zip(a[m].tolist(), b[m].tolist())}
    return pairs


def pose_errors(R, t, Rg, tg):
    """Rotation error (deg) and translation error (m) of one pose against the truth."""
    c = np.clip((np.trace(R @ Rg.T) - 1.0) / 2.0, -1.0, 1.0)
    return float(np.rad2deg(np.arccos(c))), float(np.linalg.norm(t - tg))
