"""Seeded scenes of several instances of one object class for the instance-voting tests and benchmark.

Each instance is a disc at a non-integer centre; a pixel covered by several discs belongs to the one whose
centre is nearest, so touching and overlapping discs still give one ground-truth instance per pixel.  The
field plants, per pixel, unit vectors towards its own instance's keypoints, rotated by eps ~ N(0, sigma rad)
as `pvnet_b200.synthetic.planted_field` does; the last keypoint is the instance centre.
"""
import numpy as np

# keypoint offsets from the centre (px), the last one is the centre itself
_OFFSETS = np.array([[30.0, 5.0], [-24.0, 18.0], [8.0, -33.0], [-15.0, -20.0], [36.0, 27.0], [-31.0, -6.0],
                     [12.0, 29.0], [25.0, -14.0], [0.0, 0.0]])


def instance_scene(n, seed, h=480, w=640, sigma=0.0, k=9, touching=False, radius=(40.0, 70.0)):
    """-> dict(mask uint8 [h,w], gt int32 [h,w] (1..n), centers [n,2] f64, keypoints [n,k,2] f64,
    field f32 [h,w,k,2])."""
    rng = np.random.default_rng(seed)
    centers, radii = [], []
    for _ in range(1000):
        if len(centers) == n:
            break
        r = rng.uniform(*radius)
        c = np.array([rng.uniform(r + 2, w - r - 2), rng.uniform(r + 2, h - r - 2)]) + rng.uniform(0.1, 0.9, 2)
        ok = True
        for cj, rj in zip(centers, radii):
            d = np.hypot(*(c - cj))
            gap = d - r - rj
            # touching scenes: the second disc is placed against the first one
            if (touching and len(centers) == 1 and not (-3.0 < gap < 0.5)) or d < 1.2 * max(r, rj) or gap < -3.0:
                ok = False
            if not touching and gap < 4.0:
                ok = False
        if ok:
            centers.append(c)
            radii.append(r)
    assert len(centers) == n, "scene did not fit"
    centers = np.array(centers)
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    dist = np.stack([np.hypot(xs - c[0], ys - c[1]) for c in centers])          # [n,h,w]
    inside = dist <= np.array(radii)[:, None, None]
    near = np.where(inside, dist, np.inf).argmin(0)
    gt = np.where(inside.any(0), near + 1, 0).astype(np.int32)
    kps = centers[:, None, :] + _OFFSETS[None, -k:, :]
    field = np.zeros((h, w, k, 2), np.float32)
    fg = gt > 0
    own = kps[np.maximum(gt, 1) - 1]                                              # [h,w,k,2]
    for j in range(k):
        dx, dy = own[:, :, j, 0] - xs, own[:, :, j, 1] - ys
        nrm = np.sqrt(dx * dx + dy * dy)
        nrm[nrm < 1e-3] += 1e-3
        dx, dy = dx / nrm, dy / nrm
        eps = rng.normal(0.0, sigma, size=(h, w)) if sigma > 0 else np.zeros((h, w))
        c, s = np.cos(eps), np.sin(eps)
        field[:, :, j, 0] = (c * dx - s * dy) * fg
        field[:, :, j, 1] = (s * dx + c * dy) * fg
    return dict(mask=fg.astype(np.uint8), gt=gt, centers=centers, keypoints=kps, field=field)


def match_ids(labels, gt, centers, gt_centers):
    """Relabel `labels` so each found centre takes the id of the nearest ground-truth centre."""
    out = np.zeros_like(labels)
    for j, c in enumerate(centers):
        g = int(np.argmin(np.hypot(*(gt_centers - c[None]).T)))
        out[labels == j + 1] = g + 1
    return out


def draw_center_idxs(b, I, hn, seed):
    """int32 [b,I,hn,2] raw sample words (any int32; the kernels reduce them modulo |R_i|)."""
    return np.random.default_rng(seed).integers(0, 2 ** 31 - 1, size=(b, I, hn, 2), dtype=np.int32)
