"""numpy restatement of `pvnet_refine_poses_depth` (csrc/refine.cu, DESIGN.md §28): depth-anchored pose refinement,
point-to-plane ICP of the rendered surface against a registered depth image, one object per image.  The render step,
the pixel rays, the stride rule, `block_sum`, the Gauss-Newton step and `so3_exp` are refine_oracle's own (§26); this
module restates the rest, in the kernel's operation order where the result is compared bit for bit:

1. Observed depth Zo: float32 as given, or uint16 d read as fp32(d) * fp32(depth_scale) (one rounded multiply).  A
   value <= 0 or not finite is no reading.
2. Pairs: pixel (r,c) forms a pair when the render at the round's pose covers it (Zr > 0), the mask holds it, it has a
   reading, and its four 4-neighbours are inside the image, in the mask and read.  Its ray is refine_oracle's:
   u = c + 0.5, v = r + 0.5, yn = (v - cy) / fy, xn = ((u - cx) - s yn) / fx, K read as fp32.
   - X = R^T (Zr (xn,yn,1) - t), refine_oracle.back_project's operations;
   - Y = (Zo xn, Zo yn, Zo);
   - with Q0..Q3 the neighbours' observed points at (r, c+1), (r, c-1), (r+1, c), (r-1, c): a = Q0 - Q1,
     b = Q2 - Q3, n = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0), |n| = sqrt((n0 n0 + n1 n1) + n2 n2), n = n / |n|,
     negated when (n0 Y0 + n1 Y1) + n2 Y2 > 0;
   - d = Xc - Y with Xc = refine_oracle.project's ((R[r,0] X0 + R[r,1] X1) + R[r,2] X2) + t_r, the residual
     e = (n0 d0 + n1 d1) + n2 d2, and |d| = sqrt((d0 d0 + d1 d1) + d2 d2).
   The pair is kept when |d| <= gate and e is finite.  Kept pairs are row-major; above max_points every
   ceil(n / max_points)-th from the first (refine_oracle.subsample).
3. The round's mean |e| at its starting pose: |e_i| on thread i % 256, summed by refine_oracle.block_sum, over the
   count -- bit for bit the kernel's, so the accept / undo decision is the kernel's by construction.  Round 0 gates:
   an empty mask (NO_CONTOUR), a render that covers nothing (NO_SILHOUETTE), fewer than MIN_PAIRS pairs (FEW_PAIRS)
   return the input.  A later round whose mean rose or that has fewer than MIN_PAIRS pairs is undone and the image
   stops.
4. Unless it is the last evaluation, GN_STEPS damped Gauss-Newton steps with the pairs fixed: e_i as above,
   J_i = [(R X_i) x n_i ; n_i] in (dw, dt) for R <- exp(dw) R, t <- t + dt, A = sum J J^T, g = sum J e.  numpy sums
   them here, the kernel in block_sum's fixed order with FMAs: they agree to rounding, not bit for bit.

CPU only by default (the render step is the `render=` parameter, as in refine_oracle); nothing here reads the
reference."""
from __future__ import annotations

import numpy as np

from oracle import refine_oracle as rfo


def observed_depth(depth, depth_scale=1.0):
    """depth [.., h, w] float32 or uint16 -> Zo float32, 0 where there is no reading."""
    d = np.asarray(depth)
    if d.dtype == np.uint16:
        z = d.astype(np.float32) * np.float32(depth_scale)
    else:
        z = d.astype(np.float32)
    with np.errstate(invalid="ignore"):
        return np.where((z > 0) & np.isfinite(z), z, np.float32(0)).astype(np.float32)


def rays(h, w, K):
    """-> xn, yn fp64 [h,w]: refine_oracle.back_project's normalised ray of every pixel."""
    fx, s, cx, fy, cy = rfo._camera(K)
    r, c = np.mgrid[0:h, 0:w]
    u, v = c + 0.5, r + 0.5
    yn = (v - cy) / fy
    xn = ((u - cx) - s * yn) / fx
    return xn, yn


def residuals(X, Y, n, pose):
    """-> e [m] = n . (R X + t - Y) and |R X + t - Y| [m], each operation rounded in the kernel's order."""
    P = np.asarray(pose, np.float64).reshape(3, 4)
    d = [(((P[r, 0] * X[:, 0] + P[r, 1] * X[:, 1]) + P[r, 2] * X[:, 2]) + P[r, 3]) - Y[:, r] for r in range(3)]
    dist = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    return (n[:, 0] * d[0] + n[:, 1] * d[1]) + n[:, 2] * d[2], dist


def pairs(rdepth, mask, zo, pose, K, gate, max_points):
    """One image's pairs at the fp64 pose: rendered depth [h,w] f32, mask [h,w], observed Zo [h,w] f32 (as
    `observed_depth` gives it) -> dict(idx int64 [m] row-major pixel indices, X, Y, n fp64 [m,3], count (kept pairs
    before the stride), mask_pixels, covered_pixels)."""
    rdepth = np.asarray(rdepth, np.float32)
    on = np.asarray(mask) != 0
    zo = np.asarray(zo, np.float32)
    h, w = on.shape
    read = on & (zo > 0)
    cand = (rdepth > 0) & read
    nb = np.zeros_like(cand)
    nb[1:-1, 1:-1] = read[1:-1, 2:] & read[1:-1, :-2] & read[2:, 1:-1] & read[:-2, 1:-1]
    cand &= nb
    idx = np.flatnonzero(cand)
    r, c = np.divmod(idx, w)
    xn, yn = rays(h, w, K)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    X = rfo.back_project(idx, rdepth, P, K, w)

    def point(rr, cc):
        z = zo[rr, cc].astype(np.float64)
        return np.stack([z * xn[rr, cc], z * yn[rr, cc], z], -1)

    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        Y = point(r, c)
        a = point(r, c + 1) - point(r, c - 1)
        b = point(r + 1, c) - point(r - 1, c)
        n = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                      a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], -1)
        ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        n = n / ln[:, None]
        flip = ((n[:, 0] * Y[:, 0] + n[:, 1] * Y[:, 1]) + n[:, 2] * Y[:, 2]) > 0
        n = np.where(flip[:, None], -n, n)
        e, dist = residuals(X, Y, n, P)
        keep = (dist <= gate) & np.isfinite(e)
    sel = rfo.subsample(np.flatnonzero(keep), max_points)
    return dict(idx=idx[sel], X=X[sel], Y=Y[sel], n=n[sel], count=int(keep.sum()), mask_pixels=int(on.sum()),
                covered_pixels=int((rdepth > 0).sum()))


def mean_residual(X, Y, n, pose):
    """-> (pairs, mean |e|): |e_i| on thread i % 256, summed by refine_oracle.block_sum, over the count."""
    m = len(X)
    if not m:
        return 0, float("nan")
    with np.errstate(invalid="ignore", over="ignore"):
        e, _ = residuals(X, Y, n, pose)
    return m, rfo.block_sum(np.abs(e)) / m


def jacobian(X, n, pose):
    """-> J [m,6] = [(R X) x n ; n]: d e / d(dw, dt) for R <- exp(dw) R, t <- t + dt."""
    P = np.asarray(pose, np.float64).reshape(3, 4)
    p = np.stack([(P[r, 0] * X[:, 0] + P[r, 1] * X[:, 1]) + P[r, 2] * X[:, 2] for r in range(3)], -1)
    return np.concatenate([np.cross(p, n), n], -1)


def normal_equations(X, Y, n, pose):
    """-> A [6,6], g [6] of sum e_i^2."""
    J = jacobian(X, n, pose)
    e, _ = residuals(X, Y, n, pose)
    return J.T @ J, J.T @ e


def refine_image(mask, depth, pose, K, verts, faces, near, far, gate, rounds=8, max_points=4096, depth_scale=1.0,
                 trace=None, render=None):
    """One image: mask [h,w], observed depth [h,w] (float32, or uint16 read with depth_scale), pose [3,4], K [3,3] ->
    (pose fp64 [3,4], info dict: status, pairs, dist_before, dist_after).  trace (a list) receives one dict per
    evaluation: the pose it started from, the pairs (as `pairs` returns them), their count and mean |e|, and the
    normal equations of each step it took.  render: refine_oracle.refine_image's step 1 (None: `rfo.oracle_depth`)."""
    render = rfo.oracle_depth if render is None else render
    mask = np.asarray(mask)
    h, w = mask.shape
    zo = observed_depth(depth, depth_scale)
    P = np.asarray(pose, np.float64).reshape(3, 4).copy()
    status, npairs, mean0, mean_after, mean_prev, backup = 0, 0, float("nan"), float("nan"), None, P
    for k in range(rounds + 1):
        rdepth = np.asarray(render(verts, faces, K, P.astype(np.float32), h, w, near, far), np.float32)
        pr = pairs(rdepth, mask, zo, P, K, gate, max_points)
        m, mean = mean_residual(pr["X"], pr["Y"], pr["n"], P)
        rec = dict(pose=P.copy(), n_pairs=m, mean=mean, normal_eq=[], **pr)
        if trace is not None:
            trace.append(rec)
        if k == 0:
            if pr["mask_pixels"] == 0:
                status |= rfo.NO_CONTOUR
                break
            if pr["covered_pixels"] == 0:
                status |= rfo.NO_SILHOUETTE
                break
            if m < rfo.MIN_PAIRS:
                status |= rfo.FEW_PAIRS
                break
            mean0 = mean_after = mean
        else:
            if m < rfo.MIN_PAIRS or mean > mean_prev:
                status |= rfo.REJECTED
                P = backup
                break
            mean_after = mean
        if k == rounds:
            break
        mean_prev, backup, npairs = mean, P.copy(), m
        for _ in range(rfo.GN_STEPS):
            A, g = normal_equations(pr["X"], pr["Y"], pr["n"], P)
            rec["normal_eq"].append((A, g))
            nP = rfo.gauss_newton_step(A, g, P)
            if nP is None:
                break
            P = nP
        if nP is None:
            status |= rfo.SINGULAR
            P = backup
            break
    return P, dict(status=status, pairs=npairs, dist_before=mean0, dist_after=mean_after)


def refine(mask, depth, poses, K, verts, faces, near, far, gate, rounds=8, max_points=4096, depth_scale=1.0,
           render=None):
    """mask [b,h,w], depth [b,h,w], poses [b,3,4], K [3,3] or [b,3,3] -> poses fp64 [b,3,4], info dict of [b]
    arrays."""
    mask = np.asarray(mask)
    poses = np.asarray(poses, np.float64).reshape(-1, 3, 4)
    b = len(poses)
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    out, infos = np.empty((b, 3, 4)), []
    for i in range(b):
        out[i], info = refine_image(mask[i], depth[i], poses[i], Ks[i], verts, faces, near, far, gate, rounds,
                                     max_points, depth_scale, render=render)
        infos.append(info)
    return out, {key: np.array([d[key] for d in infos]) for key in infos[0]}
