"""numpy restatement of `pvnet_refine_poses` (csrc/refine.cu, DESIGN.md §26): silhouette pose refinement, the four
steps the reference's `post_refinement` docstring lists (lib/utils/extend_utils/extend_utils.py:181-193) and leaves
unimplemented.

Per image and round, in the kernel's operation order where the result is compared bit for bit:

1. Depth at the current pose: the renderer's contract (§24, `render_oracle.render`; see below) with the pose rounded
   to fp32.
2. Silhouette: covered pixels (depth > 0) with a 4-neighbour that is uncovered or outside the image, row-major.
   Back-projection in fp64, K read as fp32 like the renderer reads it: u = c + 0.5, v = r + 0.5,
   yn = (v - cy) / fy, xn = ((u - cx) - s yn) / fx, X_cam = (Z xn, Z yn, Z), d = X_cam - t,
   X_obj[j] = (R[0,j] d0 + R[1,j] d1) + R[2,j] d2.
3. Contour: foreground mask pixels (nonzero) with a 4-neighbour that is background or outside the image, row-major.
   Both sets: above max_points, every ceil(n / max_points)-th point from the first.
4. Pairs: X_obj projected at the current pose (p_r = (R[r,0] x + R[r,1] y) + R[r,2] z, X_c = p + t,
   u = ((fx X + s Y) + cx Z) / Z, v = (fy Y + cy Z) / Z), rounded to fp32; for each contour point's centre
   (cu, cv) in fp32, dx = cu - pu, dy = cv - pv, d2 = dx dx + dy dy in fp32; the nearest is the lowest index of the
   smallest d2; the pair is dropped (index -1) when d2 > fp32(gate) * fp32(gate) or d2 is not a number.
5. The round's mean pair distance is the mean of sqrt(d2) in fp64 over its pairs, summed in k_refine_step's order
   (`block_sum`): bit for bit the kernel's, so the accept / undo decision below is the kernel's by construction, not
   to a tolerance.  Round 0 records it; a later round whose mean is above the previous round's, or that has no
   silhouette or fewer than MIN_PAIRS pairs, is rejected: the previous pose is kept and the image stops.  Otherwise, unless it is the last evaluation, GN_STEPS damped
   Gauss-Newton steps with the pairs held fixed: residual pi(X_obj) - c, Jacobian in (dw, dt) for
   R <- exp(dw) R, t <- t + dt; (A + DAMPING diag(A)) delta = -g by Cholesky.  A failed factorisation keeps the
   round's starting pose and stops the image.

The normal equations are summed with numpy here and in a fixed order on the device, where nvcc also contracts
multiplies and adds into FMAs: they agree to rounding, not bit for bit.

Step 1's renderer is a parameter (`render=` of `refine_image` and `refine`).  The default is `render_oracle.render`,
which evaluates every face at every pixel and takes seconds to minutes per 480x640 image.  The device renderer,
`pvnet_b200.render.render_mesh`, is pinned bit for bit to it for the same fp32 pose and K (tests/test_gpu_render.py),
so passing a wrapper around it checks the refinement's own steps at full size in seconds.  CPU only by default;
nothing here reads the reference."""
from __future__ import annotations

import numpy as np

from oracle import render_oracle as ro

NO_CONTOUR, NO_SILHOUETTE, FEW_PAIRS, SINGULAR, REJECTED = 1, 2, 4, 8, 16
MIN_PAIRS = 6
GN_STEPS = 3
DAMPING = 1e-3


def boundary(on):
    """on: bool [h,w] -> int64 row-major indices of the pixels that are on and have a 4-neighbour that is off or
    outside the image."""
    on = np.asarray(on, bool)
    p = np.pad(on, 1, constant_values=False)
    off_nb = ~p[:-2, 1:-1] | ~p[2:, 1:-1] | ~p[1:-1, :-2] | ~p[1:-1, 2:]
    return np.flatnonzero(on & off_nb)


def subsample(idx, max_points):
    """Every ceil(n / max_points)-th entry from the first."""
    n = len(idx)
    return idx[::max(1, -(-n // max_points))]


def _camera(K):
    k = np.asarray(K, np.float32).astype(np.float64).reshape(3, 3)
    return k[0, 0], k[0, 1], k[0, 2], k[1, 1], k[1, 2]


def back_project(idx, depth, pose, K, w):
    """Silhouette pixel indices, their fp32 depths and the fp64 pose [3,4] -> X_obj [n,3] fp64."""
    fx, s, cx, fy, cy = _camera(K)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    r, c = np.divmod(np.asarray(idx, np.int64), w)
    u, v = c + 0.5, r + 0.5
    Z = np.asarray(depth, np.float32).reshape(-1)[idx].astype(np.float64)
    yn = (v - cy) / fy
    xn = ((u - cx) - s * yn) / fx
    d = np.stack([Z * xn - P[0, 3], Z * yn - P[1, 3], Z - P[2, 3]], -1)
    return np.stack([(P[0, j] * d[:, 0] + P[1, j] * d[:, 1]) + P[2, j] * d[:, 2] for j in range(3)], -1)


def project(X, pose, K):
    """X [n,3] fp64 at the fp64 pose -> u, v fp64 (the renderer's projection)."""
    fx, s, cx, fy, cy = _camera(K)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    Xc = [((P[r, 0] * X[:, 0] + P[r, 1] * X[:, 1]) + P[r, 2] * X[:, 2]) + P[r, 3] for r in range(3)]
    return ((fx * Xc[0] + s * Xc[1]) + cx * Xc[2]) / Xc[2], (fy * Xc[1] + cy * Xc[2]) / Xc[2]


def centres(idx, w):
    """Pixel indices -> fp32 centres (c + 0.5, r + 0.5)."""
    r, c = np.divmod(np.asarray(idx, np.int64), w)
    return (c + 0.5).astype(np.float32), (r + 0.5).astype(np.float32)


def nearest_pairs(X, pose, K, con, w, gate, chunk=1024):
    """-> pair index into con int64 [n] (-1: dropped) and d2 fp32 [n] (the nearest squared distance)."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        u, v = project(X, pose, K)
    pu, pv = u.astype(np.float32), v.astype(np.float32)
    cu, cv = centres(con, w)
    g2 = np.float32(gate) * np.float32(gate)
    n = len(X)
    j = np.full(n, -1, np.int64)
    d2 = np.full(n, np.inf, np.float32)
    if len(con) == 0:
        return j, d2
    with np.errstate(invalid="ignore", over="ignore"):
        for i0 in range(0, n, chunk):
            sl = slice(i0, min(n, i0 + chunk))
            dx = cu[None, :] - pu[sl, None]
            dy = cv[None, :] - pv[sl, None]
            d = dx * dx + dy * dy
            d = np.where(np.isnan(d), np.float32(np.inf), d)
            a = np.argmin(d, axis=1)                               # first minimum: the lowest contour index
            dm = d[np.arange(len(a)), a]
            d2[sl] = dm
            j[sl] = np.where(dm <= g2, a, -1)
    return j, d2


STEP_THREADS = 256                                                  # k_refine_step's CTA


def block_sum(x, threads=STEP_THREADS):
    """Sum of fp64 x [n] in k_refine_step's order: thread t adds x[t], x[t + threads], ... in turn from 0.0; each
    warp of 32 combines its lanes by xor butterflies at offsets 16, 8, 4, 2, 1 (lane l adds lane l ^ o's value;
    fp64 addition commutes, so every lane ends with lane 0's value); then warp 0's value plus warps 1, 2, ... in
    order."""
    x = np.asarray(x, np.float64)
    rows = np.zeros((-(-len(x) // threads), threads))
    rows.reshape(-1)[:len(x)] = x
    part = np.zeros(threads)
    for row in rows:                                                # each thread's sum, in index order
        part = part + row
    lanes = part.reshape(threads // 32, 32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    total = lanes[0, 0]
    for q in range(1, threads // 32):
        total = total + lanes[q, 0]
    return float(total)


def mean_distance(j, d2):
    """-> (kept pairs, their mean distance): sqrt(fp64(d2)) of each kept pair i, summed by `block_sum` with pair i on
    thread i % 256 (a dropped pair adds nothing), over the count."""
    keep = j >= 0
    n = int(keep.sum())
    if not n:
        return 0, float("nan")
    return n, block_sum(np.where(keep, np.sqrt(d2.astype(np.float64)), 0.0)) / n


def normal_equations(X, cu, cv, pose, K):
    """Pairs X [n,3] fp64 -> contour centres (cu, cv): A [6,6] and g [6] of sum |pi(R X + t) - c|^2 in
    (dw, dt), R <- exp(dw) R, t <- t + dt."""
    fx, s, cx, fy, cy = _camera(K)
    P = np.asarray(pose, np.float64).reshape(3, 4)
    p = np.stack([(P[r, 0] * X[:, 0] + P[r, 1] * X[:, 1]) + P[r, 2] * X[:, 2] for r in range(3)], -1)
    Xc = p + P[:, 3]
    iz = 1.0 / Xc[:, 2]
    u = ((fx * Xc[:, 0] + s * Xc[:, 1]) + cx * Xc[:, 2]) * iz
    v = (fy * Xc[:, 1] + cy * Xc[:, 2]) * iz
    ru, rv = u - cu.astype(np.float64), v - cv.astype(np.float64)
    zero = np.zeros_like(iz)
    du = np.stack([fx * iz, s * iz, -(u - cx) * iz], -1)
    dv = np.stack([zero, fy * iz, -(v - cy) * iz], -1)
    Ju = np.concatenate([np.cross(p, du), du], -1)                  # d u / d(dw) = p x du for -[p]x
    Jv = np.concatenate([np.cross(p, dv), dv], -1)
    A = Ju.T @ Ju + Jv.T @ Jv
    g = Ju.T @ ru + Jv.T @ rv
    return A, g


def so3_exp(w):
    """Rodrigues, in pnp.cu's form: E = I + a [w]x + b [w]x^2."""
    wx, wy, wz = w
    th2 = wx * wx + wy * wy + wz * wz
    if th2 < 1e-16:
        a, b = 1.0 - th2 / 6.0, 0.5 - th2 / 24.0
    else:
        th = np.sqrt(th2)
        a, b = np.sin(th) / th, (1.0 - np.cos(th)) / th2
    return np.array([[1.0 - b * (wy * wy + wz * wz), -a * wz + b * wx * wy, a * wy + b * wx * wz],
                     [a * wz + b * wx * wy, 1.0 - b * (wx * wx + wz * wz), -a * wx + b * wy * wz],
                     [-a * wy + b * wx * wz, a * wx + b * wy * wz, 1.0 - b * (wx * wx + wy * wy)]])


def gauss_newton_step(A, g, pose):
    """-> the updated pose, or None when A + DAMPING diag(A) is not positive definite."""
    M = A + DAMPING * np.diag(np.diag(A))
    if not np.isfinite(M).all():
        return None
    try:
        L = np.linalg.cholesky(M)
    except np.linalg.LinAlgError:
        return None
    delta = np.linalg.solve(L.T, np.linalg.solve(L, -g))
    P = np.asarray(pose, np.float64).reshape(3, 4).copy()
    P[:, :3] = so3_exp(delta[:3]) @ P[:, :3]
    P[:, 3] = P[:, 3] + delta[3:]
    return P


def oracle_depth(verts, faces, K, pose32, h, w, near, far):
    """Step 1's default renderer: `render_oracle.render`'s depth [h,w] fp32 of one fp32 pose [3,4]."""
    return ro.render(verts, faces, K, pose32[None], h, w, near, far)[0][0]


def refine_image(mask, pose, K, verts, faces, near, far, rounds=8, gate=20.0, max_points=4096, trace=None,
                 render=None):
    """One image: mask [h,w], pose [3,4], K [3,3] -> (pose fp64 [3,4], info dict).  trace (a list) receives one dict
    per evaluation: the pose it started from, the silhouette and contour sets, X_obj, the pairs, their mean distance
    and the normal equations of each Gauss-Newton step it took.  render: step 1's renderer, called as
    `render(verts, faces, K, pose32 [3,4] fp32, h, w, near, far) -> depth [h,w] fp32` (None: `oracle_depth`)."""
    render = oracle_depth if render is None else render
    mask = np.asarray(mask)
    h, w = mask.shape
    P = np.asarray(pose, np.float64).reshape(3, 4).copy()
    con = subsample(boundary(mask != 0), max_points)
    cu_all, cv_all = centres(con, w)
    status, pairs, mean0, mean_after, mean_prev, backup = 0, 0, float("nan"), float("nan"), None, P
    for k in range(rounds + 1):
        depth = np.asarray(render(verts, faces, K, P.astype(np.float32), h, w, near, far), np.float32)
        sil = subsample(boundary(depth > 0), max_points)
        X = back_project(sil, depth, P, K, w)
        j, d2 = nearest_pairs(X, P, K, con, w, gate)
        n, m = mean_distance(j, d2)
        rec = dict(pose=P.copy(), sil=sil, con=con, X=X, pair=j, d2=d2, n=n, mean=m, normal_eq=[])
        if trace is not None:
            trace.append(rec)
        if k == 0:
            if len(con) == 0:
                status |= NO_CONTOUR
                break
            if len(sil) == 0:
                status |= NO_SILHOUETTE
                break
            if n < MIN_PAIRS:
                status |= FEW_PAIRS
                break
            mean0 = mean_after = m
        else:
            if len(sil) == 0 or n < MIN_PAIRS or m > mean_prev:
                status |= REJECTED
                P = backup
                break
            mean_after = m
        if k == rounds:
            break
        mean_prev, backup, pairs = m, P.copy(), n
        keep = j >= 0
        Xk, cu, cv = X[keep], cu_all[j[keep]], cv_all[j[keep]]
        for _ in range(GN_STEPS):
            A, g = normal_equations(Xk, cu, cv, P, K)
            rec["normal_eq"].append((A, g))
            nP = gauss_newton_step(A, g, P)
            if nP is None:
                break
            P = nP
        if nP is None:
            status |= SINGULAR
            P = backup
            break
    return P, dict(status=status, pairs=pairs, dist_before=mean0, dist_after=mean_after)


def refine(mask, poses, K, verts, faces, near, far, rounds=8, gate=20.0, max_points=4096, render=None):
    """mask [b,h,w], poses [b,3,4], K [3,3] or [b,3,3] -> poses fp64 [b,3,4], info dict of [b] arrays.  render: as
    in `refine_image`."""
    mask = np.asarray(mask)
    poses = np.asarray(poses, np.float64).reshape(-1, 3, 4)
    b = len(poses)
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    out, infos = np.empty((b, 3, 4)), []
    for i in range(b):
        out[i], info = refine_image(mask[i], poses[i], Ks[i], verts, faces, near, far, rounds, gate, max_points,
                                     render=render)
        infos.append(info)
    return out, {key: np.array([d[key] for d in infos]) for key in infos[0]}
