"""numpy restatement of `pvnet_refine_poses_instances` without keypoints (csrc/refine.cu, DESIGN.md §30): silhouette
refinement of every instance of a label map.

Virtual image v = i * L + j is instance j of image i.  Everything is `oracle/refine_oracle.py`'s (render, back-projection,
subsampling, pairs, mean distance, accept / undo, Gauss-Newton), except the two boundary sets:

- contour of instance j: the pixels of value j+1 with a 4-neighbour of value 0 or on the image border (`contour`);
  a border with another instance is not outline evidence, since either instance may be in front;
- silhouette: `refine_oracle.boundary(depth > 0)`, less the pixels whose 3x3 neighbourhood, inside the image, holds a
  nonzero value other than j+1 (`silhouette`), before the max_points stride.

Values above L are other instances.  A row with j >= num[i] is not refined: it keeps its input pose with status
NO_INSTANCE.  CPU only; nothing here reads the reference."""
from __future__ import annotations

import numpy as np

from oracle import refine_oracle as ro

NO_INSTANCE = 32


def contour(labels, j):
    """labels [h,w] integer -> row-major indices of instance j's contour."""
    lab = np.asarray(labels).astype(np.int64)
    own = lab == j + 1
    p = np.pad(lab, 1, constant_values=0)
    bg_nb = (p[:-2, 1:-1] == 0) | (p[2:, 1:-1] == 0) | (p[1:-1, :-2] == 0) | (p[1:-1, 2:] == 0)
    return np.flatnonzero(own & bg_nb)


def occluded(labels, j):
    """bool [h,w]: the pixel's 3x3 neighbourhood, inside the image, holds another instance."""
    lab = np.asarray(labels).astype(np.int64)
    other = (lab != 0) & (lab != j + 1)
    h, w = lab.shape
    p = np.pad(other, 1, constant_values=False)
    out = np.zeros((h, w), bool)
    for dr in range(3):
        for dc in range(3):
            out |= p[dr:dr + h, dc:dc + w]
    return out


def silhouette(depth, labels, j):
    """Rendered depth [h,w] -> row-major indices of instance j's silhouette (before the stride)."""
    s = ro.boundary(np.asarray(depth) > 0)
    return s[~occluded(labels, j).reshape(-1)[s]]


def refine_image(labels, j, pose, K, verts, faces, near, far, rounds=8, gate=20.0, max_points=4096, trace=None,
                 render=None):
    """Instance j of one label map: `refine_oracle.refine_image` with the two boundary rules above."""
    render = ro.oracle_depth if render is None else render
    labels = np.asarray(labels)
    h, w = labels.shape
    P = np.asarray(pose, np.float64).reshape(3, 4).copy()
    con = ro.subsample(contour(labels, j), max_points)
    cu_all, cv_all = ro.centres(con, w)
    status, pairs, mean0, mean_after, mean_prev, backup = 0, 0, float("nan"), float("nan"), None, P
    for k in range(rounds + 1):
        depth = np.asarray(render(verts, faces, K, P.astype(np.float32), h, w, near, far), np.float32)
        sil = ro.subsample(silhouette(depth, labels, j), max_points)
        X = ro.back_project(sil, depth, P, K, w)
        jj, d2 = ro.nearest_pairs(X, P, K, con, w, gate)
        n, m = ro.mean_distance(jj, d2)
        rec = dict(pose=P.copy(), sil=sil, con=con, X=X, pair=jj, d2=d2, n=n, mean=m, normal_eq=[])
        if trace is not None:
            trace.append(rec)
        if k == 0:
            if len(con) == 0:
                status |= ro.NO_CONTOUR
                break
            if len(sil) == 0:
                status |= ro.NO_SILHOUETTE
                break
            if n < ro.MIN_PAIRS:
                status |= ro.FEW_PAIRS
                break
            mean0 = mean_after = m
        else:
            if len(sil) == 0 or n < ro.MIN_PAIRS or m > mean_prev:
                status |= ro.REJECTED
                P = backup
                break
            mean_after = m
        if k == rounds:
            break
        mean_prev, backup, pairs = m, P.copy(), n
        keep = jj >= 0
        Xk, cu, cv = X[keep], cu_all[jj[keep]], cv_all[jj[keep]]
        for _ in range(ro.GN_STEPS):
            A, g = ro.normal_equations(Xk, cu, cv, P, K)
            rec["normal_eq"].append((A, g))
            nP = ro.gauss_newton_step(A, g, P)
            if nP is None:
                break
            P = nP
        if nP is None:
            status |= ro.SINGULAR
            P = backup
            break
    return P, dict(status=status, pairs=pairs, dist_before=mean0, dist_after=mean_after)


def refine(labels, num, poses, K, verts, faces, near, far, rounds=8, gate=20.0, max_points=4096, render=None,
           traces=None):
    """labels [b,h,w], num [b], poses [b,L,3,4], K [3,3] or [b,3,3] -> poses fp64 [b,L,3,4], info dict of [b,L]
    arrays.  traces (a dict) receives each present row's trace under (i, j)."""
    labels = np.asarray(labels)
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
            out[i, j], d = refine_image(labels[i], j, poses[i, j], Ks[i], verts, faces, near, far, rounds, gate,
                                        max_points, trace=tr, render=render)
            if traces is not None:
                traces[(i, j)] = tr
            for key in info:
                info[key][i, j] = d[key]
    return out, info
