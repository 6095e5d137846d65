"""numpy restatement of `pvnet_refine_poses_keypoints` (csrc/refine.cu, DESIGN.md §27): `refine_oracle`'s silhouette
refinement (§26) with the voted keypoints added to its objective.  Steps 1-4 (render, silhouette, contour, pairs) and
the mean pair distance are refine_oracle's own functions; this module adds:

5. Keypoint k (x_k fp32, P_k fp32, W_k = [[wxx, wxy], [wxy, wyy]] from fp32 weights, all widened to fp64) sits on
   lane k of one warp; a keypoint with a non-finite entry is left out (it adds zero).  Its distance at pose P is
   |W_k (pi(P_k) - x_k)|: refine_oracle.project's u, v, e = (u - x, v - y), r = (wxx eu + wxy ev, wxy eu + wyy ev),
   sqrt(r0 r0 + r1 r1), each operation rounded -- bit for bit the kernel's.  `warp_sum` adds the 32 lanes' values
   by xor butterflies, kd; the round's cost is C = m + lambda * (kd / nk), m the mean pair distance.  C replaces
   m in refine_oracle's accept / undo rule, so it too is the kernel's decision by construction.
6. Each Gauss-Newton step's system is, entry by entry, A_pair / n + (lambda / nk) * A_kp (and g alike), n the
   round's pair count, A_pair, g_pair refine_oracle.normal_equations of the pairs, and A_kp, g_kp the sums of
   J_w^T J_w and J_w^T r over the keypoints at the current pose, J_w = W_k [d u; d v] in (dw, dt).  The kernel sums
   A_kp over warp 0 by `warp_sum`'s butterflies and adds it to the pair sums after `block_sum`; numpy sums it here
   (to rounding).  The step itself is refine_oracle.gauss_newton_step.

CPU only by default (the render step is refine_oracle's `render=` parameter); nothing here reads the reference."""
from __future__ import annotations

import numpy as np

from oracle import refine_oracle as rfo


def warp_sum(x):
    """Sum of fp64 x [<= 32] over one warp, lane l holding x[l] (0.0 past the end): xor butterflies at offsets 16, 8,
    4, 2, 1 (lane l adds lane l ^ o's value), then lane 0's value."""
    lanes = np.zeros(32)
    lanes[:len(x)] = np.asarray(x, np.float64)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[np.arange(32) ^ o]
    return float(lanes[0])


class Keypoints:
    """One image's keypoint term: keypoints [nk,2], model points [nk,3], weights [nk,3] = (wxx, wxy, wyy), all read
    as fp32 and widened; lambda = keypoint_weight.  `on` marks the keypoints the term uses (every entry finite)."""

    def __init__(self, keypoints, points_3d, weights, keypoint_weight):
        self.x = np.asarray(keypoints, np.float32).astype(np.float64).reshape(-1, 2)
        self.P = np.asarray(points_3d, np.float32).astype(np.float64).reshape(-1, 3)
        self.w = np.asarray(weights, np.float32).astype(np.float64).reshape(-1, 3)
        self.nk = len(self.x)
        self.lam = float(keypoint_weight)
        self.on = np.isfinite(self.x).all(1) & np.isfinite(self.P).all(1) & np.isfinite(self.w).all(1)

    def _kept(self):
        return self.x[self.on], self.P[self.on], self.w[self.on]

    def residuals(self, pose, K):
        """-> r [nk_on,2] = W_k (pi(R P_k + t) - x_k) of the kept keypoints."""
        x, P, w = self._kept()
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            u, v = rfo.project(P, pose, K)
        eu, ev = u - x[:, 0], v - x[:, 1]
        return np.stack([w[:, 0] * eu + w[:, 1] * ev, w[:, 1] * eu + w[:, 2] * ev], -1)

    def distance_sum(self, pose, K):
        """kd: warp_sum of |r_k| on lane k (0 for a left-out keypoint), the kernel's operations."""
        d = np.zeros(self.nk)
        r = self.residuals(pose, K)
        d[self.on] = np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1])
        return warp_sum(d)

    def cost(self, m, pose, K):
        """C = m + lambda * (kd / nk)."""
        return m + self.lam * (self.distance_sum(pose, K) / self.nk)

    def jacobian(self, pose, K):
        """-> J_w [nk_on,2,6]: d r / d(dw, dt) for R <- exp(dw) R, t <- t + dt."""
        x, P, w = self._kept()
        fx, s, cx, fy, cy = rfo._camera(K)
        Pm = np.asarray(pose, np.float64).reshape(3, 4)
        p = np.stack([(Pm[r, 0] * P[:, 0] + Pm[r, 1] * P[:, 1]) + Pm[r, 2] * P[:, 2] for r in range(3)], -1)
        Xc = p + Pm[:, 3]
        iz = 1.0 / Xc[:, 2]
        u = ((fx * Xc[:, 0] + s * Xc[:, 1]) + cx * Xc[:, 2]) * iz
        v = (fy * Xc[:, 1] + cy * Xc[:, 2]) * iz
        zero = np.zeros_like(iz)
        du = np.stack([fx * iz, s * iz, -(u - cx) * iz], -1)
        dv = np.stack([zero, fy * iz, -(v - cy) * iz], -1)
        Ju = np.concatenate([np.cross(p, du), du], -1)
        Jv = np.concatenate([np.cross(p, dv), dv], -1)
        return np.stack([w[:, :1] * Ju + w[:, 1:2] * Jv, w[:, 1:2] * Ju + w[:, 2:3] * Jv], 1)

    def normal_equations(self, pose, K):
        """-> A_kp [6,6], g_kp [6]: sum_k J_w^T J_w and J_w^T r, unscaled."""
        J = self.jacobian(pose, K).reshape(-1, 6)
        r = self.residuals(pose, K).reshape(-1)
        return J.T @ J, J.T @ r

    def combine(self, A, g, n, Ak, gk):
        """The step's system: A / n + (lambda / nk) * A_kp, g likewise, each operation rounded."""
        lk = self.lam / self.nk
        return A / n + lk * Ak, g / n + lk * gk




def refine_image(mask, pose, K, verts, faces, near, far, keypoints, points_3d, weights, keypoint_weight=1.0, rounds=8,
                 gate=20.0, max_points=4096, trace=None, render=None):
    """One image: mask [h,w], pose [3,4], K [3,3], keypoints [nk,2], points_3d [nk,3], weights [nk,3] -> (pose fp64
    [3,4], info dict: refine_oracle.refine_image's keys plus "cost_before" / "cost_after").  trace (a list) receives
    one dict per evaluation: refine_oracle's record plus "cost", "kd" and "kp_eq" (the keypoint sums of each step).
    render: as in refine_oracle.refine_image."""
    render = rfo.oracle_depth if render is None else render
    kpt = Keypoints(keypoints, points_3d, weights, keypoint_weight)
    mask = np.asarray(mask)
    h, w = mask.shape
    P = np.asarray(pose, np.float64).reshape(3, 4).copy()
    con = rfo.subsample(rfo.boundary(mask != 0), max_points)
    cu_all, cv_all = rfo.centres(con, w)
    status, pairs, mean0, mean_after, backup = 0, 0, float("nan"), float("nan"), P
    cost0, cost_after, cost_prev = float("nan"), float("nan"), None
    for k in range(rounds + 1):
        depth = np.asarray(render(verts, faces, K, P.astype(np.float32), h, w, near, far), np.float32)
        sil = rfo.subsample(rfo.boundary(depth > 0), max_points)
        X = rfo.back_project(sil, depth, P, K, w)
        j, d2 = rfo.nearest_pairs(X, P, K, con, w, gate)
        n, m = rfo.mean_distance(j, d2)
        with np.errstate(invalid="ignore"):
            c = kpt.cost(m, P, K)
        rec = dict(pose=P.copy(), sil=sil, con=con, X=X, pair=j, d2=d2, n=n, mean=m, normal_eq=[], cost=c,
                   kd=kpt.distance_sum(P, K), kp_eq=[])
        if trace is not None:
            trace.append(rec)
        if k == 0:
            if len(con) == 0:
                status |= rfo.NO_CONTOUR
                break
            if len(sil) == 0:
                status |= rfo.NO_SILHOUETTE
                break
            if n < rfo.MIN_PAIRS:
                status |= rfo.FEW_PAIRS
                break
            mean0 = mean_after = m
            cost0 = cost_after = c
        else:
            if len(sil) == 0 or n < rfo.MIN_PAIRS or not c <= cost_prev:              # a NaN C is undone
                status |= rfo.REJECTED
                P = backup
                break
            mean_after, cost_after = m, c
        if k == rounds:
            break
        cost_prev, backup, pairs = c, P.copy(), n
        keep = j >= 0
        Xk, cu, cv = X[keep], cu_all[j[keep]], cv_all[j[keep]]
        for _ in range(rfo.GN_STEPS):
            A, g = rfo.normal_equations(Xk, cu, cv, P, K)
            rec["normal_eq"].append((A, g))
            Ak, gk = kpt.normal_equations(P, K)
            rec["kp_eq"].append((Ak, gk))
            nP = rfo.gauss_newton_step(*kpt.combine(A, g, n, Ak, gk), P)
            if nP is None:
                break
            P = nP
        if nP is None:
            status |= rfo.SINGULAR
            P = backup
            break
    return P, dict(status=status, pairs=pairs, dist_before=mean0, dist_after=mean_after, cost_before=cost0,
                   cost_after=cost_after)


def refine(mask, poses, K, verts, faces, near, far, keypoints, points_3d, weights, keypoint_weight=1.0, rounds=8,
           gate=20.0, max_points=4096, render=None):
    """mask [b,h,w], poses [b,3,4], K [3,3] or [b,3,3], keypoints [b,nk,2], points_3d [nk,3], weights [b,nk,3] ->
    poses fp64 [b,3,4], info dict of [b] arrays."""
    mask = np.asarray(mask)
    poses = np.asarray(poses, np.float64).reshape(-1, 3, 4)
    b = len(poses)
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    out, infos = np.empty((b, 3, 4)), []
    for i in range(b):
        out[i], info = refine_image(mask[i], poses[i], Ks[i], verts, faces, near, far, keypoints[i], points_3d,
                                     weights[i], keypoint_weight, rounds, gate, max_points, render=render)
        infos.append(info)
    return out, {key: np.array([d[key] for d in infos]) for key in infos[0]}
