"""CPU oracle for the uncertainty-PnP stage (SURVEY.md section 8 row f-1) -- TEST INFRASTRUCTURE ONLY
(same rules as oracle/pvnet_oracle.py: imported by tests/, smoke() and bench.py's CPU legs only).

Restates, in numpy/scipy, what the reference computes after the voting layers (paths relative to
the reference project):

  covariance -> weights  inv(sqrtm(cov)), zeros for cov[0,0] < 1e-6 or NaN     lib/utils/evaluation_utils.py:170-181
  4 most confident points  argsort(wxx + wxy)[-4:] (sic)                         lib/utils/extend_utils/extend_utils.py:84
  P3P initialisation       cv2.solvePnP(..., flags=SOLVEPNP_P3P) on those 4      lib/utils/extend_utils/extend_utils.py:86-88
  weighted reprojection    r_i = W_i (K (R(rvec) X_i + t) / z - x_i), W_i = [[wxx,wxy],[wxy,wyy]]
                                                                                 lib/utils/extend_utils/src/uncertainty_pnp.cpp:20-37
  minimisation             Ceres 1.14 trust-region Levenberg-Marquardt, DENSE_SCHUR, default options
                                                                                 lib/utils/extend_utils/src/uncertainty_pnp.cpp:61-92

Third-party arithmetic.  Ceres (build_ceres.sh pins 1.14.0; a prebuilt libceres.so.1.14.0 sits in the
reference tree but cannot be loaded here: libglog.so.0, libspqr, libcholmod, libopenblas and libcxsparse
are absent) and OpenCV's P3P (opencv_contrib_python 3.4.2.16 in requirements.txt).  The reference result
is "the local minimiser of the cost above reached from the P3P pose" up to Ceres' stopping rule
(function_tolerance 1e-6): this oracle minimises the same cost from the same start with
scipy.optimize.least_squares(method="lm") at tight tolerances, i.e. it returns the minimiser itself.
PARITY PIN: the reference ships no test for this stage; pinned by (1) the known-answer pose of
data/demo (cat_pose.npy reprojects cat_points_3d onto the fixture's keypoints: tests/golden/pnp_cases.npz,
made by tests/golden/make_golden_pnp.py), (2) OpenCV's own P3P and iterative PnP, run when generating
the fixtures, (3) first-order optimality of the returned pose.
Ceres itself never ran: for the weighted cases parity with the reference BINARY is unpinned.
"""
from __future__ import annotations

import numpy as np


# ------------------------------------------------------------------ weights (evaluation_utils.py:170-181)
def covariance_to_weights(cov):
    """cov [pn,2,2] -> weights [pn,3] = (wxx, wxy, wyy) of inv(sqrtm(cov)); zeros where the reference
    skips the point (cov[0,0] < 1e-6 or any NaN).  Closed form of the principal square root of a 2x2
    SPD matrix: sqrt(A) = (A + sqrt(det A) I) / sqrt(tr A + 2 sqrt(det A))."""
    cov = np.asarray(cov, np.float64)
    out = np.zeros((cov.shape[0], 3))
    for i, c in enumerate(cov):
        if c[0, 0] < 1e-6 or np.isnan(c).any():
            continue
        c = 0.5 * (c + c.T)
        det = c[0, 0] * c[1, 1] - c[0, 1] * c[1, 0]
        if not det > 0:
            continue                                  # singular / indefinite: scipy's sqrtm + inv would blow up
        s = np.sqrt(det)
        root = (c + s * np.eye(2)) / np.sqrt(c[0, 0] + c[1, 1] + 2 * s)
        w = np.linalg.inv(root)
        out[i] = (w[0, 0], w[0, 1], w[1, 1])
    return out


# ------------------------------------------------------------------ rotations
def rodrigues(r):
    r = np.asarray(r).reshape(3)
    if not np.iscomplexobj(r):
        r = r.astype(np.float64)
    th = np.sqrt(r @ r)                      # analytic in r: the Jacobian below uses complex steps
    if abs(th) < 1e-12:
        k = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
        return np.eye(3) + k
    k = r / th
    kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * kx @ kx


def rotation_to_rvec(R):
    R = np.asarray(R, np.float64)
    c = np.clip((np.trace(R) - 1) / 2, -1, 1)
    th = np.arccos(c)
    if th < 1e-10:
        return np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / 2
    if np.pi - th < 1e-6:
        a = np.sqrt(np.maximum((np.diag(R) + 1) / 2, 0))
        i = int(np.argmax(a))
        v = (R[:, i] + np.eye(3)[:, i]) / (2 * a[i])
        return th * v / np.linalg.norm(v)
    return th * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]]) / (2 * np.sin(th))


# ------------------------------------------------------------------ P3P (Grunert 1841, as in Haralick et al. 1994)
def p3p(P, f):
    """P [3,3] object points, f [3,3] unit bearing vectors -> list of (R, t) with s_i f_i = R P_i + t."""
    a, b, c = np.linalg.norm(P[1] - P[2]), np.linalg.norm(P[0] - P[2]), np.linalg.norm(P[0] - P[1])
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    a2, b2, c2 = a * a, b * b, c * c
    q, p = (a2 - c2) / b2, (a2 + c2) / b2
    coef = [(q - 1) ** 2 - 4 * c2 / b2 * ca * ca,
            4 * (q * (1 - q) * cb - (1 - p) * ca * cg + 2 * c2 / b2 * ca * ca * cb),
            2 * (q * q - 1 + 2 * q * q * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * p * ca * cb * cg
                 + 2 * (b2 - a2) / b2 * cg * cg),
            4 * (-q * (1 + q) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - p) * ca * cg),
            (1 + q) ** 2 - 4 * a2 / b2 * cg * cg]
    sols = []
    for v in np.roots(coef):
        if abs(v.imag) > 1e-6 * max(1.0, abs(v.real)):
            continue
        v = v.real
        for _ in range(12):                                    # Newton polish on the quartic, to convergence (near a
            pv = np.polyval(coef, v)                           # nearly double root it converges only linearly)
            dv = np.polyval(np.polyder(coef), v)
            if dv == 0:
                break
            v -= pv / dv
            if abs(pv / dv) < 1e-15 * max(1.0, abs(v)):
                break
        den = 2 * (cg - v * ca)
        if abs(den) < 1e-14 or v <= 0:
            continue
        u = ((q - 1) * v * v - 2 * q * cb * v + 1 + q) / den
        s1sq = b2 / (1 + v * v - 2 * v * cb)
        if u <= 0 or s1sq <= 0:
            continue
        s1 = np.sqrt(s1sq)
        Q = f * np.array([s1, u * s1, v * s1])[:, None]

        def frame(X):
            e1 = X[1] - X[0]
            e1 = e1 / np.linalg.norm(e1)
            e3 = np.cross(e1, X[2] - X[0])
            e3 = e3 / np.linalg.norm(e3)
            return np.stack([e1, np.cross(e3, e1), e3], 1)
        R = frame(Q) @ frame(P).T
        sols.append((R, Q[0] - R @ P[0]))
    return sols


def p3p_init(points_2d, points_3d, K, idxs):
    """First three of `idxs` solve, the fourth disambiguates (smallest reprojection error), like
    OpenCV's SOLVEPNP_P3P.  Returns (R, t) or None."""
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    uv = points_2d[idxs]
    f = np.stack([(uv[:, 0] - cx) / fx, (uv[:, 1] - cy) / fy, np.ones(4)], 1)
    f = f / np.linalg.norm(f, axis=1, keepdims=True)
    best = None
    for R, t in p3p(points_3d[idxs[:3]], f[:3]):
        x = R @ points_3d[idxs[3]] + t
        e = np.hypot(fx * x[0] / x[2] + cx - uv[3, 0], fy * x[1] / x[2] + cy - uv[3, 1])
        if best is None or e < best[0]:
            best = (e, R, t)
    return None if best is None else (best[1], best[2])


# ------------------------------------------------------------------ the cost (uncertainty_pnp.cpp:20-37)
def residuals(pose6, points_2d, weights, points_3d, K):
    R = rodrigues(pose6[:3])
    X = points_3d @ R.T + pose6[3:]
    dx = K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2] - points_2d[:, 0]
    dy = K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2] - points_2d[:, 1]
    return np.stack([weights[:, 0] * dx + weights[:, 1] * dy, weights[:, 1] * dx + weights[:, 2] * dy], 1).ravel()


def jacobian(pose6, *args):
    """d residuals / d pose6 by complex-step differentiation (exact to rounding)."""
    cols = []
    for j in range(6):
        x = np.asarray(pose6, np.complex128).copy()
        x[j] += 1e-30j
        cols.append(residuals(x, *args).imag / 1e-30)
    return np.stack(cols, 1)


def uncertainty_pnp(points_2d, weights_2d, points_3d, camera_matrix, use_cv2_init=False):
    """extend_utils.py:63-114 -> Rt [3,4] float64.  weights_2d [pn,3] = (wxx, wxy, wyy)."""
    from scipy.optimize import least_squares
    points_2d = np.asarray(points_2d, np.float64)
    weights_2d = np.asarray(weights_2d, np.float64)
    points_3d = np.asarray(points_3d, np.float64)
    K = np.asarray(camera_matrix, np.float64)
    pn = points_2d.shape[0]
    assert points_3d.shape[0] == pn and pn >= 4
    idxs = np.argsort(weights_2d[:, 0] + weights_2d[:, 1], kind="stable")[-4:]          # :84
    init = None
    if use_cv2_init:
        import cv2
        ok, r, t = cv2.solvePnP(points_3d[idxs][None], points_2d[idxs][None], K, np.zeros((8, 1)), None, None, False,
                                flags=cv2.SOLVEPNP_P3P)
        if ok:
            init = (rodrigues(r.ravel()), t.ravel())
    if init is None:
        init = p3p_init(points_2d, points_3d, K, idxs)
    if init is None:
        init = (np.eye(3), np.array([0.0, 0.0, 1.0]))
    x0 = np.concatenate([rotation_to_rvec(init[0]), init[1]])
    if pn == 4:                                                                           # :90-94
        return np.concatenate([init[0], init[1][:, None]], 1)
    sol = least_squares(residuals, x0, jac=jacobian, args=(points_2d, weights_2d, points_3d, K), method="lm",
                        xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=2000)
    x = sol.x
    args = (points_2d, weights_2d, points_3d, K)
    for _ in range(12):                       # MINPACK stops near 1e-10: Gauss-Newton polish to the stationary point
        J, r = jacobian(x, *args), residuals(x, *args)
        d = np.linalg.solve(J.T @ J, -J.T @ r)
        x = x + d
        if np.abs(d).max() < 1e-15:
            break
    return np.concatenate([rodrigues(x[:3]), x[3:, None]], 1)
