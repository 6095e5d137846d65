"""CPU oracle for the device EPnP (pvnet_b200/csrc/epnp.cu) -- TEST INFRASTRUCTURE ONLY.

A numpy fp64 restatement, step for step, of what the kernel computes for one image: the EPnP of Lepetit,
Moreno-Noguer and Fua ("EPnP: An Accurate O(n) Solution to the PnP Problem", IJCV 81(2), 2009), which the
reference reaches through `cv2.solvePnP(..., flags=cv2.SOLVEPNP_EPNP)` in lib/utils/evaluation_utils.py:19-52.

  1. control points: c0 = centroid of the object points; c1..c3 = c0 + sqrt(lambda_k / n) v_k from the PCA of the
     centred points, largest variance first.  The PCA is a cyclic one-sided (Hestenes) Jacobi started from the
     identity (`pca3`); the signs of its v_k decide which control points EPnP uses, and with noisy image points the
     pose depends on them.  These signs are the ones OpenCV's output shows.
  2. barycentric coordinates alpha [n,4] of every object point (closed form: the v_k are orthonormal).
  3. M^T M (12x12) of the 2n x 12 system M from fx, fy, cx, cy, summed from 40 per-point moments.
  4. v[0..3]: the eigenvectors of its four smallest eigenvalues, v[0] the smallest.
  5. L (6x10) and rho (6) over the control-point pairs (0,1),(0,2),(0,3),(1,2),(1,3),(2,3).
  6. betas by three linearisations, N = 1: (b11, b12, b13, b14); N = 2: (b11, b12, b22); N = 3: (b11, b12, b22,
     b13, b23), each followed by 5 Gauss-Newton steps on all four betas.
  7. per N: camera-frame control points sum_k beta_k v[k], flipped as a whole when the first object point lands
     behind the camera (z < 0); R, t by the SVD Procrustes fit, a reflection made a rotation by negating its
     third row (`procrustes`); mean reprojection error in
     pixels.
  8. the N with the smallest error; a later N must be strictly smaller to win (N = 1, then 2, then 3).

Status bit 1: the smallest PCA eigenvalue is <= PCA_DEGENERATE (1e-10) times the largest (coplanar or collinear
object points).  The control points then use that floor in place of the eigenvalue, so they stay distinct and the
pose is still computed.
"""
from __future__ import annotations

import numpy as np

PAIRS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
GN_STEPS = 5
PCA_DEGENERATE = 1e-10
PCA_SWEEPS = 30
STATUS_DEGENERATE = 1


def pca3(A):
    """Eigen-decomposition of the symmetric PSD 3x3 A by cyclic one-sided Jacobi on its rows, from V = I, at most
    PCA_SWEEPS sweeps over the pairs (0,1), (0,2), (1,2).  Each rotation leaves the larger row norm in the lower
    index.  -> (lam [3] descending, V [3,3] whose ROWS are the unit eigenvectors)."""
    A = np.array(A, np.float64)
    V = np.eye(3)
    w = (A * A).sum(1)
    for _ in range(PCA_SWEEPS):
        changed = False
        for i, j in ((0, 1), (0, 2), (1, 2)):
            a, b, p = w[i], w[j], A[i] @ A[j]
            if not abs(p) > 2.2e-15 * np.sqrt(a * b):
                continue
            p *= 2.0
            beta = a - b
            gamma = np.hypot(p, beta)
            if beta < 0:
                s = np.sqrt((gamma - beta) * 0.5 / gamma)
                c = p / (gamma * s * 2.0)
            else:
                c = np.sqrt((gamma + beta) / (gamma * 2.0))
                s = p / (gamma * c * 2.0)
            A[i], A[j] = c * A[i] + s * A[j], -s * A[i] + c * A[j]
            V[i], V[j] = c * V[i] + s * V[j], -s * V[i] + c * V[j]
            w[i], w[j] = A[i] @ A[i], A[j] @ A[j]
            changed = True
        if not changed:
            break
    lam = np.sqrt((A * A).sum(1))
    order = np.argsort(-lam, kind="stable")
    return lam[order], V[order]


def procrustes(H):
    """R from the SVD H = U S V^T of the cross-covariance H = sum (pc - pc0)(pw - pw0)^T: R = U V^T, and where that
    is a reflection (det < 0) its third row is negated, which makes it a rotation.  (This, not the closest rotation
    U diag(1, 1, -1) V^T, is the fix whose poses OpenCV's output shows: the two differ only where the fit is a
    reflection, and there the pose is poor either way; but the fix changes the reprojection error, and so which N
    wins.)"""
    U, _, Vt = np.linalg.svd(H)
    R = U @ Vt
    if np.linalg.det(R) < 0:
        R[2] = -R[2]
    return R


def _lstsq(A, b):
    return np.linalg.lstsq(A, b, rcond=None)[0]


def _gauss_newton(L, rho, betas):
    b = np.array(betas, np.float64)
    for _ in range(GN_STEPS):
        J = np.stack([2 * L[:, 0] * b[0] + L[:, 1] * b[1] + L[:, 3] * b[2] + L[:, 6] * b[3],
                      L[:, 1] * b[0] + 2 * L[:, 2] * b[1] + L[:, 4] * b[2] + L[:, 7] * b[3],
                      L[:, 3] * b[0] + L[:, 4] * b[1] + 2 * L[:, 5] * b[2] + L[:, 8] * b[3],
                      L[:, 6] * b[0] + L[:, 7] * b[1] + L[:, 8] * b[2] + 2 * L[:, 9] * b[3]], 1)
        q = np.array([b[0] * b[0], b[0] * b[1], b[1] * b[1], b[0] * b[2], b[1] * b[2], b[2] * b[2],
                      b[0] * b[3], b[1] * b[3], b[2] * b[3], b[3] * b[3]])
        b = b + _lstsq(J, rho - L @ q)
    return b


def _betas(L, rho, N):
    """The linearised betas of step 6 before Gauss-Newton."""
    if N == 1:
        x = _lstsq(L[:, [0, 1, 3, 6]], rho)                 # b11 b12 b13 b14
        b0 = np.sqrt(abs(x[0]))
        s = -1.0 if x[0] < 0 else 1.0
        return np.array([b0, s * x[1] / b0, s * x[2] / b0, s * x[3] / b0])
    x = _lstsq(L[:, [0, 1, 2]] if N == 2 else L[:, [0, 1, 2, 3, 4]], rho)   # b11 b12 b22 (b13 b23)
    if x[0] < 0:
        b0, b1 = np.sqrt(-x[0]), (np.sqrt(-x[2]) if x[2] < 0 else 0.0)
    else:
        b0, b1 = np.sqrt(x[0]), (np.sqrt(x[2]) if x[2] > 0 else 0.0)
    if x[1] < 0:
        b0 = -b0
    return np.array([b0, b1, x[3] / b0 if N == 3 else 0.0, 0.0])


def epnp(points_2d, points_3d, camera_matrix):
    """points_2d [n,2], points_3d [n,3] (float32 values, as the device reads them), camera_matrix [3,3] (fx, fy, cx,
    cy are read).  -> dict(pose [3,4], N (1..3), status, errors [3] (mean reprojection error of N = 1, 2, 3, pixels),
    eig [12] (eigenvalues of M^T M, ascending), gap, pca [3]).  gap = min over k < 4 of (eig[k+1] - eig[k]) / eig[11]:
    where it is tiny the four null-space vectors, and so the start of Gauss-Newton, are set by rounding rather than
    by the problem; with 5 points M has a two-dimensional null space and the gap is at rounding level."""
    x = np.asarray(points_2d, np.float64)
    P = np.asarray(points_3d, np.float64)
    K = np.asarray(camera_matrix, np.float64)
    fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    n = len(P)
    status = 0
    # 1. control points
    c0 = P.sum(0) / n
    D = P - c0
    A = D.T @ D
    lam, V = pca3(A)
    if not lam[2] > PCA_DEGENERATE * lam[0]:
        status |= STATUS_DEGENERATE
    sk = np.sqrt(np.maximum(lam, PCA_DEGENERATE * lam[0]) / n)
    C = np.stack([c0] + [c0 + sk[k] * V[k] for k in range(3)])
    # 2. barycentric coordinates
    a = (D @ V.T) / sk                                       # [n,3]
    alpha = np.concatenate([1.0 - a.sum(1, keepdims=True), a], 1)
    # 3. M^T M from the moments of (alpha_j alpha_k) x (1, cx - u, cy - v, (cx - u)^2 + (cy - v)^2)
    du, dv = cx - x[:, 0], cy - x[:, 1]
    aa = alpha[:, :, None] * alpha[:, None, :]               # [n,4,4]
    S1 = aa.sum(0)
    Su = (aa * du[:, None, None]).sum(0)
    Sv = (aa * dv[:, None, None]).sum(0)
    Sw = (aa * (du * du + dv * dv)[:, None, None]).sum(0)
    MtM = np.zeros((12, 12))
    for j in range(4):
        for k in range(4):
            B = MtM[3 * j:3 * j + 3, 3 * k:3 * k + 3]
            B[0, 0] = fx * fx * S1[j, k]
            B[1, 1] = fy * fy * S1[j, k]
            B[0, 2] = fx * Su[j, k]
            B[2, 0] = fx * Su[j, k]
            B[1, 2] = fy * Sv[j, k]
            B[2, 1] = fy * Sv[j, k]
            B[2, 2] = Sw[j, k]
    # 4. null-space basis
    eig, U = np.linalg.eigh(MtM)
    v = [U[:, k].reshape(4, 3) for k in range(4)]
    # 5. L and rho
    L = np.zeros((6, 10))
    rho = np.zeros(6)
    for r, (i, j) in enumerate(PAIRS):
        d = [vk[i] - vk[j] for vk in v]
        L[r] = [d[0] @ d[0], 2 * d[0] @ d[1], d[1] @ d[1], 2 * d[0] @ d[2], 2 * d[1] @ d[2], d[2] @ d[2],
                2 * d[0] @ d[3], 2 * d[1] @ d[3], 2 * d[2] @ d[3], d[3] @ d[3]]
        rho[r] = (C[i] - C[j]) @ (C[i] - C[j])
    # Procrustes moments: with pc_i = sum_j alpha_ij ccs_j, the centred cross-covariance sum (pc_i - pc0)(p_i - c0)^T
    # is sum_{k=1..3} (ccs_k - ccs_0) Q_k^T, Q_k = sum_i a_ik (p_i - c0) = A V_k / s_k, and pc0 = ccs_0
    Q = (V @ A) / sk[:, None]                                # [3,3] rows Q_k
    poses, errors = [], []
    for N in (1, 2, 3):
        b = _gauss_newton(L, rho, _betas(L, rho, N))
        ccs = sum(b[k] * v[k] for k in range(4))             # [4,3]
        if alpha[0] @ ccs[:, 2] < 0:
            ccs = -ccs
        H = (ccs[1:] - ccs[0]).T @ Q
        R = procrustes(H)
        t = ccs[0] - R @ c0
        Xc = P @ R.T + t
        err = np.mean(np.hypot(fx * Xc[:, 0] / Xc[:, 2] + cx - x[:, 0], fy * Xc[:, 1] / Xc[:, 2] + cy - x[:, 1]))
        poses.append(np.concatenate([R, t[:, None]], 1))
        errors.append(err)
    best = 0
    if errors[1] < errors[best]:
        best = 1
    if errors[2] < errors[best]:
        best = 2
    return dict(pose=poses[best], N=best + 1, status=status, errors=np.array(errors), eig=eig,
                gap=np.diff(eig[:5]).min() / eig[11], pca=lam)


def selection_tie(errors, rel=1e-9):
    """True where the chosen N is not separated from another N by more than `rel` of the larger error (plus rel px):
    rounding, not the problem, then decides which N wins."""
    e = np.sort(np.asarray(errors, np.float64))
    return bool(e[1] - e[0] <= rel * (e[1] + 1.0))
