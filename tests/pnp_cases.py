"""Seeded uncertainty-PnP problems, regenerated from their names: object points, generating pose, intrinsics,
float32 keypoints and float32 covariances or weights.  Shared by tests/test_pnp_cases_cpu.py (the fp64 oracle on
them) and tests/test_gpu_pnp_edges.py (the device solver against the oracle).

Every problem of one batch shares its object points and camera matrix, as one `pvnet_uncertainty_pnp` call does.
Regimes:
  cat      the LINEMOD cat's 9 keypoints (tests/golden/pnp_cases.npz), LINEMOD intrinsics, 0.5-1.5 m
  cloud    a random 0.2 m cloud, LINEMOD intrinsics, 0.5-1.5 m
  close    a random 0.2 m cloud at 0.25-0.4 m
  aniso_K  a random 0.2 m cloud, fx = 420, fy = 910 and a principal point far off the image centre
  mm       a random 0.2 m cloud in millimetres (object points and translation x 1000), LINEMOD intrinsics
"""
import os
import zlib

import numpy as np

from oracle import pnp_oracle as pn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_cases.npz")
K_LINEMOD = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])
K_ANISO = np.array([[420.0, 0., 505.5], [0., 910.0, 61.25], [0., 0., 1.]])
REGIMES = ("cat", "cloud", "close", "aniso_K", "mm")

# noise-free pn == 4 batches: (name, regime); each holds P3P_BATCH images, more than the 592 above which the solver
# puts 4 warps in one CTA
P3P_BATCH = 1024
P3P_BATCHES = [("cat_a", "cat"), ("cat_b", "cat"), ("cloud_a", "cloud"), ("cloud_b", "cloud"), ("close", "close"),
               ("aniso_K", "aniso_K"), ("mm", "mm")]
# Images where the fp64 oracle's P3P, given the EXACT (float64) projections, misses the generating pose by more than
# 1e-6: the quartic has a nearly double root there (the camera near P3P's danger cylinder), which fp64 cannot separate
# to that accuracy.  45 of 7168; tests/test_pnp_cases_cpu.py checks that no other image misses.
ORACLE_ILL_CONDITIONED = {
    "cat_a": (50, 234, 481, 504, 984),
    "cat_b": (193, 625, 629, 825),
    "cloud_a": (89, 96, 173, 194, 234, 243, 250, 305, 390, 422, 456, 552, 681, 730, 760, 770, 790),
    "close": (482, 659),
    "aniso_K": (322, 333, 351, 379, 535, 614, 758, 804, 813, 817, 871, 933, 941, 981),
    "mm": (587, 848, 892),
}

# point count -> regime of its noisy batch (random intrinsics for the random clouds)
POINT_COUNTS = {5: "cat", 6: "close", 7: "aniso_K", 8: "mm", 9: "cat", 16: "mm", 17: "cloud", 31: "close", 32: "cloud"}


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


def unit(regime):
    """Length unit of the regime in metres^-1: translation errors are divided by it before they are compared."""
    return 1000.0 if regime == "mm" else 1.0


def camera(regime, rng=None):
    """3x3 float64; rng given: random intrinsics (fx, fy in [400, 900], principal point anywhere near the image)."""
    if rng is not None:
        fx, fy = rng.uniform(400, 900, 2)
        return np.array([[fx, 0, rng.uniform(200, 450)], [0, fy, rng.uniform(150, 330)], [0, 0, 1.0]])
    return K_ANISO if regime == "aniso_K" else K_LINEMOD


def object_points(regime, pn_, rng):
    """float32 [pn,3] in the regime's unit."""
    if regime == "cat":
        cat = np.load(GOLDEN)["points_3d"]
        assert pn_ <= len(cat)
        P = cat[rng.choice(len(cat), pn_, replace=False)]
    else:
        P = rng.uniform(-0.1, 0.1, (pn_, 3))
    return (P * unit(regime)).astype(np.float32)


def poses(regime, n, rng):
    """R [n,3,3], t [n,3] (t in the regime's unit)."""
    R = np.stack([pn.rodrigues(rng.normal(0, 1.0, 3)) for _ in range(n)])
    lo, hi = (0.25, 0.4) if regime == "close" else (0.5, 1.5)
    z = rng.uniform(lo, hi, n)
    t = np.stack([rng.uniform(-0.15, 0.15, n) * z, rng.uniform(-0.15, 0.15, n) * z, z], 1)
    return R, t * unit(regime)


def project(P, R, t, K):
    """float64 pixels [n,pn,2] of the object points P [pn,3] under poses R [n,3,3], t [n,3]."""
    X = np.einsum("nij,pj->npi", R, np.asarray(P, np.float64)) + t[:, None]
    return np.stack([K[0, 0] * X[..., 0] / X[..., 2] + K[0, 2], K[1, 1] * X[..., 1] / X[..., 2] + K[1, 2]], -1)


def iso_weights(rng, n, pn_):
    """float32 [n,pn,3] isotropic weights k I with distinct keys k in shuffled order."""
    k = np.stack([rng.permutation(pn_) for _ in range(n)]).astype(np.float32) * 0.25 + 0.5
    return np.stack([k, np.zeros_like(k), k], -1)


def random_cov(rng, shape):
    """float64 [*shape,2,2] anisotropic, correlated covariances (pixels^2)."""
    A = rng.normal(0, 1, shape + (2, 2))
    return A @ np.swapaxes(A, -1, -2) + 0.2 * np.eye(2)


def noisy(rng, uv, cov):
    """uv + a draw of N(0, cov) per keypoint, as float32."""
    L = np.linalg.cholesky(cov)
    return (uv + np.einsum("...ij,...j->...i", L, rng.normal(0, 1, uv.shape))).astype(np.float32)


def pose_error(Rt, R, t, u=1.0):
    """max(|dR|, |dt| / u) of a [3,4] pose against (R, t)."""
    return max(np.abs(Rt[:, :3] - R).max(), np.abs(Rt[:, 3] - t).max() / u)


def p3p_batch(name):
    """Noise-free pn == 4 problems: dict(P float32 [4,3], K, R [n,3,3], t [n,3], kp float32 [n,4,2],
    w float32 [n,4,3] (isotropic, distinct keys in shuffled order, so every image solves from its own three points),
    unit)."""
    regime = dict(P3P_BATCHES)[name]
    rng = _rng("p3p/" + name)
    P = object_points(regime, 4, rng)
    K = camera(regime)
    R, t = poses(regime, P3P_BATCH, rng)
    kp = project(P, R, t, K).astype(np.float32)
    return dict(P=P, K=K, R=R, t=t, kp=kp, w=iso_weights(rng, P3P_BATCH, 4), unit=unit(regime))


def oracle_p3p(kp, w, P, K):
    """The oracle's pn == 4 answer (P3P on argsort(wxx + wxy), first three solve) on the float32 inputs, or None."""
    idxs = np.argsort(w[:, 0].astype(np.float64) + w[:, 1], kind="stable")[-4:]
    got = pn.p3p_init(kp.astype(np.float64), P.astype(np.float64), K, idxs)
    return None if got is None else np.concatenate([got[0], got[1][:, None]], 1)


# ------------------------------------------------------------------ weights that make the selection order matter
def cov_from_weight(W):
    """float32 covariance whose inv(sqrtm) is the SPD 2x2 W (float64 [2,2])."""
    return np.linalg.inv(W @ W).astype(np.float32)


W_NEGATIVE_KEY = np.array([[1.0, -2.0], [-2.0, 5.0]])       # SPD, wxx + wxy = -1
FILTERED_COVS = {
    "tiny": np.array([[5e-7, 0.0], [0.0, 1.0]], np.float32),           # cov[0,0] < 1e-6
    "nan": np.array([[1.0, np.nan], [0.0, 1.0]], np.float32),          # a NaN element
    "indefinite": np.array([[1.0, 2.0], [2.0, 1.0]], np.float32),      # not positive definite
}


def noisy_problems(name, pn_, n, regime="cloud"):
    """Noisy problems with random anisotropic covariances: dict(P, K, R, t, kp float32 [n,pn,2],
    cov float32 [n,pn,2,2], unit)."""
    rng = _rng(name)
    P = object_points(regime, pn_, rng)
    K = camera(regime, rng if regime in ("cloud", "close", "mm") else None)
    R, t = poses(regime, n, rng)
    cov = random_cov(rng, (n, pn_))
    kp = noisy(rng, project(P, R, t, K), cov)
    return dict(P=P, K=K, R=R, t=t, kp=kp, cov=cov.astype(np.float32), unit=unit(regime))
