"""GPU: pvnet_uncertainty_pnp at its edges, against the fp64 oracle (oracle/pnp_oracle.py) on the same float32
inputs, with the problems of tests/pnp_cases.py.

- P3P at scale: 7,168 noise-free pn == 4 images (every regime, 4 warps per CTA) return the generating pose as
  closely as the oracle's own P3P does on the same float32 keypoints.
- Selection order: pn == 4 with noisy keypoints, so that which three points solve changes the answer.
- Point counts 5..32, launch shapes around the 1-warp / 4-warp switch, filtered keypoints, and the invariances
  of the cost under exact rescaling of the weights and of the object points."""
import numpy as np
import pytest
import torch

from oracle import pnp_oracle as pn
from pvnet_b200 import extend_utils as eu
from tests import pnp_cases as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _solve(kp, P, K, w=None, cov=None):
    poses, info = eu.uncertainty_pnp_batched(
        torch.from_numpy(np.ascontiguousarray(kp)).to(DEV), P, K,
        weights_2d=None if w is None else torch.from_numpy(np.ascontiguousarray(w, np.float32)).to(DEV),
        cov=None if cov is None else torch.from_numpy(np.ascontiguousarray(cov, np.float32)).to(DEV),
        return_info=True)
    return poses.cpu().numpy(), info.cpu().numpy()


def _weights32(cov):
    """float32 weights [..., 3] of float32 covariances [..., 2, 2] (the oracle's closed form, rounded)."""
    flat = cov.reshape(-1, 2, 2)
    return pn.covariance_to_weights(flat).astype(np.float32).reshape(cov.shape[:-2] + (3,))


def _cosines(Rt, kp, w, P, K):
    """|(J^T r)_j| / (|J_j| |r|) at the pose Rt of the oracle's fp64 cost: the cosine between the residual vector and
    each Jacobian column, zero at a stationary point whatever the units of the six parameters."""
    x = np.concatenate([pn.rotation_to_rvec(Rt[:, :3]), Rt[:, 3]])
    args = (kp.astype(np.float64), np.asarray(w, np.float64), P.astype(np.float64), K)
    J, r = pn.jacobian(x, *args), pn.residuals(x, *args)
    return np.abs(J.T @ r) / (np.linalg.norm(J, axis=0) * np.linalg.norm(r))


# ------------------------------------------------------------------ P3P at scale
def test_p3p_at_scale_returns_the_generating_pose():
    """Bar per image: |device - truth| <= max(1e-6, 4 |oracle - truth|), both P3P on the same float32 keypoints (their
    rounding alone moves the pose by up to ~5e-4), and status bit 1 clear wherever the oracle found a solution.
    Translation errors are in metres (the mm batch's are divided by 1000).  The images listed in
    pc.ORACLE_ILL_CONDITIONED (a nearly double quartic root even on exact input) are held to the status bit only."""
    total, failed, worst = 0, [], (0.0, None)
    for name, _ in pc.P3P_BATCHES:
        c = pc.p3p_batch(name)
        poses, info = _solve(c["kp"], c["P"], c["K"], w=c["w"])
        listed = set(pc.ORACLE_ILL_CONDITIONED.get(name, ()))
        for i in range(pc.P3P_BATCH):
            ref = pc.oracle_p3p(c["kp"][i], c["w"][i], c["P"], c["K"])
            if ref is None:
                continue
            total += 1
            err = pc.pose_error(poses[i], c["R"][i], c["t"][i], c["unit"])
            bar = max(1e-6, 4 * pc.pose_error(ref, c["R"][i], c["t"][i], c["unit"]))
            if info[i, 0] & 1 or (i not in listed and not err <= bar):
                failed.append((name, i, err, bar, int(info[i, 0])))
            if i not in listed and err > worst[0]:
                worst = (err, (name, i))
    assert total >= 4096
    assert not failed, f"{len(failed)} of {total} images: worst {worst}; first {failed[:8]}"


# ------------------------------------------------------------------ which four points, in which order
SELECTION = ("distinct", "all_equal", "zero_weight", "negative_key")


def _selection_case(kind, n=256):
    c = pc.noisy_problems("select/" + kind, 4, n, "cloud")
    rng = np.random.default_rng(len(kind))
    w = _weights32(c["cov"])
    if kind == "all_equal":
        w[:] = w[:, :1]
    elif kind == "zero_weight":
        w[np.arange(n), rng.integers(0, 4, n)] = 0.0
    elif kind == "negative_key":
        neg = pn.covariance_to_weights(pc.cov_from_weight(pc.W_NEGATIVE_KEY)[None])[0].astype(np.float32)
        w[np.arange(n), rng.integers(0, 4, n)] = neg * rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    return c, w


def _min_root_gap(kp, w, P, K):
    """Smallest distance between two roots (complex included) of the Grunert quartic the P3P start solves: the same
    coefficients as oracle/pnp_oracle.p3p, on the points argsort(wxx + wxy, stable)[-4:] selects."""
    idxs = np.argsort(w[:, 0].astype(np.float64) + w[:, 1], kind="stable")[-4:]
    uv, Q = kp.astype(np.float64)[idxs], P.astype(np.float64)[idxs]
    f = np.stack([(uv[:, 0] - K[0, 2]) / K[0, 0], (uv[:, 1] - K[1, 2]) / K[1, 1], np.ones(4)], 1)
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    a2, b2, c2 = ((Q[1] - Q[2]) ** 2).sum(), ((Q[0] - Q[2]) ** 2).sum(), ((Q[0] - Q[1]) ** 2).sum()
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    q, p = (a2 - c2) / b2, (a2 + c2) / b2
    coef = [(q - 1) ** 2 - 4 * c2 / b2 * ca * ca,
            4 * (q * (1 - q) * cb - (1 - p) * ca * cg + 2 * c2 / b2 * ca * ca * cb),
            2 * (q * q - 1 + 2 * q * q * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * p * ca * cb * cg
                 + 2 * (b2 - a2) / b2 * cg * cg),
            4 * (-q * (1 + q) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - p) * ca * cg),
            (1 + q) ** 2 - 4 * a2 / b2 * cg * cg]
    r = np.roots(coef)
    return min(abs(a - b) for j, a in enumerate(r) for b in r[j + 1:])


@pytest.mark.parametrize("kind", SELECTION)
def test_p3p_selection_order_matches_stable_argsort(kind):
    """pn == 4 returns the P3P pose from argsort(wxx + wxy, stable)[-4:], first three solving.  Noisy keypoints make
    every choice of three give a different pose (~1e-3 apart), so only the reference's order matches to 1e-8.
    Well-conditioned images are those whose quartic has its four roots pairwise at least 2e-2 apart.  Where two
    roots are closer, the pose follows the fp64 rounding of the quartic's coefficients, which device and oracle
    round differently.  Observed differences there reach 4e-5.  Those images are held to 1e-4 instead, which still
    separates the reference's order from any other."""
    c, w = _selection_case(kind)
    poses, info = _solve(c["kp"], c["P"], c["K"], w=w)
    P64 = c["P"].astype(np.float64)
    err = np.array([np.abs(poses[i] - pn.uncertainty_pnp(c["kp"][i], w[i], P64, c["K"])).max() for i in range(len(w))])
    gap = np.array([_min_root_gap(c["kp"][i], w[i], c["P"], c["K"]) for i in range(len(w))])
    assert (info[:, 0] == 0).all(), info[info[:, 0] != 0]
    assert (gap >= 2e-2).sum() >= 0.7 * len(w), (gap >= 2e-2).sum()
    bad = np.flatnonzero(err >= np.where(gap >= 2e-2, 1e-8, 1e-4))
    assert not len(bad), (len(bad), [(int(i), err[i], gap[i]) for i in bad[:8]])


# ------------------------------------------------------------------ point counts
LINEAR_END = {(5, 9), (5, 22)}          # (point count, image) whose LM ends linearly: bar 5e-8


@pytest.mark.parametrize("pn_", sorted(pc.POINT_COUNTS))
def test_point_count_matches_oracle_and_is_stationary(pn_):
    """1e-8 against the oracle minimiser; independently of it, the fp64 gradient of the cost at the device pose is
    orthogonal to the residual: |(J^T r)_j| <= 1e-6 |J_j| |r| for each of the six parameters; status 0.  Image 22 of
    the 5-point batch starts from a P3P pose whose first step overshoots in depth and needs ~240 iterations.  Images
    where Gauss-Newton ends linearly (a last step below 1e-9 that leaves more than 1e-9) are held to the stopping
    rule's limit, 5e-8, as in the filtered-keypoint tests: image 9 of the 5-point batch stops 1.04e-8 from the
    oracle after 6 iterations."""
    c = pc.noisy_problems(f"count/{pn_}", pn_, 32, pc.POINT_COUNTS[pn_])
    poses, info = _solve(c["kp"], c["P"], c["K"], cov=c["cov"])
    P64 = c["P"].astype(np.float64)
    bad, worst_cos = [], 0.0
    for i in range(len(poses)):
        w = pn.covariance_to_weights(c["cov"][i])
        ref = pn.uncertainty_pnp(c["kp"][i], w, P64, c["K"])
        d = np.abs(poses[i] - ref)
        err = max(d[:, :3].max(), d[:, 3].max() / c["unit"])
        if not err < (5e-8 if (pn_, i) in LINEAR_END else 1e-8):
            bad.append((i, err, int(info[i, 1])))
        worst_cos = max(worst_cos, _cosines(poses[i], c["kp"][i], w, c["P"], c["K"]).max())
    assert (info[:, 0] == 0).all(), info[info[:, 0] != 0]
    assert not bad, bad
    assert worst_cos < 1e-6, worst_cos


# ------------------------------------------------------------------ launch shape
@pytest.fixture(scope="module")
def launch_case():
    c = pc.noisy_problems("launch", 9, 1000, "cat")
    ref = [_solve(c["kp"][s], c["P"], c["K"], cov=c["cov"][s]) for s in (slice(0, 500), slice(500, 1000))]
    return c, np.concatenate([r[0] for r in ref]), np.concatenate([r[1] for r in ref])


@pytest.mark.parametrize("b", [1, 592, 593, 594, 595, 596, 1000])
def test_launch_shape_does_not_change_the_answer(launch_case, b):
    """One warp per CTA up to b = 592, four above, with every partial last CTA: each image's pose and info equal,
    bit for bit, the same problem solved in a one-warp-per-CTA batch of 500."""
    c, ref_pose, ref_info = launch_case
    poses, info = _solve(c["kp"][:b], c["P"], c["K"], cov=c["cov"][:b])
    assert np.array_equal(poses, ref_pose[:b]), np.flatnonzero((poses != ref_pose[:b]).any(axis=(1, 2)))
    assert np.array_equal(info, ref_info[:b])


# ------------------------------------------------------------------ filtered keypoints
@pytest.mark.parametrize("entry", ["cov", "weights_2d"])
@pytest.mark.parametrize("kind", sorted(pc.FILTERED_COVS))
def test_filtered_keypoints_match_oracle(kind, entry):
    """1 to pn - 4 points per image get a covariance the reference skips (weight 0); their coordinates stay finite.
    The cov entry computes the weights in fp64 on the device, the weights_2d entry reads them rounded to float32: the
    oracle gets the same weights in each case."""
    n, pn_ = 48, 9
    c = pc.noisy_problems("filtered/" + kind, pn_, n, "cat")
    rng = np.random.default_rng(7)
    cov = c["cov"].copy()
    for i in range(n):
        cov[i, rng.choice(pn_, 1 + i % (pn_ - 4), replace=False)] = pc.FILTERED_COVS[kind]
    w32 = _weights32(cov)
    poses, info = _solve(c["kp"], c["P"], c["K"], **({"cov": cov} if entry == "cov" else {"w": w32}))
    worst = 0.0
    for i in range(n):
        w = pn.covariance_to_weights(cov[i]) if entry == "cov" else w32[i]
        assert (w[:, 0] == 0).sum() == 1 + i % (pn_ - 4)
        ref = pn.uncertainty_pnp(c["kp"][i], w, c["P"].astype(np.float64), c["K"])
        worst = max(worst, np.abs(poses[i] - ref).max())
    assert (info[:, 0] == 0).all(), info[info[:, 0] != 0]
    # 5e-8, the limit of the solver's stopping rule: it stops after a step below 1e-9, and on these large-residual
    # problems (up to 5 of 9 points filtered, the rest noisy) Gauss-Newton converges only linearly, so that last step
    # can leave a few 1e-8 (observed 1.9e-8)
    assert worst < 5e-8, worst


@pytest.mark.parametrize("entry", ["cov", "weights_2d"])
def test_filtered_point_outranks_a_negative_key(entry):
    """pn = 6: two valid points with wxx + wxy < 0 sort below a filtered point (key 0), so the filtered point is one of
    the four P3P points -- exactly as the reference's argsort puts it there."""
    n, pn_ = 48, 6
    c = pc.noisy_problems("filtered/negative_key", pn_, n, "cloud")
    rng = np.random.default_rng(11)
    cov = c["cov"].copy()
    filtered = []
    for i in range(n):
        j = rng.permutation(pn_)
        cov[i, j[0]] = pc.FILTERED_COVS["tiny"]
        for k in j[1:3]:
            cov[i, k] = pc.cov_from_weight(pc.W_NEGATIVE_KEY * rng.uniform(0.5, 2.0))
        filtered.append(j[0])
    w32 = _weights32(cov)
    poses, info = _solve(c["kp"], c["P"], c["K"], **({"cov": cov} if entry == "cov" else {"w": w32}))
    worst = 0.0
    for i in range(n):
        w = pn.covariance_to_weights(cov[i]) if entry == "cov" else w32[i]
        assert filtered[i] in np.argsort(w[:, 0] + w[:, 1], kind="stable")[-4:]
        ref = pn.uncertainty_pnp(c["kp"][i], w, c["P"].astype(np.float64), c["K"])
        worst = max(worst, np.abs(poses[i] - ref).max())
    assert (info[:, 0] == 0).all(), info[info[:, 0] != 0]
    assert worst < 1e-8, worst


# ------------------------------------------------------------------ invariances
@pytest.mark.parametrize("scale", [2.0 ** -7, 2.0 ** 7])
def test_weight_scale_leaves_the_pose_bitwise_unchanged(scale):
    """Scaling every weight by a power of two scales the residuals, the Jacobian, the normal equations, the damping and
    the Cholesky factors exactly, and leaves every LM step and acceptance ratio bit for bit the same: a pose that
    changes means a threshold on an absolute quantity fired."""
    c = pc.noisy_problems("invariance/weights", 9, 64, "cat")
    w = _weights32(c["cov"])
    base, base_info = _solve(c["kp"], c["P"], c["K"], w=w)
    poses, info = _solve(c["kp"], c["P"], c["K"], w=w * np.float32(scale))
    assert np.array_equal(poses, base), np.flatnonzero((poses != base).any(axis=(1, 2)))
    assert np.array_equal(info, base_info)


def test_object_scale_scales_the_translation():
    """Object points x 1024 (exact in float32): same quartic, a P3P start scaled exactly; the stopping rule on |step|
    mixes radians and lengths, so R to 1e-8 and t to 1e-8 relative."""
    c = pc.noisy_problems("invariance/points", 9, 64, "cat")
    base, base_info = _solve(c["kp"], c["P"], c["K"], cov=c["cov"])
    poses, info = _solve(c["kp"], c["P"] * np.float32(1024), c["K"], cov=c["cov"])
    assert (base_info[:, 0] == 0).all() and (info[:, 0] == 0).all()
    assert np.abs(poses[:, :, :3] - base[:, :, :3]).max() < 1e-8
    rel = np.linalg.norm(poses[:, :, 3] - 1024 * base[:, :, 3], axis=1) / np.linalg.norm(1024 * base[:, :, 3], axis=1)
    assert rel.max() < 1e-8, rel.max()
