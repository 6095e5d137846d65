"""CPU: the keypoint-anchored objective of oracle/refine_keypoints_oracle.py (the contract of `pvnet_refine_poses_keypoints`,
DESIGN.md §27): its Jacobian, its limit at a large keypoint weight (the uncertainty-PnP pose), the rotation the
silhouette cannot see, the accept rule, and a known answer.  The device is held to this oracle in
tests/test_gpu_refine_keypoints.py."""
import numpy as np
import pytest
import torch

from oracle import pnp_oracle as pno
from oracle import refine_keypoints_oracle as rko
from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import refine_keypoint_cases as rkc
from tests import render_cases as rc

H, W = 120, 160
K_TOOL = rc.camera_for(H, W, 300.0)
MESH = rf.tool_mesh()
PTS = rkc.tool_keypoints()


def scene(b, seed, sigma=1.0):
    """§26's three-box scene: true poses, starts 3 degrees and 1 cm away, the truth's masks, and keypoints at the
    true projections plus `sigma` px of noise with their float32 weights."""
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    masks = np.stack([ro.render(*MESH, K_TOOL, p.astype(np.float32)[None], H, W, rf.NEAR, rf.FAR)[0][0] > 0
                      for p in Pt])
    kp, cov = rkc.keypoint_votes(Pt, K_TOOL, PTS, sigma, np.random.default_rng(seed + 100))
    return Pt, P0, masks, kp, rkc.isotropic_weights(cov)


def test_warp_sum_is_the_xor_butterfly():
    x = np.random.default_rng(0).normal(size=23) * 10.0 ** np.arange(23)
    lanes = np.zeros(32)
    lanes[:23] = x
    for o in (16, 8, 4, 2, 1):
        lanes = np.array([lanes[i] + lanes[i ^ o] for i in range(32)])
    assert rko.warp_sum(x) == lanes[0]
    assert rko.warp_sum([1.5] * 32) == 48.0


def test_keypoint_jacobian_matches_central_differences():
    rng = np.random.default_rng(1)
    K = rc.camera_for(H, W, 300.0)
    K[0, 1] = 0.8                                                            # skew: read as the renderer reads it
    pose = rf.true_poses(1, rng)[0]
    kp = rng.uniform(0, W, (8, 2)).astype(np.float32)
    wts = rng.uniform(0.2, 2.0, (8, 3)).astype(np.float32)
    wts[:, 1] *= 0.3
    term = rko.Keypoints(kp, PTS, wts, 1.0)
    J = term.jacobian(pose, K)
    h = 1e-6
    for j in range(6):
        d = np.zeros(6)
        d[j] = h
        Pp, Pm = pose.copy(), pose.copy()
        Pp[:, :3] = rfo.so3_exp(d[:3]) @ pose[:, :3]
        Pm[:, :3] = rfo.so3_exp(-d[:3]) @ pose[:, :3]
        Pp[:, 3] += d[3:]
        Pm[:, 3] -= d[3:]
        fd = (term.residuals(Pp, K) - term.residuals(Pm, K)) / (2 * h)
        # central differences are exact to O(h^2) ~ 1e-12 of the curvature, plus 1e-16 / h of rounding
        assert np.abs(fd - J[:, :, j]).max() <= 1e-6 * max(1.0, np.abs(J[:, :, j]).max()), j


def test_a_non_finite_keypoint_is_left_out():
    kp = np.zeros((5, 2), np.float32)
    kp[2, 0] = np.nan
    w = np.ones((5, 3), np.float32)
    w[4, 1] = np.inf
    term = rko.Keypoints(kp, PTS[:5], w, 1.0)
    assert term.on.tolist() == [True, True, False, True, False]
    pose = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    assert np.isfinite(term.distance_sum(pose, K_TOOL)) and term.jacobian(pose, K_TOOL).shape == (3, 2, 6)


def test_a_large_keypoint_weight_gives_the_uncertainty_pnp_pose():
    """lambda = 1e6 makes the pair term about 1e-7 of the keypoint term, so the steps go to the minimiser of the
    weighted reprojection error: `pnp_oracle.uncertainty_pnp` with the same float32 weights and the fp32-rounded K.
    Three damped steps per round reach it to ~1e-8 in the pose's entries by the second or third round; the round
    after that can be undone, because C sums the weighted distances, not their squares, and its minimiser lies
    ~1e-6 away.  Hence: every returned entry within 1e-5, and the closest evaluated pose within 1e-7."""
    Pt, P0, masks, kp, wts = scene(3, 0)
    K64 = K_TOOL.astype(np.float32).astype(np.float64)
    for i in range(3):
        ref = pno.uncertainty_pnp(kp[i].astype(np.float64), wts[i].astype(np.float64), PTS.astype(np.float64), K64)
        tr = []
        P, info = rko.refine_image(masks[i], P0[i], K_TOOL, *MESH, rf.NEAR, rf.FAR, keypoints=kp[i], points_3d=PTS,
                                   weights=wts[i], keypoint_weight=1e6, trace=tr)
        assert info["status"] & ~rfo.REJECTED == 0
        assert np.abs(P - ref).max() <= 1e-5, (i, np.abs(P - ref).max())
        assert min(np.abs(t["pose"] - ref).max() for t in tr) <= 1e-7, i
        assert np.abs(P0[i] - ref).max() > 1e-2                              # it did move there


def test_keypoints_hold_the_rotation_the_silhouette_cannot_see():
    """`singular_scene`: no contour pair constrains the rotation about the optical axis, so the silhouette alone
    stops with SINGULAR at the input.  The true projections of five points off that axis (cov = 0.25 I) make the
    system regular, and a start turned 3 degrees about the axis comes back."""
    (v, f), K, pose, mask = rf.singular_scene()
    pts = rkc.singular_scene_keypoints()
    u, vv = rfo.project(pts.astype(np.float64), pose, K)
    kp = np.stack([u, vv], -1).astype(np.float32)
    wts = rkc.isotropic_weights(np.broadcast_to(0.25 * np.eye(2), (5, 2, 2)))
    P0 = pose.copy()
    P0[:, :3] = rf.axis_angle([0.0, 0.0, np.deg2rad(3.0)]) @ P0[:, :3]
    P, info = rfo.refine_image(mask, P0, K, v, f, 0.05, 5.0)
    assert info["status"] == rfo.SINGULAR and np.array_equal(P, P0)
    P, info = rko.refine_image(mask, P0, K, v, f, 0.05, 5.0, keypoints=kp, points_3d=pts, weights=wts)
    assert info["status"] & rfo.SINGULAR == 0
    assert rf.pose_error(P, pose)[0] < 1e-3 < 2.9 < rf.pose_error(P0, pose)[0]
    assert info["cost_after"] < info["cost_before"]


@pytest.fixture(scope="module")
def known_answer():
    """The 8-image 120x160 batch of §26's known-answer test, keypoints with 1 px noise, silhouette-only and
    keypoint-anchored at lambda = 0.25 (the default, DESIGN.md §27) and 1."""
    Pt, P0, masks, kp, wts = scene(8, 0)
    runs = {None: [], 0.25: [], 1.0: []}
    for lam in runs:
        for i in range(8):
            kw = {} if lam is None else dict(keypoints=kp[i], points_3d=PTS, weights=wts[i], keypoint_weight=lam)
            tr = []
            P, info = (rfo if lam is None else rko).refine_image(masks[i], P0[i], K_TOOL, *MESH, rf.NEAR, rf.FAR,
                                                                   trace=tr, **kw)
            runs[lam].append((P, info, tr))
    return Pt, P0, runs


def test_cost_never_rises(known_answer):
    """The returned C is at most the input C in every image, and each kept round lowered C."""
    _, _, runs = known_answer
    for lam in (0.25, 1.0):
        for P, info, tr in runs[lam]:
            assert info["cost_after"] <= info["cost_before"], lam
            costs = [t["cost"] for t in tr]
            kept = costs if not info["status"] & rfo.REJECTED else costs[:-1]
            assert all(b <= a for a, b in zip(kept, kept[1:])), costs
            assert info["cost_after"] == kept[-1] and info["cost_before"] == costs[0]
            if info["status"] & rfo.REJECTED:
                assert costs[-1] > costs[-2] and np.array_equal(P, tr[-2]["pose"])


def test_known_answer_keypoints_lower_the_rotation_error(known_answer):
    """Starts 3 degrees off; seeded 1 px keypoint noise.  Pinned from this seed: silhouette-only ends at a mean
    rotation error of 3.18 degrees (no better than the start: the outline holds the in-plane rotation, not the
    others), anchored at lambda = 0.25 at 1.07 and at lambda = 1 at 1.32.  The anchored result is not better in
    every image (image 3: 1.13 against 0.54 at lambda = 0.25), so the mean is asserted."""
    Pt, P0, runs = known_answer
    err = {lam: np.array([rf.pose_error(r[0], Pt[i])[0] for i, r in enumerate(runs[lam])]) for lam in runs}
    start = np.array([rf.pose_error(P0[i], Pt[i])[0] for i in range(8)])
    assert np.allclose(start, 3.0)
    assert err[None].mean() == pytest.approx(3.18, abs=0.01)
    assert err[0.25].mean() == pytest.approx(1.07, abs=0.01)
    assert err[1.0].mean() == pytest.approx(1.32, abs=0.01)
    assert err[0.25].mean() < 0.4 * err[None].mean() and err[1.0].mean() < 0.5 * err[None].mean()
    assert (err[0.25] < err[None]).sum() == 7


def test_refine_poses_with_keypoints_has_no_cpu_path():
    from pvnet_b200.refine import refine_poses
    v, f = MESH
    with pytest.raises(RuntimeError, match="CUDA"):
        refine_poses(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 3, 4), torch.eye(3), torch.from_numpy(v),
                     torch.from_numpy(f), rf.NEAR, rf.FAR, keypoints=torch.zeros(1, 8, 2),
                     points_3d=torch.from_numpy(PTS), cov=torch.eye(2).expand(1, 8, 2, 2))
