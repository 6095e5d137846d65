"""CPU: the depth-anchored objective of oracle/refine_depth_oracle.py (the contract of `pvnet_refine_poses_depth`,
DESIGN.md §28): its Jacobian, the observed normals, the pair predicate at image and mask borders, the distance along
the optical axis that the silhouette cannot hold, known answers from §26's starts, and the accept rule.  The device
is held to this oracle in tests/test_gpu_refine_depth.py."""
import numpy as np
import pytest
import torch

from oracle import refine_depth_oracle as rdo
from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import render_cases as rc

H, W = 120, 160
K_TOOL = rc.camera_for(H, W, 300.0)
MESH = rf.tool_mesh()


def render(P, mesh=MESH, h=H, w=W):
    return ro.render(*mesh, K_TOOL, np.asarray(P, np.float32)[None], h, w, rf.NEAR, rf.FAR)[0][0]


def plane(half=1.0):
    """A square of side 2 half in the z = 0 plane, two triangles."""
    v = np.array([[-half, -half, 0], [half, -half, 0], [half, half, 0], [-half, half, 0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def test_jacobian_matches_central_differences():
    rng = np.random.default_rng(1)
    pose = rf.true_poses(1, rng)[0]
    X = rng.uniform(-0.06, 0.06, (20, 3))
    Y = X @ pose[:, :3].T + pose[:, 3] + rng.normal(0, 0.003, (20, 3))
    n = rng.normal(size=(20, 3))
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    J = rdo.jacobian(X, n, pose)
    h = 1e-6
    for j in range(6):
        d = np.zeros(6)
        d[j] = h
        Pp, Pm = pose.copy(), pose.copy()
        Pp[:, :3] = rfo.so3_exp(d[:3]) @ pose[:, :3]
        Pm[:, :3] = rfo.so3_exp(-d[:3]) @ pose[:, :3]
        Pp[:, 3] += d[3:]
        Pm[:, 3] -= d[3:]
        fd = (rdo.residuals(X, Y, n, Pp)[0] - rdo.residuals(X, Y, n, Pm)[0]) / (2 * h)
        # O(h^2) curvature plus 1e-16 / h of rounding
        assert np.abs(fd - J[:, j]).max() <= 1e-8, j
    A, g = rdo.normal_equations(X, Y, n, pose)
    e = rdo.residuals(X, Y, n, pose)[0]
    assert np.allclose(A, J.T @ J) and np.allclose(g, J.T @ e)


def test_the_normal_of_a_plane_rendered_at_a_known_pose():
    """A tilted 2 m square 0.6 m away fills the image: every pair's observed normal is the plane's normal turned
    towards the camera.  The fp32 depths bend it by at most 0.0012 degrees (measured: 0.0012 max, 0.00035 median)."""
    v, f = plane()
    P = np.hstack([rf.axis_angle([0.3, -0.4, 0.2]), [[0.01], [-0.02], [0.6]]])
    d = render(P, (v, f))
    assert (d > 0).all()
    pr = rdo.pairs(d, d > 0, d, P, K_TOOL, 1.0, 10 ** 6)
    assert len(pr["idx"]) == (H - 2) * (W - 2)                            # every pixel but the image's border
    nt = P[:, 2] * (-1.0 if P[:, 2] @ P[:, 3] > 0 else 1.0)
    ang = np.degrees(np.arccos(np.clip(pr["n"] @ nt, -1, 1)))
    assert ang.max() < 0.002
    assert ((pr["n"] * pr["Y"]).sum(1) < 0).all()
    assert np.abs(rdo.residuals(pr["X"], pr["Y"], pr["n"], P)[0]).max() < 1e-6


def test_the_pair_predicate_at_image_and_mask_borders():
    """A flat depth over a 12x14 image: a pair needs its pixel and its four 4-neighbours inside the image, in the mask
    and read, and the render's coverage at the pixel itself."""
    h, w = 12, 14
    K = rc.camera_for(h, w, 20.0)
    P = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    zo = np.full((h, w), 0.5, np.float32)
    mask = np.ones((h, w), np.uint8)
    mask[5, 6] = 0                                                          # a mask hole
    mask[:, 12:] = 0                                                        # a mask edge
    zo[2, 3] = 0                                                            # no reading
    zo[8, 2] = np.nan                                                       # not a number: no reading
    zo[9, 9] = -1.0                                                         # negative: no reading
    rd = np.full((h, w), 0.5, np.float32)
    rd[10, 5] = 0                                                           # not covered by the render
    pr = rdo.pairs(rd, mask, rdo.observed_depth(zo), P, K, 1.0, 10 ** 6)
    want = np.zeros((h, w), bool)
    read = (mask != 0) & (np.nan_to_num(zo) > 0)
    for r in range(1, h - 1):
        for c in range(1, w - 1):
            want[r, c] = (read[r, c] and read[r, c - 1] and read[r, c + 1] and read[r - 1, c] and read[r + 1, c]
                          and rd[r, c] > 0)
    assert np.array_equal(pr["idx"], np.flatnonzero(want))
    for r, c in ((5, 6), (5, 5), (5, 7), (4, 6), (6, 6), (2, 3), (2, 4), (3, 3), (8, 3), (9, 9), (10, 5), (6, 11),
                 (0, 4), (4, 0)):
        assert not want[r, c], (r, c)
    assert pr["count"] == want.sum() and pr["mask_pixels"] == mask.sum() and pr["covered_pixels"] == h * w - 1
    # a flat plane at z = 0.5 facing the camera: n = (0, 0, -1), R X + t = Y at this pose, residual 0
    assert np.allclose(pr["n"], [0, 0, -1], atol=1e-12)
    assert np.abs(pr["X"] + P[:, 3] - pr["Y"]).max() < 1e-12
    assert np.abs(rdo.residuals(pr["X"], pr["Y"], pr["n"], P)[0]).max() < 1e-12
    # the stride: every ceil(n / max_points)-th pair from the first
    sub = rdo.pairs(rd, mask, rdo.observed_depth(zo), P, K, 1.0, 7)
    assert np.array_equal(sub["idx"], pr["idx"][::-(-len(pr["idx"]) // 7)])
    # the gate is in the poses' units: 1 cm off along z drops every pair at gate 0.009, keeps them at 0.011
    Q = P.copy()
    Q[2, 3] = 0.51
    rd2 = np.where(rd > 0, np.float32(0.51), np.float32(0))
    assert len(rdo.pairs(rd2, mask, zo.clip(0), Q, K, 0.009, 10 ** 6)["idx"]) == 0
    assert len(rdo.pairs(rd2, mask, zo.clip(0), Q, K, 0.011, 10 ** 6)["idx"]) == want.sum()


def test_observed_depth_reads_uint16_with_one_rounded_multiply():
    d = np.array([[0, 1, 523, 65535]], np.uint16)
    z = rdo.observed_depth(d, 1e-3)
    assert z.dtype == np.float32
    assert np.array_equal(z, d.astype(np.float32) * np.float32(1e-3))
    assert z[0, 0] == 0


def test_an_optical_axis_start_is_held_by_depth_not_by_the_silhouette():
    """Starts 2 cm behind the truth along the optical axis (t_z only), the truth's coverage as the mask and its
    render as the depth.  Measured on these six images: silhouette-only refinement ends 3.02 mm from the true
    translation on average (0.64-11.6 mm), depth refinement 0.0003 mm (at most 0.0014 mm)."""
    rng = np.random.default_rng(21)
    Pt = rf.true_poses(6, rng)
    P0 = rdc.along_axis(Pt, 0.02)
    es, ed = [], []
    for i in range(6):
        d = render(Pt[i])
        Ps, _ = rfo.refine_image(d > 0, P0[i], K_TOOL, *MESH, rf.NEAR, rf.FAR)
        Pd, info = rdo.refine_image(d > 0, d, P0[i], K_TOOL, *MESH, rf.NEAR, rf.FAR, rdc.GATE)
        assert info["status"] & ~rfo.REJECTED == 0
        es.append(rf.pose_error(Ps, Pt[i])[1])
        ed.append(rf.pose_error(Pd, Pt[i])[1])
    es, ed = np.array(es), np.array(ed)
    assert es.mean() == pytest.approx(3.02e-3, abs=1e-5)
    assert ed.max() < 2e-6 and ed.mean() < 1e-6
    assert (ed < es).all()


@pytest.fixture(scope="module")
def known_answer():
    """§26's known-answer batch: 8 images at 120x160, starts 3 degrees and 1 cm away, the truth's coverage as the
    mask; observed depth the truth's render, clean and with seeded 1 mm noise."""
    rng = np.random.default_rng(0)
    Pt = rf.true_poses(8, rng)
    P0 = rf.perturb(Pt, rng)
    dep = np.stack([render(p) for p in Pt])
    runs = {}
    for name, obs in (("clean", dep), ("noisy", rdc.noisy(dep, 1e-3, np.random.default_rng(5)))):
        runs[name] = []
        for i in range(8):
            tr = []
            P, info = rdo.refine_image(dep[i] > 0, obs[i], P0[i], K_TOOL, *MESH, rf.NEAR, rf.FAR, rdc.GATE, trace=tr)
            runs[name].append((P, info, tr))
    return Pt, P0, runs


def test_known_answer_convergence(known_answer):
    """Pinned from these seeds (8 rounds): clean depth ends at mean errors of 0.071 degrees and 0.85 mm, 1 mm noise
    at 0.72 degrees and 1.82 mm, from 3 degrees and 10 mm.  Every image's translation error falls; with noise one
    image's rotation error rises (image 7, from 3 to 5.3 degrees, while its translation error
    falls), so the rotation is asserted per image only without noise."""
    Pt, P0, runs = known_answer
    start = np.array([rf.pose_error(P0[i], Pt[i]) for i in range(8)])
    assert np.allclose(start[:, 0], 3.0) and np.allclose(start[:, 1], 0.01)
    err = {k: np.array([rf.pose_error(r[0], Pt[i]) for i, r in enumerate(v)]) for k, v in runs.items()}
    assert err["clean"][:, 0].mean() == pytest.approx(0.0707, abs=0.001)
    assert err["clean"][:, 1].mean() == pytest.approx(0.847e-3, abs=0.01e-3)
    assert err["noisy"][:, 0].mean() == pytest.approx(0.725, abs=0.005)
    assert err["noisy"][:, 1].mean() == pytest.approx(1.816e-3, abs=0.01e-3)
    assert (err["clean"][:, 0] < start[:, 0]).all()
    assert (err["noisy"][:, 0] < start[:, 0]).sum() == 7 and err["noisy"][7, 0] == pytest.approx(5.27, abs=0.01)
    for k in runs:
        assert (err[k][:, 1] < start[:, 1]).all(), k
        assert all(r[1]["status"] & ~rfo.REJECTED == 0 for r in runs[k])


def test_the_mean_never_rises(known_answer):
    """The returned mean |e| is at most the input's in every image, and each kept round lowered it; an undone round
    returns the pose it started from."""
    _, _, runs = known_answer
    for k, rs in runs.items():
        for P, info, tr in rs:
            assert info["dist_after"] <= info["dist_before"], k
            means = [t["mean"] for t in tr]
            kept = means if not info["status"] & rfo.REJECTED else means[:-1]
            assert all(b <= a for a, b in zip(kept, kept[1:])), means
            assert info["dist_after"] == kept[-1] and info["dist_before"] == means[0]
            if info["status"] & rfo.REJECTED:
                assert means[-1] > means[-2] and np.array_equal(P, tr[-2]["pose"])


def test_degenerate_images_return_their_input():
    rng = np.random.default_rng(3)
    Pt = rf.true_poses(1, rng)[0]
    d = render(Pt)
    for mask, depth, pose, status in ((np.zeros_like(d), d, Pt, rfo.NO_CONTOUR),
                                      (d > 0, d, rdc.along_axis(Pt[None], -2.0)[0], rfo.NO_SILHOUETTE),
                                      (d > 0, np.zeros_like(d), Pt, rfo.FEW_PAIRS)):
        P, info = rdo.refine_image(mask, depth, pose, K_TOOL, *MESH, rf.NEAR, rf.FAR, rdc.GATE)
        assert info["status"] == status and np.array_equal(P, pose)
    P, info = rdo.refine_image(d > 0, d, Pt, K_TOOL, *MESH, rf.NEAR, rf.FAR, rdc.GATE, rounds=0)
    assert info["status"] == 0 and np.array_equal(P, Pt)


def test_refine_poses_depth_has_no_cpu_path():
    from pvnet_b200.refine import refine_poses_depth
    v, f = MESH
    with pytest.raises(RuntimeError, match="CUDA"):
        refine_poses_depth(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 8, 8), torch.zeros(1, 3, 4),
                           torch.eye(3), torch.from_numpy(v), torch.from_numpy(f), rf.NEAR, rf.FAR, gate=0.03)
