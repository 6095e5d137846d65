"""CPU: the stages of oracle/refine_oracle.py (the contract of `pvnet_refine_poses`, DESIGN.md §26) on hand-built
cases, and its refinement on a known answer.  The device is held to this oracle in tests/test_gpu_refine.py."""
import numpy as np
import pytest
import torch

from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import render_cases as rc


def rowmajor(w, pixels):
    return np.array([r * w + c for r, c in pixels], np.int64)


def test_boundary_of_a_2x2_square_is_all_four_pixels_in_row_major_order():
    m = np.zeros((4, 5), bool)
    m[1:3, 2:4] = True
    assert np.array_equal(rfo.boundary(m), rowmajor(5, [(1, 2), (1, 3), (2, 2), (2, 3)]))


def test_boundary_around_a_one_pixel_hole():
    m = np.zeros((7, 7), bool)
    m[1:6, 1:6] = True
    m[3, 3] = False
    ring = [(r, c) for r in range(1, 6) for c in range(1, 6) if r in (1, 5) or c in (1, 5)]
    hole = [(2, 3), (3, 2), (3, 4), (4, 3)]
    expect = rowmajor(7, sorted(ring + hole))
    assert np.array_equal(rfo.boundary(m), expect)
    assert 3 * 7 + 3 not in rfo.boundary(m) and 2 * 7 + 2 not in rfo.boundary(m)   # the hole; a diagonal neighbour


def test_boundary_at_the_image_edge_and_of_nothing():
    assert np.array_equal(rfo.boundary(np.ones((3, 4), bool)), rowmajor(4, [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0),
                                                                           (1, 3), (2, 0), (2, 1), (2, 2), (2, 3)]))
    assert np.array_equal(rfo.boundary(np.ones((1, 1), bool)), [0])
    assert len(rfo.boundary(np.zeros((5, 5), bool))) == 0


def test_subsample_keeps_every_ceil_n_over_max_th_point():
    idx = np.arange(100, 110)
    assert np.array_equal(rfo.subsample(idx, 4), [100, 103, 106, 109])
    assert np.array_equal(rfo.subsample(idx, 5), [100, 102, 104, 106, 108])
    assert np.array_equal(rfo.subsample(idx, 10), idx)
    assert np.array_equal(rfo.subsample(idx, 1), [100])


def test_back_projection_inverts_the_renderers_projection():
    rng = np.random.default_rng(3)
    h, w = 61, 83
    K = rc.camera_for(h, w, 70.0)
    K[0, 1] = 1.7                                                              # skew, read as the renderer reads it
    K[:2, 2] += (2.3, -1.9)
    idx = rng.choice(h * w, 500, replace=False)
    depth = rng.uniform(0.3, 3.0, h * w).astype(np.float32)
    r, c = np.divmod(idx, w)
    # the camera part alone: identity pose
    eye = np.hstack([np.eye(3), np.zeros((3, 1))])
    u, v = rfo.project(rfo.back_project(idx, depth, eye, K, w), eye, K)
    assert np.abs(u - (c + 0.5)).max() <= 1e-12 and np.abs(v - (r + 0.5)).max() <= 1e-12
    # at a pose: R^T inverts R only to rounding
    P = rf.true_poses(1, rng)[0]
    X = rfo.back_project(idx, depth, P, K, w)
    u, v = rfo.project(X, P, K)
    assert np.abs(u - (c + 0.5)).max() <= 1e-9 and np.abs(v - (r + 0.5)).max() <= 1e-9
    assert np.array_equal(u.astype(np.float32), (c + 0.5).astype(np.float32))
    assert np.array_equal(v.astype(np.float32), (r + 0.5).astype(np.float32))


def test_nearest_pair_ties_go_to_the_lowest_contour_index_and_the_gate_drops():
    w = 20
    K = rc.camera_for(20, 20, 30.0)
    eye = np.hstack([np.eye(3), np.zeros((3, 1))])
    # a point that projects onto pixel (5, 5)'s centre
    X = rfo.back_project(np.array([5 * w + 5]), np.full(w * w, 2.0, np.float32), eye, K, w)
    for con, expect in (([5 * w + 7, 5 * w + 3], 0), ([5 * w + 3, 5 * w + 7], 0), ([9 * w + 9, 5 * w + 3, 3 * w + 5], 1)):
        j, d2 = rfo.nearest_pairs(X, eye, K, np.array(con), w, gate=20.0)
        assert j[0] == expect and d2[0] == 4.0
    j, d2 = rfo.nearest_pairs(X, eye, K, np.array([5 * w + 8]), w, gate=2.99)
    assert j[0] == -1 and d2[0] == 9.0
    j, _ = rfo.nearest_pairs(X, eye, K, np.array([5 * w + 8]), w, gate=3.0)            # d2 <= gate^2 is kept
    assert j[0] == 0
    j, d2 = rfo.nearest_pairs(X, eye, K, np.array([], np.int64), w, gate=20.0)
    assert j[0] == -1 and d2[0] == np.inf


H, W = 120, 160
K_TOOL = rc.camera_for(H, W, 300.0)


def truth_masks(P, K=K_TOOL):
    v, f = rf.tool_mesh()
    return np.stack([ro.render(v, f, K, p.astype(np.float32)[None], H, W, rf.NEAR, rf.FAR)[0][0] > 0 for p in P])


def proj_error(P, Pt, K=K_TOOL):
    """The 2D projection error: mean pixel distance of the mesh's vertices projected at the two poses."""
    v = rf.tool_mesh()[0].astype(np.float64)
    a, b = np.stack(rfo.project(v, P, K), -1), np.stack(rfo.project(v, Pt, K), -1)
    return float(np.linalg.norm(a - b, axis=1).mean())


def test_known_answer_refinement_lowers_the_distance_every_kept_round_and_ends_closer():
    """The mask is the truth's coverage; the start is 3 degrees and 1 cm away.  What a silhouette fixes is the
    outline, so "closer" is measured by the 2D projection error: it falls in every image, from 3.4-6.2 px to
    0.25-3.9 px, and on average below 0.35 of where it started."""
    rng = np.random.default_rng(0)
    Pt = rf.true_poses(8, rng)
    P0 = rf.perturb(Pt, rng)
    masks = truth_masks(Pt)
    v, f = rf.tool_mesh()
    before, after = [], []
    for i in range(len(Pt)):
        tr = []
        P, info = rfo.refine_image(masks[i], P0[i], K_TOOL, v, f, rf.NEAR, rf.FAR, rounds=8, trace=tr)
        means = [t["mean"] for t in tr]
        kept = means if not info["status"] & rfo.REJECTED else means[:-1]
        assert all(b < a for a, b in zip(kept, kept[1:])), means
        assert info["dist_before"] == means[0] and info["dist_after"] == kept[-1] < means[0]
        assert info["status"] & ~rfo.REJECTED == 0
        if info["status"] & rfo.REJECTED:
            assert np.array_equal(P, tr[-2]["pose"]) or len(tr) == 1
        before.append(proj_error(P0[i], Pt[i]))
        after.append(proj_error(P, Pt[i]))
        assert after[-1] < before[-1], (i, before[-1], after[-1])
    assert np.mean(after) < 0.35 * np.mean(before), (before, after)


def test_status_bits_and_the_input_returned():
    rng = np.random.default_rng(5)
    Pt = rf.true_poses(1, rng)
    v, f = rf.tool_mesh()
    m = truth_masks(Pt)[0]
    empty = np.zeros_like(m)
    P, info = rfo.refine_image(empty, Pt[0], K_TOOL, v, f, rf.NEAR, rf.FAR)
    assert info["status"] == rfo.NO_CONTOUR and np.array_equal(P, Pt[0]) and np.isnan(info["dist_before"])
    behind = Pt[0].copy()
    behind[2, 3] = -1.0
    P, info = rfo.refine_image(m, behind, K_TOOL, v, f, rf.NEAR, rf.FAR)
    assert info["status"] == rfo.NO_SILHOUETTE and np.array_equal(P, behind)
    far_mask = np.zeros_like(m)
    far_mask[:10, :10] = True                                                  # a blob far from the render
    P, info = rfo.refine_image(far_mask, Pt[0], K_TOOL, v, f, rf.NEAR, rf.FAR, gate=5.0)
    assert info["status"] == rfo.FEW_PAIRS and np.array_equal(P, Pt[0])
    P, info = rfo.refine_image(m, Pt[0], K_TOOL, v, f, rf.NEAR, rf.FAR, rounds=0)
    assert info["status"] == 0 and np.array_equal(P, Pt[0]) and info["dist_before"] == info["dist_after"]


def test_refine_poses_has_no_cpu_path():
    from pvnet_b200.refine import refine_poses
    v, f = rf.tool_mesh()
    with pytest.raises(RuntimeError, match="CUDA"):
        refine_poses(torch.zeros(1, 8, 8, dtype=torch.uint8), torch.zeros(1, 3, 4), torch.eye(3), torch.from_numpy(v),
                     torch.from_numpy(f), rf.NEAR, rf.FAR)
