"""CPU: the edges of oracle/refine_oracle.py that `pvnet_refine_poses` (csrc/refine.cu, DESIGN.md §26) is held to at
full size in tests/test_gpu_refine_edges.py -- the mask builders that give exact contour counts, a nearest-pair tie
that straddles the kernel's 2 048-point contour tiles, the mean distance summed in the kernel's order, and the
SINGULAR status."""
import numpy as np
import pytest

from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import render_cases as rc

H, W = 240, 320
K = rc.camera_for(H, W, 500.0)


@pytest.fixture(scope="module")
def scene():
    """The tool at a true pose in the lower half of the image and a start 3 degrees and 1 cm away: true pose, start,
    the truth's coverage and the depth at the start."""
    rng = np.random.default_rng(7)
    Pt = rf.true_poses(1, rng)
    Pt[:, 1, 3] += 0.06                                                         # room above it for padding
    P0 = rf.perturb(Pt, rng)
    v, f = rf.tool_mesh()
    on = ro.render(v, f, K, Pt.astype(np.float32), H, W, rf.NEAR, rf.FAR)[0][0] > 0
    depth0 = ro.render(v, f, K, P0.astype(np.float32), H, W, rf.NEAR, rf.FAR)[0][0]
    return Pt[0], P0[0], on, depth0


@pytest.mark.parametrize("n", [2047, 2048, 2049, 4096, 4097, 6145])
@pytest.mark.parametrize("holes", [0, 40])
def test_mask_builder_reaches_exact_contour_counts(scene, n, holes):
    _, _, on, _ = scene
    m = rf.with_contour_count(on, n, holes=holes, seed=n)
    con = rfo.boundary(m)
    assert len(con) == n
    assert (on & ~m).sum() == holes and (m & ~on).sum() == n - len(rfo.boundary(on)) - 4 * holes
    assert set(rfo.boundary(on)) <= set(con)                                    # the object's own contour is kept
    # the stride rule at the caps the GPU tests use
    for mp in (4096, 10000):
        stride = max(1, -(-n // mp))
        assert len(rfo.subsample(con, mp)) == -(-n // stride) <= mp


def test_isolated_pixels_and_holes_each_count_as_expected():
    on = np.zeros((20, 20), bool)
    on[4:16, 4:16] = True
    base = len(rfo.boundary(on))
    hs = rf.hole_sites(on)
    assert len(hs) and all(4 <= r < 16 and 4 <= c < 16 for r, c in zip(*np.divmod(hs, 20)))
    m = on.copy().reshape(-1)
    m[hs[0]] = False
    assert len(rfo.boundary(m.reshape(20, 20))) == base + 4
    ss = rf.speckle_sites(on)
    m = on.copy().reshape(-1)
    m[ss] = True
    assert len(rfo.boundary(m.reshape(20, 20))) == base + len(ss)
    with pytest.raises(AssertionError):
        rf.with_contour_count(on, base - 1)
    # a mask that fills the image: no hole site within two pixels of the border, where a neighbour is already contour
    full = np.ones((12, 13), bool)
    hs = rf.hole_sites(full)
    r, c = np.divmod(hs, 13)
    assert len(hs) and r.min() >= 2 and c.min() >= 2 and r.max() <= 9 and c.max() <= 10
    n = len(rfo.boundary(full)) + 4 * len(hs)
    assert len(rfo.boundary(rf.with_contour_count(full, n, holes=len(hs)))) == n


def test_a_tie_across_the_first_tile_boundary_goes_to_the_lower_index(scene):
    """The silhouette point's two nearest contour pixels are index 2047 (the last of the kernel's first 2 048-point
    tile) and one in a later tile, at the same fp32 d2; the pair is the lower index."""
    _, P0, on, depth0 = scene
    m, i, lo, hi = rf.straddling_tie(on, depth0, P0, K)
    assert lo == 2047 and hi >= 2048
    sil = rfo.boundary(depth0 > 0)
    con = rfo.boundary(m)
    d = rf.round0_d2(sil, depth0, P0, K, con, W)
    assert d[i, lo] == d[i, hi] == d[i].min()
    X = rfo.back_project(sil, depth0, P0, K, W)
    j, d2 = rfo.nearest_pairs(X, P0, K, con, W, 20.0)
    assert j[i] == lo and d2[i] == d[i, lo]
    # the padding is nobody's pair: every other pair is the unpadded mask's, shifted by the padding
    j0, d20 = rfo.nearest_pairs(X, P0, K, rfo.boundary(on), W, 20.0)
    assert np.array_equal(j >= 0, j0 >= 0) and np.array_equal(d2[j >= 0], d20[j0 >= 0])
    assert np.array_equal(j[j >= 0], j0[j0 >= 0] + lo - j0[i])


def literal_block_sum(x):
    """k_refine_step's reduction written out thread by thread and lane by lane."""
    part = [0.0] * 256
    for t in range(256):
        for i in range(t, len(x), 256):
            part[t] = part[t] + float(x[i])
    warps = []
    for wp in range(8):
        v = part[32 * wp:32 * wp + 32]
        for o in (16, 8, 4, 2, 1):
            v = [v[lane] + v[lane ^ o] for lane in range(32)]
        warps.append(v[0])
    total = warps[0]
    for q in range(1, 8):
        total = total + warps[q]
    return total


@pytest.mark.parametrize("n", [1, 31, 255, 256, 257, 1000, 4096, 6145])
def test_block_sum_is_the_kernels_order(n):
    rng = np.random.default_rng(n)
    x = np.sqrt(rng.integers(0, 400, n).astype(np.float32).astype(np.float64)) * rng.uniform(0.5, 2.0, n)
    assert rfo.block_sum(x) == literal_block_sum(x)


def test_block_sum_differs_from_numpys_sum():
    """The kernel's order is not numpy's pairwise sum: on these sums of square roots the two round differently, so a
    mean compared only to a tolerance could flip the accept / undo decision where two rounds' means are close."""
    rng = np.random.default_rng(0)
    differ = 0
    for _ in range(50):
        x = np.sqrt(rng.integers(0, 400, 3000).astype(np.float64))
        differ += rfo.block_sum(x) != float(x.sum())
    assert differ >= 10, differ


def test_mean_distance_skips_dropped_pairs_in_place():
    """A dropped pair adds nothing on its thread; the kept pairs keep their silhouette index's thread."""
    rng = np.random.default_rng(1)
    d2 = rng.integers(0, 400, 2000).astype(np.float32)
    j = np.where(rng.random(2000) < 0.3, -1, 5)
    n, m = rfo.mean_distance(j, d2)
    x = np.where(j >= 0, np.sqrt(d2.astype(np.float64)), 0.0)
    assert n == int((j >= 0).sum()) and m == literal_block_sum(x) / n
    assert rfo.mean_distance(np.full(3, -1), d2[:3])[0] == 0 and np.isnan(rfo.mean_distance(np.full(3, -1), d2[:3])[1])


def test_singular_through_refine_image():
    """`SINGULAR` needs A + 1e-3 diag(A) not positive definite.  A = sum J^T J is positive semidefinite, so with
    every diagonal entry positive the damped matrix is positive definite (scaled by its diagonal, its eigenvalues lie
    in [1e-3, 6 + 1e-3]) and fp64 Cholesky succeeds: it fails only on a zero diagonal entry or a non-finite sum.
    A zero entry needs every pair's point to leave one parameter's projection exactly unchanged; here every silhouette
    point lies on the optical axis line through the object's origin, so no rotation about that axis moves it."""
    (v, f), Ks, pose, mask = rf.singular_scene()
    tr = []
    P, info = rfo.refine_image(mask, pose, Ks, v, f, 0.05, 5.0, trace=tr)
    assert info["status"] == rfo.SINGULAR and info["pairs"] == 6
    assert info["dist_before"] == info["dist_after"] == 0.0
    assert np.array_equal(P, pose) and len(tr) == 1
    A, _ = tr[0]["normal_eq"][0]
    assert A[2, 2] == 0.0 and not A[2].any() and (np.delete(np.diag(A), 2) > 0).all()


def test_gauss_newton_step_refuses_a_zero_diagonal_and_non_finite_sums():
    rng = np.random.default_rng(2)
    J = rng.normal(size=(20, 6))
    A, g = J.T @ J, rng.normal(size=6)
    pose = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    assert rfo.gauss_newton_step(A, g, pose) is not None
    for k in range(6):
        Z = A.copy()
        Z[k, :] = Z[:, k] = 0.0
        assert rfo.gauss_newton_step(Z, g, pose) is None, k
    for bad in (np.nan, np.inf):
        B = A.copy()
        B[1, 3] = B[3, 1] = bad
        assert rfo.gauss_newton_step(B, g, pose) is None
