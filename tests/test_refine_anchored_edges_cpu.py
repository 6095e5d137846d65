"""CPU: the edge scenes of tests/test_gpu_refine_anchored_edges.py hit the edges they exist for, on the oracles
(oracle/refine_depth_oracle.py, oracle/refine_keypoints_oracle.py) with `render_oracle` on meshes of a few faces:
exact pair counts, the stride, the flat face's normals and SINGULAR, a residual that is not a number, exact zero
residuals, the later-round undo, and the keypoint term at camera depth 0 and at a lambda that rounds away."""
import numpy as np
import pytest

from oracle import refine_depth_oracle as rdo
from oracle import refine_keypoints_oracle as rko
from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import refine_keypoint_cases as rkc
from tests import render_cases as rc


def render(mesh, K, P, h, w):
    return ro.render(*mesh, K, np.asarray(P, np.float32)[None], h, w, rf.NEAR, rf.FAR)[0][0]


def test_subsample_is_a_rank_and_stride_loop():
    """refine_oracle.subsample against the kernel's loop written out: count n, stride = ceil(n / max_points) when
    n > max_points, keep rank % stride == 0 at rank / stride."""
    for n in (0, 1, 5, 6, 7, 4095, 4096, 4097, 8191, 12289):
        idx = np.arange(n) * 3 + 1
        for mp in (1, 2, 7, max(1, -(-n // 2)), max(1, n - 1), max(1, n), n + 1, 4096):
            stride = -(-n // mp) if n > mp else 1
            out = np.full(mp, -1)
            for rank in range(n):
                if rank % stride == 0:
                    out[rank // stride] = idx[rank]
            kept = -(-n // stride) if n else 0
            assert np.array_equal(rfo.subsample(idx, mp), out[:kept]), (n, mp)
            assert kept <= mp


def test_strips_give_five_and_six_pairs_and_a_full_plane_every_inner_pixel():
    h, w = 24, 32
    mesh, K, P = rdc.tilted_plane(h, w, 40.0)
    d = render(mesh, K, P, h, w)
    assert (d > 0).all()
    for cols, n in ((7, 5), (8, 6)):
        pr = rdo.pairs(d, rdc.strip((h, w), 10, 12, 3, cols), d, P, K, rdc.GATE, 4096)
        assert pr["count"] == n and np.array_equal(pr["idx"], 11 * w + np.arange(13, 13 + n))
    P0 = rf.perturb(P[None], np.random.default_rng(2), 1.0, 0.003)[0]
    st = [rdo.refine_image(rdc.strip((h, w), 10, 12, 3, c), d, P0, K, *mesh, rf.NEAR, rf.FAR, rdc.GATE, rounds=2)[1]
          ["status"] for c in (7, 8)]
    assert st[0] == rfo.FEW_PAIRS and st[1] & ~rfo.REJECTED == 0
    pr = rdo.pairs(d, np.ones((h, w)), d, P, K, rdc.GATE, 4096)
    assert pr["count"] == (h - 2) * (w - 2)


def test_a_plane_over_several_chunks_straddles_them():
    """70 x 80 = 5600 pixels: the stride-1 pairs of a plane filling the image run across the 4096-pixel chunk and
    the 16-pixel thread spans; at max_points 7 every 749th is kept."""
    h, w = 70, 80
    mesh, K, P = rdc.tilted_plane(h, w, 100.0)
    d = render(mesh, K, P, h, w)
    pr = rdo.pairs(d, np.ones((h, w)), d, P, K, rdc.GATE, 10 ** 5)
    n = pr["count"]
    assert n == 68 * 78 > 4096 and rdc.straddles(pr["idx"], 4096) and rdc.straddles(pr["idx"], 16)
    sub = rdo.pairs(d, np.ones((h, w)), d, P, K, rdc.GATE, 7)
    assert np.array_equal(sub["idx"], pr["idx"][::-(-n // 7)]) and len(sub["idx"]) == 7


@pytest.mark.parametrize("h,w", [(1, 1), (2, 9), (9, 2), (3, 3)])
def test_tiny_images_have_at_most_one_pair(h, w):
    mesh, K, P = rdc.tilted_plane(h, w, 4.0 * max(h, w))
    d = render(mesh, K, P, h, w)
    assert (d > 0).all()
    pr = rdo.pairs(d, np.ones((h, w)), d, P, K, rdc.GATE, 4096)
    assert pr["count"] == (h == w == 3)
    assert rdo.refine_image(np.ones((h, w)), d, P, K, *mesh, rf.NEAR, rf.FAR, rdc.GATE)[1]["status"] == rfo.FEW_PAIRS


def test_the_flat_face_is_singular():
    h, w = 24, 32
    mesh, K, P = rdc.flat_face(h, w, 40.0)
    d = render(mesh, K, P, h, w)
    assert (d == np.float32(0.5)).all()
    pr = rdo.pairs(d, np.ones((h, w)), d, P, K, rdc.GATE, 4096)
    assert np.array_equal(pr["n"], np.tile([0.0, 0.0, -1.0], (len(pr["n"]), 1)))
    A, _ = rdo.normal_equations(pr["X"], pr["Y"], pr["n"], P)
    assert (np.diag(A)[[2, 3, 4]] == 0).all()
    P0 = rdc.along_axis(P[None], 0.002)[0]
    Pr, info = rdo.refine_image(np.ones((h, w)), d, P0, K, *mesh, rf.NEAR, rf.FAR, rdc.GATE)
    assert info["status"] == rfo.SINGULAR and np.array_equal(Pr, P0)


def test_a_normal_of_zero_length_gives_a_residual_that_is_not_a_number():
    """tiny_ray_scene: the centre's |d| is far below the gate, but |n| = 0 and e = NaN, so only the residual's
    finiteness drops it; a subnormal reading is a reading."""
    (v, f), K, P, centre, nb = rdc.tiny_ray_scene()
    d = render((v, f), K, P, 12, 12)
    assert (d == np.float32(0.5)).all()
    obs = d.copy()
    obs.reshape(-1)[nb] = np.float32(1e-45)
    zo = rdo.observed_depth(obs)
    assert (zo.reshape(-1)[nb] > 0).all()
    pr = rdo.pairs(d, np.ones((12, 12)), zo, P, K, rdc.GATE, 4096)
    assert centre not in pr["idx"] and pr["count"] > 6
    # the centre's pair, built as `pairs` builds it, fails only the finiteness test
    r, c = divmod(centre, 12)
    xn, yn = rdo.rays(12, 12, K)
    Q = [zo[rr, cc].astype(np.float64) * np.array([xn[rr, cc], yn[rr, cc], 1.0])
         for rr, cc in ((r, c + 1), (r, c - 1), (r + 1, c), (r - 1, c))]
    a, b = Q[0] - Q[1], Q[2] - Q[3]
    n = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])
    assert n[2] != 0 and (n[0] * n[0] + n[1] * n[1]) + n[2] * n[2] == 0
    X = rfo.back_project(np.array([centre]), d, P, K, 12)
    Y = (zo[r, c].astype(np.float64) * np.array([xn[r, c], yn[r, c], 1.0]))[None]
    with np.errstate(all="ignore"):
        e, dist = rdo.residuals(X, Y, (n / 0.0)[None], P)
    assert dist[0] <= rdc.GATE and np.isnan(e[0])


def test_a_start_at_its_own_render_has_exactly_zero_residuals():
    mesh = rdc.tilted_tool()
    K = rc.camera_for(120, 160, 300.0)
    P = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    d = render(mesh, K, P, 120, 160)
    tr = []
    Pr, info = rdo.refine_image(d > 0, d, P, K, *mesh, rf.NEAR, rf.FAR, rdc.GATE, rounds=3, trace=tr)
    assert info["status"] == 0 and np.array_equal(Pr, P)
    assert [x["mean"] for x in tr] == [0.0] * 4 and tr[0]["n_pairs"] > 1000


def test_the_shrinking_strip_is_undone_at_its_third_evaluation():
    m, dt, P0, K = rdc.shrinking_strip(rfo.oracle_depth)
    tr = []
    P, info = rdo.refine_image(m, dt, P0, K, *rf.tool_mesh(), rf.NEAR, rf.FAR, rdc.GATE, rounds=3, trace=tr)
    assert info["status"] == rfo.REJECTED and [x["n_pairs"] for x in tr][1:] == [7, 3]
    assert np.array_equal(P, tr[1]["pose"])


def test_a_point_at_camera_depth_zero():
    rng = np.random.default_rng(0)
    for P in rf.true_poses(20, rng):
        X = rkc.point_at_zero_depth(P)
        assert X.dtype == np.float32 and rkc.camera_depth(P, X) == 0.0
    P = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    assert rkc.camera_depth(P, np.array([0.0, 0.0, -0.5], np.float32)) == 0.0


def keypoint_scene(seed=91, h=120, w=160):
    K = rc.camera_for(h, w, 300.0)
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(1, rng)[0]
    P0 = rf.perturb(Pt[None], rng)[0]
    mask = render(rf.tool_mesh(), K, Pt, h, w) > 0
    pts = rkc.tool_keypoints()
    kp, cov = rkc.keypoint_votes(Pt[None], K, pts, 1.0, rng)
    return K, P0, mask, pts, kp[0], rkc.isotropic_weights(cov)[0]


def test_a_round_whose_cost_is_not_a_number_is_undone():
    """A zero-weight keypoint adds nothing to the steps; placed at camera depth 0 at the pose the first round
    reaches, it makes that round's C NaN, and the round is undone: the returned C is the input's."""
    K, P0, mask, pts, kp, wts = keypoint_scene()
    wts[7] = 0.0
    kw = dict(keypoints=kp, weights=wts, keypoint_weight=0.5)
    P1, i1 = rko.refine_image(mask, P0, K, *rf.tool_mesh(), rf.NEAR, rf.FAR, points_3d=pts, rounds=1, **kw)
    assert i1["status"] == 0
    p = pts.copy()
    p[7] = rkc.point_at_zero_depth(P1)
    tr = []
    with np.errstate(all="ignore"):
        P, info = rko.refine_image(mask, P0, K, *rf.tool_mesh(), rf.NEAR, rf.FAR, points_3d=p, rounds=3, trace=tr,
                                   **kw)
    assert np.array_equal(tr[1]["pose"], P1) and np.isnan(tr[1]["cost"]) and tr[1]["mean"] < tr[0]["mean"]
    assert info["status"] == rfo.REJECTED and np.array_equal(P, P0)
    assert info["cost_after"] == info["cost_before"] == i1["cost_before"]


def test_a_keypoint_at_camera_depth_zero_at_the_start_is_singular():
    K = rc.camera_for(120, 160, 300.0)
    Pt = np.hstack([rf.axis_angle([0.02, -0.03, 0.01]), [[0.0], [0.0], [0.5]]])
    mask = render(rf.tool_mesh(), K, Pt, 120, 160) > 0
    P0 = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    pts = rkc.tool_keypoints().copy()
    pts[7] = (0.0, 0.0, -0.5)
    u, vv = rfo.project(pts[:7].astype(np.float64), Pt, K)
    kp = np.concatenate([np.stack([u, vv], -1), [[80.0, 60.0]]]).astype(np.float32)
    with np.errstate(all="ignore"):
        P, info = rko.refine_image(mask, P0, K, *rf.tool_mesh(), rf.NEAR, rf.FAR, kp, pts, np.ones((8, 3), np.float32))
    assert info["status"] == rfo.SINGULAR and np.array_equal(P, P0) and np.isnan(info["cost_before"])


def test_a_lambda_that_rounds_away_leaves_singular_scene_singular():
    """lambda / nk times the keypoint sums underflows to 0 at lambda = 1e-323, so the dw_z row stays exactly zero;
    at 1e-300 the keypoints already hold it."""
    (v, f), K, pose, m = rf.singular_scene()
    pts = rkc.singular_scene_keypoints()
    u, vv = rfo.project(pts.astype(np.float64), pose, K)
    kp = np.stack([u, vv], -1).astype(np.float32)
    wts = rkc.isotropic_weights(np.broadcast_to(0.25 * np.eye(2), (5, 2, 2)))
    P0 = pose.copy()
    P0[:, :3] = rf.axis_angle([0.0, 0.0, np.deg2rad(3.0)]) @ P0[:, :3]
    st = {lam: rko.refine_image(m, P0, K, v, f, 0.05, 5.0, kp, pts, wts, lam)[1]["status"]
          for lam in (0.0, 1e-323, 1e-300, 0.25)}
    assert st[0.0] == st[1e-323] == rfo.SINGULAR
    assert st[1e-300] & rfo.SINGULAR == 0 and st[0.25] & rfo.SINGULAR == 0
