"""CPU: the pose-evaluation oracle (oracle/eval_oracle.py + pvo_find_nearest_point_idx in oracle/eval_oracle.c)
gives the known answers: its nearest-point search agrees with a float64 brute force on tie-free data and keeps the
lowest index on ties, and its metrics give the expected values for poses whose metrics are known in closed form."""
import numpy as np
import pytest

from oracle import eval_oracle as eo
from oracle import pnp_oracle as pno

K_LINEMOD = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])


def _brute(ref, que):
    d = ((que[:, None, :].astype(np.float64) - ref[None].astype(np.float64)) ** 2).sum(-1)
    return d.argmin(1)


@pytest.mark.parametrize("dim", [2, 3])
def test_search_matches_float64_brute_force(dim):
    rng = np.random.default_rng(dim)
    ref = rng.normal(size=(700, dim)).astype(np.float32)
    que = rng.normal(size=(333, dim)).astype(np.float32)
    got = eo.find_nearest_point_idx(ref, que)
    want = _brute(ref, que)
    d = ((que[:, None].astype(np.float64) - ref[None]) ** 2).sum(-1)
    d.sort(1)
    clear = (d[:, 1] - d[:, 0]) > 1e-5 * (1 + d[:, 0])        # margin far above fp32 rounding: no near-ties
    assert clear.mean() > 0.95
    assert np.array_equal(got[clear], want[clear])
    b = eo.find_nearest_point_idx(np.stack([ref, ref[::-1]]), np.stack([que, que]))
    assert np.array_equal(b[0], got) and np.array_equal(b[1][clear], 699 - want[clear])


def test_search_ties_keep_lowest_index_and_nan_never_wins():
    rng = np.random.default_rng(1)
    base = rng.normal(size=(50, 3)).astype(np.float32)
    ref = np.concatenate([base, base, base])                     # every point three times
    que = base[rng.permutation(50)] + np.float32(1e-3)
    got = eo.find_nearest_point_idx(ref, que)
    assert (got < 50).all()
    assert np.array_equal(got, _brute(base, que))
    ref2 = ref.copy()
    ref2[:10] = np.nan
    got2 = eo.find_nearest_point_idx(ref2, base[:10])
    assert np.array_equal(got2, np.arange(50, 60))               # the NaN copies lose to the next copy
    assert (eo.find_nearest_point_idx(np.full((5, 2), np.nan, np.float32), np.zeros((3, 2), np.float32)) == 0).all()


def _pose(rvec, t):
    return np.concatenate([pno.rodrigues(np.asarray(rvec, np.float64)), np.asarray(t, np.float64)[:, None]], 1)


def _cloud(n=500, seed=0):
    return np.random.default_rng(seed).uniform(-0.05, 0.05, (n, 3)).astype(np.float32)


def test_identical_poses_give_zeros():
    P = _pose([0.3, -0.2, 0.1], [0.02, -0.01, 0.7])
    for sym in (False, True):
        m, _ = eo.pose_metrics_one(P, P, _cloud(), K_LINEMOD, symmetric=sym, sym_proj=sym)
        assert np.array_equal(m[:3], np.zeros(3))
        # tr(R R^T) rounds to within an ulp of 3 and arccos turns that into ~1e-6 degrees, as in the reference
        assert 0.0 <= m[3] < 1e-5


def test_pure_translation():
    G = _pose([0.3, -0.2, 0.1], [0.02, -0.01, 0.7])
    P = G.copy()
    P[:, 3] += np.array([0.0, 0.03, 0.0])
    m, _ = eo.pose_metrics_one(P, G, _cloud(), K_LINEMOD)
    assert abs(m[0] - 0.03) < 1e-12 and abs(m[2] - 3.0) < 1e-9 and m[3] < 1e-5
    add_ok, _, cm_ok = eo.passes(m[None], diameter=0.5)
    assert add_ok[0] and cm_ok[0]


def test_six_degree_rotation_fails_5cm5deg():
    G = _pose([0.0, 0.0, 0.0], [0.0, 0.0, 0.8])
    P = _pose([0.0, np.deg2rad(6.0), 0.0], [0.0, 0.0, 0.8])
    m, _ = eo.pose_metrics_one(P, G, _cloud(), K_LINEMOD)
    assert abs(m[3] - 6.0) < 1e-9 and m[2] == 0.0
    assert not eo.passes(m[None], diameter=0.1)[2][0]


def test_symmetric_cloud_add_s_zero():
    half = _cloud(300, seed=3)
    cloud = np.concatenate([half, half * np.array([-1, -1, 1], np.float32)])   # invariant under 180 deg about z
    G = _pose([0.2, 0.1, -0.3], [0.01, 0.02, 0.6])
    Rz = pno.rodrigues(np.array([0.0, 0.0, np.pi]))
    P = G.copy()
    P[:, :3] = G[:, :3] @ Rz
    m_sym, idx = eo.pose_metrics_one(P, G, cloud, K_LINEMOD, symmetric=True, sym_proj=True)
    m, _ = eo.pose_metrics_one(P, G, cloud, K_LINEMOD)
    assert m_sym[0] < 1e-9 and m_sym[1] < 1e-6
    assert m[0] > 0.01 and m[1] > 1.0
    assert abs(m[3] - 180.0) < 1e-5


def test_principal_point_shift_moves_projection():
    G = _pose([0.1, 0.2, 0.3], [0.0, 0.0, 0.9])
    P = G.copy()
    P[:, 3] += np.array([0.004, 0.0, 0.0])
    cloud = _cloud()
    m0, _ = eo.pose_metrics_one(P, G, cloud, K_LINEMOD)
    K2 = K_LINEMOD.copy()
    K2[0, 2] += 17.0
    K2[1, 2] -= 4.0
    m1, _ = eo.pose_metrics_one(P, G, cloud, K2)
    assert abs(m1[1] - m0[1]) < 1e-9                            # both projections shift alike: the error does not move
    # the same shift applied to the prediction alone moves each point by exactly (17, -4) pixels
    Pg = eo.project(K2, eo.transform(G, cloud))
    P0 = eo.project(K_LINEMOD, eo.transform(G, cloud))
    assert np.abs(Pg - P0 - np.array([17.0, -4.0])).max() < 1e-9
    # a skewed K changes the error of a vertical offset, as the full 3x3 product implies
    P = G.copy()
    P[:, 3] += np.array([0.0, 0.004, 0.0])
    m0, _ = eo.pose_metrics_one(P, G, cloud, K_LINEMOD)
    Ks = K_LINEMOD.copy()
    Ks[0, 1] = 30.0
    ms, _ = eo.pose_metrics_one(P, G, cloud, Ks)
    Pp, Gp = eo.transform(P, cloud), eo.transform(G, cloud)
    want = np.mean(np.linalg.norm(eo.project(Ks, Pp) - eo.project(Ks, Gp), axis=1))
    assert abs(ms[1] - want) < 1e-9 and abs(ms[1] - m0[1]) > 1e-3
