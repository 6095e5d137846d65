"""GPU: keypoint-anchored (`refine_poses(..., keypoints=)`, DESIGN.md §27) and depth-anchored (`refine_poses_depth`,
§28) refinement against oracle/refine_keypoints_oracle.py and oracle/refine_depth_oracle.py at their edges -- every
keypoint count's lane layout, lanes turned off by non-finite inputs, keypoints behind the camera and at camera depth
0, the depth pairs' count-then-rank stride, the 6-pair minimum, image borders and tiny images, readings that are
not readings, the gate at exact equality, a residual that is not a number, uint16 and strided inputs, and every
status on the device.  The oracles render with `render_mesh` (tests/refine_cases.device_depth).  First-round pairs,
X, Y and n bit for bit, the first step's sums to 1e-12, every round's pose to 1e-9, and status, pairs, dist_before
and cost_before bit for bit."""
import math

import numpy as np
import pytest
import torch

from oracle import refine_depth_oracle as rdo
from oracle import refine_keypoints_oracle as rko
from oracle import refine_oracle as rfo
from pvnet_b200 import refine
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import refine_keypoint_cases as rkc
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RENDER = rf.device_depth(DEV)
TOOL = rf.tool_mesh()
GATE = rdc.GATE


def t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def kof(K, i):
    return K if K.ndim == 2 else K[i]


def coverage(mesh, K, P, h, w):
    return render_mesh(t(mesh[0]), t(mesh[1]), t(K), t(P, torch.float32), h, w, rf.NEAR, rf.FAR).cpu().numpy()


def same(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


def close(a, b):
    return same(a, b) or abs(a - b) <= 1e-9 * max(1.0, abs(b))


def check_sums(ne, A, g):
    Ad = np.zeros((6, 6))
    Ad[np.triu_indices(6)] = ne[:21]
    Ad = Ad + np.triu(Ad, 1).T
    if not (np.isfinite(A).all() and np.isfinite(g).all()):
        assert not (np.isfinite(Ad).all() and np.isfinite(ne[21:]).all())
        return
    assert np.abs(Ad - A).max() <= 1e-12 * np.abs(A).max()
    assert np.abs(ne[21:] - g).max() <= 1e-12 * max(np.abs(g).max(), 1e-300)


def scene_k(b, h, w, f, rng):
    """Per-image K about f with skew and principal-point offsets, float32 [b,3,3]."""
    K = np.stack([rc.camera_for(h, w, f * rng.uniform(0.9, 1.1)) for _ in range(b)])
    K[:, 0, 1] = rng.normal(0, 1.0, b)
    K[:, :2, 2] += rng.normal(0, 2.0, (b, 2))
    return K.astype(np.float32)


# ---- keypoint term ----

def kp_check(mask, P0, K, pts, kp, lam, rounds=3, cov=None, wts=None, mesh=TOOL, gate=20.0):
    """The device at rounds = 0..rounds against rko.refine_image per image -> [(P, info, trace)] of the full run."""
    mask = np.asarray(mask)
    kw = dict(keypoints=t(kp), points_3d=t(pts), keypoint_weight=lam)
    if cov is not None:
        kw["cov"] = t(cov)
        from pvnet_b200 import extend_utils as eu
        wts = eu.covariance_to_weights(t(cov)).cpu().numpy()
    else:
        kw["weights_2d"] = t(wts)
    args = (t(mask, torch.uint8), t(P0), t(K), t(mesh[0]), t(mesh[1]), rf.NEAR, rf.FAR)
    out, info, tr = refine.refine_poses(*args, rounds=rounds, gate=gate, return_info=True, trace=True, **kw)
    per_k = [refine.refine_poses(*args, rounds=k, gate=gate, **kw).cpu().numpy() for k in range(rounds)]
    per_k.append(out.cpu().numpy())
    info = {x: y.cpu().numpy() for x, y in info.items()}
    tr = {x: y.cpu().numpy() for x, y in tr.items()}
    res = []
    for i in range(len(P0)):
        otr = []
        with np.errstate(all="ignore"):
            P, oi = rko.refine_image(mask[i], P0[i], kof(K, i), *mesh, rf.NEAR, rf.FAR, kp[i], pts, wts[i], lam,
                                     rounds=rounds, gate=gate, trace=otr, render=RENDER)
        if otr[0]["normal_eq"]:
            check_sums(tr["normal_eq"][i], *otr[0]["normal_eq"][0])
            check_sums(tr["keypoint_eq"][i], *otr[0]["kp_eq"][0])
        for k in range(rounds + 1):
            want = otr[k]["pose"] if k < len(otr) - 1 else P
            assert np.abs(per_k[k][i] - want).max() <= 1e-9, (i, k)
        assert int(info["status"][i]) == oi["status"] and int(info["pairs"][i]) == oi["pairs"], (i, info["status"][i],
                                                                                                oi)
        assert same(info["dist_before"][i], oi["dist_before"]) and same(info["cost_before"][i], oi["cost_before"]), i
        assert close(info["dist_after"][i], oi["dist_after"]) and close(info["cost_after"][i], oi["cost_after"]), i
        if np.isfinite(info["cost_before"][i]) and np.isfinite(info["cost_after"][i]):
            assert info["cost_after"][i] <= info["cost_before"][i], i
        res.append((P, oi, otr))
    return res


def kp_scene(b, h, w, f, seed, pts, sigma=1.5):
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    K = scene_k(b, h, w, f, rng)
    mask = coverage(TOOL, K, Pt, h, w) > 0
    kp, cov = rkc.keypoint_votes(Pt, K, pts, sigma, rng)
    cov = cov * rng.uniform(0.5, 4.0, (b, len(pts), 1, 1)).astype(np.float32)
    return Pt, P0, K, mask, kp, cov


@pytest.mark.parametrize("nk", [4, 5, 17, 31, 32])
def test_keypoint_counts_fill_their_lanes(nk):
    """nk keypoints on lanes 0..nk-1 of warp 0 and the rest off; lambda / nk with this nk.  Both weight forms."""
    pts = rkc.spread_keypoints(nk, seed=nk)
    Pt, P0, K, mask, kp, cov = kp_scene(2, 480, 640, 600.0, 40 + nk, pts)
    kp_check(mask, P0, K, pts, kp, 0.5, cov=cov)
    wts = rkc.isotropic_weights(cov)
    wts[:, :, 1] = 0.2 * wts[:, :, 0]                                          # an off-diagonal weight too
    res = kp_check(mask, P0, K, pts, kp, 2.0, wts=wts)
    assert all(r[1]["status"] & ~rfo.REJECTED == 0 for r in res)


def test_non_finite_inputs_turn_off_their_own_lane():
    """Image 0: a NaN keypoint coordinate; 1: +inf and -inf weights; 2: every keypoint off; 3: clean.  Then a NaN in
    points_3d turns one lane off in every image.  lambda / nk keeps the full nk; each image equals its own call."""
    pts = rkc.tool_keypoints()
    Pt, P0, K, mask, kp, cov = kp_scene(4, 480, 640, 600.0, 71, pts)
    wts = rkc.isotropic_weights(cov)
    kp[0, 3, 1] = np.nan
    wts[1, 5, 2] = np.inf                                                      # the last of the eight values
    wts[1, 6, 0] = -np.inf
    kp[2] = np.nan
    res = kp_check(mask, P0, K, pts, kp, 1.0, wts=wts)
    assert [rko.Keypoints(kp[i], pts, wts[i], 1.0).on.sum() for i in range(4)] == [7, 6, 0, 8]
    assert res[2][2][0]["kd"] == 0.0 and res[2][1]["cost_before"] == res[2][1]["dist_before"]
    pts_nan = pts.copy()
    pts_nan[2, 1] = np.nan
    res2 = kp_check(mask, P0, K, pts_nan, kp, 1.0, wts=wts)
    assert [rko.Keypoints(kp[i], pts_nan, wts[i], 1.0).on.sum() for i in range(4)] == [6, 5, 0, 7]
    assert res2[3][1]["cost_before"] != res[3][1]["cost_before"]
    for P3 in (pts, pts_nan):
        args = (t(mask, torch.uint8), t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR)
        full, fi = refine.refine_poses(*args, keypoints=t(kp), points_3d=t(P3), weights_2d=t(wts),
                                       keypoint_weight=1.0, return_info=True)
        for i in range(4):
            one, oi = refine.refine_poses(t(mask[i:i + 1], torch.uint8), t(P0[i:i + 1]), t(K[i]), t(TOOL[0]),
                                          t(TOOL[1]), rf.NEAR, rf.FAR, keypoints=t(kp[i:i + 1]), points_3d=t(P3),
                                          weights_2d=t(wts[i:i + 1]), keypoint_weight=1.0, return_info=True)
            assert torch.equal(one[0], full[i]), i
            assert all(torch.equal(torch.nan_to_num(oi[x][0]), torch.nan_to_num(fi[x][i])) for x in fi), i


def test_keypoints_behind_the_camera_and_at_camera_depth_zero():
    """Image 0: one keypoint's model point 10 cm behind the camera at the start.  Image 1: R = I, t = (0, 0, 0.5) and
    the point (0, 0, -0.5), at camera depth 0 exactly: its distance is NaN, the first step's sums are not finite,
    and the image stops SINGULAR at its input."""
    h, w = 480, 640
    rng = np.random.default_rng(81)
    K = scene_k(2, h, w, 600.0, rng)
    Pt = rf.true_poses(2, rng)
    P0 = rf.perturb(Pt, rng)
    P0[1] = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    Pt[1] = rf.perturb(P0[1:2], rng, 2.0, 0.005)[0]
    mask = coverage(TOOL, K, Pt, h, w) > 0
    pts = np.repeat(rkc.tool_keypoints()[None], 2, 0)
    kp, cov = rkc.keypoint_votes(Pt, K, pts[0], 1.0, rng)
    wts = rkc.isotropic_weights(cov)
    behind = P0[0, :, :3].T @ (np.array([0.0, 0.0, -0.1]) - P0[0, :, 3])      # camera (0, 0, -0.1) at the start
    for i, X in ((0, behind), (1, np.array([0.0, 0.0, -0.5]))):
        p = pts[0].copy()
        p[7] = X
        res = kp_check(mask[i:i + 1], P0[i:i + 1], K[i], p, kp[i:i + 1], 0.5, wts=wts[i:i + 1])
        z = rkc.camera_depth(P0[i], p[7])
        if i == 0:
            assert z < 0 and np.isfinite(res[0][2][0]["kd"])
        else:
            assert z == 0.0 and np.isnan(res[0][2][0]["kd"])
            assert res[0][1]["status"] == rfo.SINGULAR and np.array_equal(res[0][0], P0[1])


def test_a_cost_that_is_not_a_number_is_undone():
    """A keypoint with zero weights adds exactly nothing to the steps, wherever it is.  Placed at camera depth 0
    exactly at the pose the first round's steps reach (read back from the device), it makes the second evaluation's
    C NaN (the oracle's C at that pose is NaN too): the round is undone, REJECTED, and the returned C is the input's.
    The oracle's own steps end within rounding of that pose, not on it, so this case is held to the oracle's rule
    at the device's pose rather than to an oracle run."""
    h, w = 480, 640
    pts = rkc.tool_keypoints()
    Pt, P0, K, mask, kp, cov = kp_scene(1, h, w, 600.0, 91, pts)
    wts = rkc.isotropic_weights(cov)
    wts[0, 7] = 0.0
    args = (t(mask, torch.uint8), t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR)
    kw = dict(keypoints=t(kp), weights_2d=t(wts), keypoint_weight=0.5, return_info=True)
    P1, i1 = refine.refine_poses(*args, rounds=1, points_3d=t(pts), **kw)
    assert int(i1["status"][0]) == 0                                           # the first round's steps were kept
    P1 = P1[0].cpu().numpy()
    p = pts.copy()
    p[7] = rkc.point_at_zero_depth(P1)
    assert rkc.camera_depth(P0[0], p[7]) != 0.0
    term = rko.Keypoints(kp[0], p, wts[0], 0.5)
    with np.errstate(all="ignore"):
        assert np.isnan(term.cost(0.0, P1, K[0])) and np.isfinite(term.cost(0.0, P0[0], K[0]))
    for rounds in (1, 3):
        out, info = refine.refine_poses(*args, rounds=rounds, points_3d=t(p), **kw)
        info = {x: y.cpu().numpy() for x, y in info.items()}
        assert np.array_equal(out[0].cpu().numpy(), P0[0]) and info["status"][0] == refine.REJECTED, rounds
        assert info["cost_after"][0] == i1["cost_before"][0].item() == info["cost_before"][0], rounds
        assert info["dist_after"][0] == info["dist_before"][0], rounds


def test_keypoint_statuses():
    """SINGULAR with keypoints on: `singular_scene`, its five keypoints and a lambda so small that lambda / nk times
    every keypoint sum rounds to 0 (tests/test_refine_anchored_edges_cpu.py finds it); keypoint_weight = 0; and a
    second round whose render leaves the image (keypoints pull the pose 0.4 m sideways), which is undone."""
    (v, f), K, pose, m = rf.singular_scene()
    pts = rkc.singular_scene_keypoints()
    u, vv = rfo.project(pts.astype(np.float64), pose, K)
    kp = np.stack([u, vv], -1).astype(np.float32)[None]
    wts = rkc.isotropic_weights(np.broadcast_to(0.25 * np.eye(2), (1, 5, 2, 2)))
    P0 = pose.copy()
    P0[:, :3] = rf.axis_angle([0.0, 0.0, np.deg2rad(3.0)]) @ P0[:, :3]
    for lam, st in ((1e-323, rfo.SINGULAR), (0.0, rfo.SINGULAR), (0.25, 0)):
        res = kp_check(m[None], P0[None], K, pts, kp, lam, wts=wts, mesh=(v, f))
        assert res[0][1]["status"] & ~rfo.REJECTED == st, lam
    pts8 = rkc.tool_keypoints()
    Pt, P0, K, mask, kp, cov = kp_scene(2, 96, 128, 150.0, 93, pts8)
    res = kp_check(mask, P0, K, pts8, kp, 0.0, cov=cov)                           # keypoint_weight = 0
    away = Pt.copy()
    away[:, 0, 3] += 0.4
    kp_far, _ = rkc.keypoint_votes(away, K, pts8, 0.0, np.random.default_rng(0))
    res = kp_check(mask, P0, K, pts8, kp_far, 1e4, rounds=2, cov=cov)
    for P, oi, otr in res:
        assert oi["status"] == rfo.REJECTED and len(otr) == 2 and otr[1]["n"] < rfo.MIN_PAIRS


# ---- depth term ----

def depth_check(mask, obs, P0, K, mesh=TOOL, gate=GATE, rounds=3, max_points=4096, depth_scale=1.0):
    """The device at rounds = 0..rounds against rdo.refine_image per image -> [(P, info, trace)] of the full run."""
    mask, obs = np.asarray(mask), np.asarray(obs)
    args = (t(mask), t(obs), t(P0), t(K), t(mesh[0]), t(mesh[1]), rf.NEAR, rf.FAR, gate)
    kw = dict(max_points=max_points, depth_scale=depth_scale)
    out, info, tr = refine.refine_poses_depth(*args, rounds=rounds, return_info=True, trace=True, **kw)
    per_k = [refine.refine_poses_depth(*args, rounds=k, **kw).cpu().numpy() for k in range(rounds)]
    per_k.append(out.cpu().numpy())
    info = {x: y.cpu().numpy() for x, y in info.items()}
    tr = {x: y.cpu().numpy() for x, y in tr.items()}
    res = []
    for i in range(len(P0)):
        otr = []
        P, oi = rdo.refine_image(mask[i], obs[i], P0[i], kof(K, i), *mesh, rf.NEAR, rf.FAR, gate, rounds=rounds,
                                 max_points=max_points, depth_scale=depth_scale, trace=otr, render=RENDER)
        o = otr[0]
        m = len(o["idx"])
        assert tr["counts"][i].tolist() == [m, o["count"], o["mask_pixels"], o["covered_pixels"]], i
        assert np.array_equal(tr["pair_idx"][i, :m], o["idx"]), i
        for key in ("X", "Y", "n"):
            assert np.array_equal(tr[key][i, :m].view(np.uint64), o[key].view(np.uint64)), (i, key)
        if o["normal_eq"]:
            check_sums(tr["normal_eq"][i], *o["normal_eq"][0])
        for k in range(rounds + 1):
            want = otr[k]["pose"] if k < len(otr) - 1 else P
            assert np.abs(per_k[k][i] - want).max() <= 1e-9, (i, k)
        assert int(info["status"][i]) == oi["status"] and int(info["pairs"][i]) == oi["pairs"], (i, info["status"][i],
                                                                                                oi)
        assert same(info["dist_before"][i], oi["dist_before"]) and close(info["dist_after"][i], oi["dist_after"]), i
        res.append((P, oi, otr))
    return res


def tool_depth_scene(b, h, w, f, seed, depth=(0.45, 0.6)):
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(b, rng, depth=depth)
    P0 = rf.perturb(Pt, rng)
    K = scene_k(b, h, w, f, rng)
    obs = coverage(TOOL, K, Pt, h, w)
    return Pt, P0, K, (obs > 0).astype(np.uint8), obs


def test_the_pair_stride_at_every_cap():
    """One 480x640 image with n > 4096 pairs, at max_points 1, 2, 7, ceil(n/2), n - 1, n, n + 1 and the default;
    its stride-1 pairs run across 4096-pixel chunks and 16-pixel thread spans.  Then b = 64 at ceil(n/2)."""
    Pt, P0, K, mask, obs = tool_depth_scene(1, 480, 640, 600.0, 7, depth=(0.4, 0.4))
    _, tr = refine.refine_poses_depth(t(mask), t(obs), t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR, GATE,
                                      rounds=0, max_points=10 ** 5, trace=True)
    n = int(tr["counts"][0, 1])
    assert n > 4096, n
    for mp in (1, 2, 7, -(-n // 2), n - 1, n, n + 1, 4096):
        res = depth_check(mask, obs, P0, K, rounds=2, max_points=mp)
        o = res[0][2][0]
        assert o["count"] == n and len(o["idx"]) == -(-n // -(-n // mp)), mp
        assert (res[0][1]["status"] == rfo.FEW_PAIRS) == (len(o["idx"]) < 6), mp
        if mp > n:
            assert rdc.straddles(o["idx"], 4096) and rdc.straddles(o["idx"], 16)
    Pt, P0, K, mask, obs = tool_depth_scene(64, 480, 640, 600.0, 8, depth=(0.4, 0.45))
    res = depth_check(mask, obs, P0, K, rounds=1, max_points=-(-n // 2))
    assert sum(r[2][0]["count"] > -(-n // 2) for r in res) >= 1


def test_the_six_pair_minimum_borders_and_tiny_images():
    """3 x 7 and 3 x 8 mask strips on a tilted plane: exactly 5 pairs (FEW_PAIRS) and 6 (refined).  A plane filling
    the image: pairs on rows and columns 1 and h - 2 / w - 2, none on the outer ones.  1x1, 2xN, Nx2 and 3x3."""
    h, w = 24, 32
    mesh, K, P = rdc.tilted_plane(h, w, 40.0)
    obs = coverage(mesh, K, P[None], h, w)[0]
    P0 = rf.perturb(P[None], np.random.default_rng(2), 1.0, 0.003)[0]
    masks = np.stack([rdc.strip((h, w), 10, 12, 3, 7), rdc.strip((h, w), 10, 12, 3, 8), np.ones((h, w), np.uint8)])
    res = depth_check(masks, np.stack([obs] * 3), np.stack([P0] * 3), K, mesh=mesh, rounds=2)
    assert [len(r[2][0]["idx"]) for r in res[:2]] == [5, 6]
    assert res[0][1]["status"] == rfo.FEW_PAIRS and res[1][1]["status"] & ~rfo.REJECTED == 0
    r, c = np.divmod(res[2][2][0]["idx"], w)
    assert r.min() == 1 and r.max() == h - 2 and c.min() == 1 and c.max() == w - 2
    for hh, ww in ((1, 1), (2, 9), (9, 2), (3, 3)):
        mesh, K, P = rdc.tilted_plane(hh, ww, 4.0 * max(hh, ww))
        obs = coverage(mesh, K, P[None], hh, ww)
        assert (obs > 0).all()
        res = depth_check(np.ones((1, hh, ww), np.uint8), obs, P[None], K, mesh=mesh, rounds=1)
        assert res[0][1]["status"] == rfo.FEW_PAIRS and len(res[0][2][0]["idx"]) == (hh == ww == 3)


def test_readings_that_are_not_readings():
    """Single pixels inside the object read NaN, +inf, -inf, -1, -0.0 (no reading: neither they nor their four
    neighbours pair) and the least fp32 subnormal (a reading: its neighbours still pair).  Then the tiny-ray scene,
    whose centre pixel lies on the surface but whose normal is 0 / 0: dropped by the residual's finiteness alone."""
    h, w = 120, 160
    Pt, P0, K, mask, obs = tool_depth_scene(1, h, w, 300.0, 13)
    sites = rf.hole_sites((mask[0] > 0) & (coverage(TOOL, K, P0, h, w)[0] > 0))
    pick = sites[np.linspace(0, len(sites) - 1, 6).astype(int)]
    vals = np.array([np.nan, np.inf, -np.inf, -1.0, -0.0, 1e-45], np.float32)
    obs = obs.copy()
    obs.reshape(-1)[pick] = vals
    assert obs.reshape(-1)[pick[5]] > 0
    res = depth_check(mask, obs, P0, K, rounds=2)
    idx = set(res[0][2][0]["idx"].tolist())
    for p in pick[:5]:
        assert not {p, p - 1, p + 1, p - w, p + w} & idx, p
    assert {pick[5] - 1, pick[5] + 1, pick[5] - w, pick[5] + w} & idx
    mesh, K, P, centre, nb = rdc.tiny_ray_scene()
    obs = coverage(mesh, K, P[None], 12, 12)
    obs.reshape(1, -1)[0, nb] = np.float32(1e-45)
    res = depth_check(np.ones((1, 12, 12), np.uint8), obs, P[None], K, mesh=mesh, rounds=1)
    o = res[0][2][0]
    assert centre not in o["idx"] and o["count"] > 6


def test_the_gate_at_exact_equality():
    """gate = |R X + t - Y| of one pair as the oracle computes it keeps that pair; nextafter(gate, 0) drops it."""
    Pt, P0, K, mask, obs = tool_depth_scene(1, 120, 160, 300.0, 17)
    o = depth_check(mask, obs, P0, K, rounds=0)[0][2][0]
    _, dist = rdo.residuals(o["X"], o["Y"], o["n"], P0[0])
    j = int(np.argsort(dist)[len(dist) // 2])
    gate = float(dist[j])
    kept = depth_check(mask, obs, P0, K, gate=gate, rounds=1)[0][2][0]
    assert o["idx"][j] in kept["idx"]
    dropped = depth_check(mask, obs, P0, K, gate=float(np.nextafter(gate, 0.0)), rounds=1)[0][2][0]
    assert o["idx"][j] not in dropped["idx"] and len(dropped["idx"]) < len(kept["idx"])


def test_uint16_readings_strided_depth_and_masks():
    """uint16 readings 0, 1 and 65535, read at 1e-3 and at a scale where fp32(65535) * scale overflows to inf (no
    reading); a non-contiguous depth view; an int64 mask of 256 and a strided bool mask."""
    h, w = 120, 160
    Pt, P0, K, mask, obs = tool_depth_scene(2, h, w, 300.0, 19)
    d16 = rdc.as_u16_mm(obs)
    sites = rf.hole_sites(mask[0] > 0)
    d16[0].reshape(-1)[sites[::4][:6]] = [0, 1, 65535, 0, 1, 65535]
    for scale in (1e-3, 6e33):
        with np.errstate(over="ignore"):
            assert np.isinf(np.float32(65535) * np.float32(scale)) == (scale > 1)
        res = depth_check(mask, d16, P0, K, rounds=2, depth_scale=scale)
        d32 = d16.astype(np.float32) * np.float32(scale)
        args = (t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR, GATE)
        a, ia = refine.refine_poses_depth(t(mask), t(d16), *args, depth_scale=scale, return_info=True)
        b_, ib = refine.refine_poses_depth(t(mask), t(d32), *args, return_info=True)
        assert torch.equal(a, b_) and all(torch.equal(torch.nan_to_num(ia[x]), torch.nan_to_num(ib[x])) for x in ia)
        assert (res[0][1]["status"] == rfo.FEW_PAIRS) == (scale > 1)
    args = (t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR, GATE)
    ref, ri = refine.refine_poses_depth(t(mask), t(obs), *args, return_info=True)
    wide = torch.zeros((2, h, 2 * w), dtype=torch.float32, device=DEV)
    wide[:, :, 1::2] = t(obs)
    wmask = torch.zeros((2, h, 2 * w), dtype=torch.bool, device=DEV)
    wmask[:, :, ::2] = t(mask > 0)
    for m, d in ((t(mask), wide[:, :, 1::2]), (t(mask, torch.int64) * 256, t(obs)), (wmask[:, :, ::2], t(obs))):
        assert not d.is_contiguous() or not m.is_contiguous() or int(m.max()) == 256
        out, oi = refine.refine_poses_depth(m, d, *args, return_info=True)
        assert torch.equal(out, ref) and all(torch.equal(torch.nan_to_num(oi[x]), torch.nan_to_num(ri[x])) for x in ri)


def test_depth_statuses_and_a_mixed_batch():
    """SINGULAR: a flat face at R = I, every normal (0, 0, -1).  A start already at its own render: every residual
    0, the step 0, and equal means are kept (status 0).  REJECTED at the third evaluation with fewer than six pairs.
    Then one batch of an ordinary image, a SINGULAR front-face rectangle, a 5-pair strip and the shrinking strip:
    each equals its own call bit for bit."""
    mesh, K, P = rdc.flat_face(24, 32, 40.0)
    obs = coverage(mesh, K, P[None], 24, 32)
    P0 = rdc.along_axis(P[None], 0.002)
    res = depth_check(np.ones((1, 24, 32), np.uint8), obs, P0, K, mesh=mesh, rounds=2)
    assert res[0][1]["status"] == rfo.SINGULAR and np.array_equal(res[0][2][0]["n"], np.tile([0.0, 0.0, -1.0],
                                                                                           (len(res[0][2][0]["n"]), 1)))
    tool = rdc.tilted_tool()
    K = rc.camera_for(120, 160, 300.0)
    P = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])[None]
    obs = coverage(tool, K, P, 120, 160)
    res = depth_check((obs > 0).astype(np.uint8), obs, P, K, mesh=tool, rounds=3)
    assert res[0][1]["status"] == 0 and [r["mean"] for r in res[0][2]] == [0.0] * 4
    m, dt, P0, K = rdc.shrinking_strip(RENDER)
    res = depth_check(m[None], dt[None], P0[None], K, rounds=3)
    assert res[0][1]["status"] == rfo.REJECTED and res[0][2][2]["n_pairs"] < 6
    h, w = 60, 80
    Pt, Pa, Ka, ma, oa = tool_depth_scene(1, h, w, 150.0, 23)
    Pf = np.hstack([np.eye(3), [[0.0], [0.0], [0.5]]])
    of = coverage(TOOL, K, Pf[None], h, w)[0]
    mf = rdc.strip((h, w), 28, 28, 5, 20)
    assert (of[28:33, 28:48] == of[28, 30]).all()
    masks = np.stack([ma[0], mf, rdc.strip((h, w), 28, 28, 3, 7), m])
    obs = np.stack([oa[0], of, of, dt])
    P0s = np.stack([Pa[0], rdc.along_axis(Pf[None], 0.002)[0], Pf, P0])
    Ks = np.stack([Ka[0], K, K, K])
    res = depth_check(masks, obs, P0s, Ks, rounds=3)
    assert [r[1]["status"] for r in res][1:] == [rfo.SINGULAR, rfo.FEW_PAIRS, rfo.REJECTED]
    args = (t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR, GATE)
    full, fi = refine.refine_poses_depth(t(masks), t(obs), t(P0s), t(Ks), *args, return_info=True)
    for i in range(4):
        one, oi = refine.refine_poses_depth(t(masks[i:i + 1]), t(obs[i:i + 1]), t(P0s[i:i + 1]), t(Ks[i]), *args,
                                            return_info=True)
        assert torch.equal(one[0], full[i]), i
        assert all(torch.equal(torch.nan_to_num(oi[x][0]), torch.nan_to_num(fi[x][i])) for x in fi), i
