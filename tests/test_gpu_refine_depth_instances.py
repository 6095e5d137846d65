"""GPU: `refine_poses_depth_instances` (DESIGN.md §31) against `refine_poses_depth` on each instance's own mask and
against `refine_instances` of tests/refine_depth_instance_cases.py (a loop over
oracle/refine_depth_oracle.py).

- L = 1 on a {0,1} map is bit for bit `refine_poses_depth` on that mask (poses, info, trace), for every label dtype,
  float32 depth and uint16 depth with a scale.
- Composited scenes of overlapping lumpy meshes, per-image K, b = 2, L = 4 with one absent row: every present row is
  bit for bit `refine_poses_depth` on its own mask, the first round matches the oracle bit for bit, the absent row
  passes through, instances touch and lose pairs to the rule, one instance touches the image border.
- Degenerate rows (no readings, render off-screen, an empty instance, num = 0) keep their input and leave the others
  alone.
- No host synchronisation, run-to-run identity, graph replay with new labels, depth, poses and num.
- Accuracy after keypoint-anchored `refine_poses_instances`, printed and bounded."""
import numpy as np
import pytest
import torch

from oracle import refine_depth_oracle as rdo
from pvnet_b200 import refine as rfn
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import refine_depth_instance_cases as ric

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 240, 320
MESH = rf.lumpy_mesh()
GATE = rdc.GATE


def t(a, dt=None):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV, dtype=dt)


def mesh():
    return t(MESH[0]), t(MESH[1])


def scene(xs, zs, seed, K, hole=None):
    rng = np.random.default_rng(seed)
    P = ric.poses_at(xs, zs, rng)
    lab, obs = ric.composite(rf.device_depth(DEV), MESH, K, P, H, W, hole=hole, rng=rng)
    return lab, obs, P


def batch(seed=0, hole=True):
    """b = 2, L = 4, per-image K: image 0 holds three overlapping instances (row 3 absent), image 1 four, the first
    crossing the left border.  -> labels [2,H,W] int64, depth [2,H,W] f32, true poses, starts 2 degrees and 5 mm off
    [2,4,3,4], num, K [2,3,3]."""
    K = np.stack([ric.linemod_k(H, W), ric.linemod_k(H, W, 1.05)])
    K[1, 0, 2] += 3.0
    l0, o0, P0 = scene((-0.08, 0.0, 0.08), (0.5, 0.52, 0.54), seed, K[0], (100, 150, 12) if hole else None)
    l1, o1, P1 = scene((-0.17, -0.06, 0.02, 0.10), (0.5, 0.53, 0.51, 0.55), seed + 1, K[1])
    Pt = np.stack([np.concatenate([P0, np.eye(3, 4)[None] * 3.0]), P1])
    rng = np.random.default_rng(seed + 2)
    Ps = np.stack([rf.perturb(p, rng, deg=2.0, dist=0.005) for p in Pt])
    Ps[0, 3] = np.eye(3, 4) * 3.0
    return np.stack([l0, l1]), np.stack([o0, o1]), Pt, Ps, np.array([3, 4], np.int32), K


def per_mask(lab, obs, Ps, K, i, j, **kw):
    v, f = mesh()
    return rfn.refine_poses_depth(t(lab[i] == j + 1, torch.uint8)[None], t(obs[i])[None], t(Ps[i, j])[None], t(K[i]),
                                  v, f, rf.NEAR, rf.FAR, GATE, **kw)


def assert_info_equal(a, b, i=0, j=0):
    """a: a one-image call's info, b: the instance call's; row (i, j) of b is a's image."""
    for key in a:
        assert torch.equal(torch.nan_to_num(a[key][0]), torch.nan_to_num(b[key][i, j])), key


def assert_trace_rows_equal(ta, tb, v):
    """a one-image call's trace against row v of the instance call's; entries past the kept count are not written."""
    assert torch.equal(ta["counts"][0], tb["counts"][v])
    assert torch.equal(torch.nan_to_num(ta["normal_eq"][0]), torch.nan_to_num(tb["normal_eq"][v]))
    m = int(ta["counts"][0, 0])
    for key in ("pair_idx", "X", "Y", "n"):
        assert torch.equal(ta[key][0, :m], tb[key][v, :m]), key


@pytest.mark.parametrize("ldtype", [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64])
@pytest.mark.parametrize("u16", [False, True])
def test_one_instance_equals_refine_poses_depth(ldtype, u16):
    K = ric.linemod_k(H, W)
    lab, obs, P = scene((0.0,), (0.5,), 1, K)
    P0 = rf.perturb(P, np.random.default_rng(2))
    depth, kw = t(obs), {}
    if u16:
        depth, kw = t(rdc.as_u16_mm(obs)), dict(depth_scale=1e-3)
    v, f = mesh()
    a, ia, ta = rfn.refine_poses_depth(t(lab[None] != 0, torch.uint8), depth[None], t(P0), t(K), v, f, rf.NEAR,
                                       rf.FAR, GATE, return_info=True, trace=True, **kw)
    b, ib, tb = rfn.refine_poses_depth_instances(t(lab[None]).to(ldtype), t(np.ones(1, np.int32)), depth[None],
                                                 t(P0[:, None]), t(K), v, f, rf.NEAR, rf.FAR, GATE, return_info=True,
                                                 trace=True, **kw)
    assert torch.equal(a, b[:, 0])
    assert_info_equal(ia, ib)
    assert_trace_rows_equal(ta, tb, 0)
    assert int(ia["pairs"][0]) > 100 and int(ia["status"][0]) & ~rfn.REJECTED == 0


def test_scene_rows_equal_their_masks_and_the_oracle():
    lab, obs, Pt, Ps, num, K = batch()
    v, f = mesh()
    R = 4
    out, info, tr = rfn.refine_poses_depth_instances(t(lab), t(num), t(obs), t(Ps), t(K), v, f, rf.NEAR, rf.FAR,
                                                     GATE, rounds=R, return_info=True, trace=True)
    # the absent row passes through
    assert torch.equal(out[0, 3].cpu(), torch.from_numpy(Ps[0, 3])) and int(info["status"][0, 3]) == rfn.NO_INSTANCE
    assert int(info["pairs"][0, 3]) == 0 and torch.isnan(info["dist_before"][0, 3])
    assert (tr["counts"][3] == 0).all()
    # every present row is refine_poses_depth on its own mask, bit for bit
    for i in range(2):
        for j in range(num[i]):
            a, ia, ta = per_mask(lab, obs, Ps, K, i, j, rounds=R, return_info=True, trace=True)
            assert torch.equal(a[0], out[i, j]), (i, j)
            assert_info_equal(ia, info, i, j)
            assert_trace_rows_equal(ta, tr, i * 4 + j)
    # the oracle, from the same renders
    traces = {}
    ref, rinfo = ric.refine_instances(lab, num, obs, Ps, K, *MESH, rf.NEAR, rf.FAR, GATE, rounds=R,
                                      render=rf.device_depth(DEV), traces=traces)
    tr = {x: y.cpu().numpy() for x, y in tr.items()}
    st = info["status"].cpu().numpy()
    np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=0, atol=1e-9)
    assert np.array_equal(info["pairs"].cpu().numpy(), rinfo["pairs"])
    lost = 0
    render = rf.device_depth(DEV)
    for (i, j), otr in traces.items():
        o, vv = otr[0], i * 4 + j
        m = len(o["idx"])
        assert tr["counts"][vv].tolist() == [m, o["count"], o["mask_pixels"], o["covered_pixels"]], (i, j)
        assert m > 100, (i, j)
        assert np.array_equal(tr["pair_idx"][vv, :m], o["idx"]), (i, j)
        for key in ("X", "Y", "n"):
            assert np.array_equal(tr[key][vv, :m].view(np.uint64), o[key].view(np.uint64)), (i, j, key)
        A, g = o["normal_eq"][0]
        ne = tr["normal_eq"][vv]
        want = np.concatenate([A[np.triu_indices(6)], g])
        np.testing.assert_allclose(ne, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
        if st[i, j] != rinfo["status"][i, j]:          # an undo at convergence, where the two means agree to rounding
            assert st[i, j] ^ rinfo["status"][i, j] == rfn.REJECTED and len(otr) == R + 1, (i, j)
            assert abs(otr[-1]["mean"] - otr[-2]["mean"]) <= 1e-9 * rinfo["dist_before"][i, j], (i, j)
        # the same pixels with every instance in the mask: the pixels the rule drops
        rd = render(*MESH, K[i], Ps[i, j].astype(np.float32), H, W, rf.NEAR, rf.FAR)
        union = rdo.pairs(rd, lab[i] != 0, rdo.observed_depth(obs[i]), Ps[i, j], K[i], GATE, H * W)
        lost += int((lab[i].reshape(-1)[union["idx"]] == j + 1).sum()) - o["count"]
    assert lost > 0
    assert (lab[1][:, 0] == 1).any() and (lab[1][:, 0] == 1).sum() < H      # instance (1, 0) crosses the left border
    assert rinfo["status"][0, 3] == ric.NO_INSTANCE


def test_degenerate_rows_keep_their_input_and_leave_the_others_alone():
    lab, obs, Pt, Ps, num, K = batch(seed=5, hole=False)
    obs = obs.copy()
    Ps = Ps.copy()
    obs[0][lab[0] == 2] = 0                                     # instance (0, 1) has no readings
    Ps[1, 2, 2, 3] = -1.0                                       # instance (1, 2) renders off-screen (behind)
    num = np.array([4, 4], np.int32)                            # row (0, 3) is present but has no pixel
    v, f = mesh()
    out, info = rfn.refine_poses_depth_instances(t(lab), t(num), t(obs), t(Ps), t(K), v, f, rf.NEAR, rf.FAR, GATE,
                                                 return_info=True)
    st = info["status"].cpu().numpy()
    assert st[0, 1] == rfn.FEW_PAIRS and st[1, 2] == rfn.NO_SILHOUETTE and st[0, 3] == rfn.NO_CONTOUR
    for i, j in ((0, 1), (1, 2), (0, 3)):
        assert torch.equal(out[i, j].cpu(), torch.from_numpy(Ps[i, j])), (i, j)
    for i in range(2):
        for j in range(4):
            a, ia = per_mask(lab, obs, Ps, K, i, j, return_info=True)
            assert torch.equal(a[0], out[i, j]), (i, j)
            assert_info_equal(ia, info, i, j)
    assert st[0, 0] & ~rfn.REJECTED == 0 and st[1, 0] & ~rfn.REJECTED == 0
    z, iz = rfn.refine_poses_depth_instances(t(lab), t(np.zeros(2, np.int32)), t(obs), t(Ps), t(K), v, f, rf.NEAR,
                                             rf.FAR, GATE, return_info=True)
    assert torch.equal(z.cpu(), torch.from_numpy(Ps)) and (iz["status"] == rfn.NO_INSTANCE).all()
    assert (iz["pairs"] == 0).all() and torch.isnan(iz["dist_after"]).all()


def test_no_host_synchronisation_run_to_run_identical_and_graph_replay():
    labA, obsA, _, PsA, numA, K = batch(seed=9)
    labB, obsB, _, PsB, _, _ = batch(seed=12, hole=False)
    numB = np.array([1, 3], np.int32)
    v, f = mesh()
    k = t(K)
    args = (t(labA), t(numA), t(obsA), t(PsA), k, v, f, rf.NEAR, rf.FAR, GATE)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a, ia = rfn.refine_poses_depth_instances(*args, return_info=True)
        b, ib = rfn.refine_poses_depth_instances(*args, return_info=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a, b) and all(torch.equal(torch.nan_to_num(ia[x]), torch.nan_to_num(ib[x])) for x in ia)
    sl, sn, sd, sp = (x.clone() for x in args[:4])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        rfn.refine_poses_depth_instances(sl, sn, sd, sp, k, v, f, rf.NEAR, rf.FAR, GATE, rounds=4)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, info = rfn.refine_poses_depth_instances(sl, sn, sd, sp, k, v, f, rf.NEAR, rf.FAR, GATE, rounds=4,
                                                     return_info=True)
    for lab, num, obs, Ps in ((labA, numA, obsA, PsA), (labB, numB, obsB, PsB)):
        for x, y in ((sl, lab), (sn, num), (sd, obs), (sp, Ps)):
            x.copy_(t(y))
        g.replay()
        eager, ie = rfn.refine_poses_depth_instances(t(lab), t(num), t(obs), t(Ps), k, v, f, rf.NEAR, rf.FAR, GATE,
                                                     rounds=4, return_info=True)
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
        assert all(torch.equal(torch.nan_to_num(info[x]), torch.nan_to_num(ie[x])) for x in ie)
    assert (info["status"][0, 1:] == rfn.NO_INSTANCE).all()


def test_bad_arguments_raise():
    lab, obs, _, Ps, num, K = batch(seed=3, hole=False)
    v, f = mesh()
    L, n, d, p, k = t(lab), t(num), t(obs), t(Ps), t(K)
    ok = dict(near=rf.NEAR, far=rf.FAR, gate=GATE)
    rfn.refine_poses_depth_instances(L, n, d, p, k, v, f, **ok, rounds=0)
    bad = [((L.float(), n, d, p, k), ok),                                       # float labels
           ((L[0], n, d, p, k), ok),                                            # [H,W] labels
           ((L[:1], n, d, p, k), ok),                                           # batch mismatch
           ((L, n[:1], d, p, k), ok),                                           # num shape
           ((L, n, d[:1], p, k), ok),                                           # depth batch
           ((L, n, d[:, :, :-1], p, k), ok),                                    # depth size
           ((L, n, d.double(), p, k), ok),                                      # float64 depth
           ((L, n, d.to(torch.int32), p, k), ok),                               # int32 depth
           ((L, n, d, p[:, :, :2], k), ok),                                     # poses [b,L,2,4]
           ((L, n, d, torch.zeros(2, 33, 3, 4, device=DEV, dtype=torch.float64), k), ok),      # L = 33
           ((L, n, d, p, k[:1]), ok),                                           # K batch
           ((L, n, d, p, k), dict(ok, gate=0.0)),
           ((L, n, d, p, k), dict(ok, gate=float("inf"))),
           ((L, n, d, p, k), dict(ok, rounds=-1)),
           ((L, n, d, p, k), dict(ok, max_points=0)),
           ((L, n, d, p, k), dict(ok, max_points=(2 ** 31 - 1) // 9 // 8 + 1)),
           ((L, n, d, p, k), dict(ok, depth_scale=0.0)),
           ((L, n, d, p, k), dict(ok, near=1.0, far=0.5))]
    for args, kw in bad:
        with pytest.raises(ValueError):
            rfn.refine_poses_depth_instances(*args, v, f, **kw)
    big = torch.zeros(33, 8, 8, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):                                             # b * L = 1056
        rfn.refine_poses_depth_instances(big, torch.ones(33, dtype=torch.int32, device=DEV),
                                         torch.zeros(33, 8, 8, device=DEV), torch.zeros(33, 32, 3, 4, device=DEV), k[0],
                                         v, f, **ok)
    with pytest.raises(RuntimeError, match="CUDA"):
        rfn.refine_poses_depth_instances(L, n, d.cpu(), p, k, v, f, **ok)


# the largest translation error of depth refinement per instance started straight from these scenes' 3 degree / 1 cm
# starts, oracle on the CPU (mean 3.92 mm, largest 6.51 mm; DESIGN.md §31): the device chain, which starts from
# keypoint-anchored poses, must end with a mean below it
TRANS_BOUND_MM = 6.5


def test_accuracy_after_keypoint_anchored_refinement():
    """Seeded composited scenes of three overlapping instances, 3 degrees and 1 cm off: the start, keypoint-anchored
    `refine_poses_instances` and that followed by `refine_poses_depth_instances`."""
    v, f = mesh()
    pts = MESH[0][::15][:9]
    errs = {"start": [], "keypoints": [], "+ depth": []}
    for seed in range(6):
        K = ric.linemod_k(H, W)
        lab, obs, P = scene((-0.08, 0.0, 0.08), (0.5, 0.52, 0.54), 10 + seed, K)
        rng = np.random.default_rng(100 + seed)
        P0 = rf.perturb(P, rng, deg=3.0, dist=0.01)[None]
        kp = np.stack([np.stack(rf.rfo.project(pts.astype(np.float64), p, K), -1) for p in P])
        kp = kp + rng.normal(0, 1.0, kp.shape)
        wgt = np.tile([1.0, 0.0, 1.0], (1, 3, 9, 1))
        num = t(np.array([3], np.int32))
        a = rfn.refine_poses_instances(t(lab[None]), num, t(P0), t(K), v, f, rf.NEAR, rf.FAR,
                                       keypoints=t(kp[None], torch.float32), points_3d=t(pts, torch.float32),
                                       weights_2d=t(wgt, torch.float32))
        b, info = rfn.refine_poses_depth_instances(t(lab[None]), num, t(obs[None]), a, t(K), v, f, rf.NEAR, rf.FAR,
                                                   GATE, return_info=True)
        assert (info["dist_after"] <= info["dist_before"]).all()
        assert (info["status"] & ~rfn.REJECTED == 0).all()
        for name, Q in (("start", P0), ("keypoints", a.cpu().numpy()), ("+ depth", b.cpu().numpy())):
            errs[name] += [(*rf.pose_error(Q[0, j], P[j]), abs(Q[0, j, 2, 3] - P[j, 2, 3])) for j in range(3)]
    mean = {}
    for name, e in errs.items():
        mean[name] = np.array(e, np.float64).mean(0)
        print(f"{name}: rotation {mean[name][0]:.3f} deg, translation {1e3 * mean[name][1]:.2f} mm, "
              f"optical axis {1e3 * mean[name][2]:.2f} mm")
    assert mean["+ depth"][1] < mean["keypoints"][1]
    assert 1e3 * mean["+ depth"][1] < TRANS_BOUND_MM
