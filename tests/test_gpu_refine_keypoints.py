"""GPU: keypoint-anchored refinement (`refine_poses(..., keypoints=)`, `pvnet_refine_poses_keypoints`, DESIGN.md §27)
against oracle/refine_keypoints_oracle.py -- the first step's pair and keypoint sums to 1e-12, every round's pose to 1e-9, the
same accept / undo decisions -- its large-weight limit (the uncertainty-PnP pose), degenerate images, no host
synchronisation, graph replay, the keypoint-less path against the parent commit's poses, and
`PoseKeypointPipeline(refine=)`."""
import numpy as np
import pytest
import torch

from oracle import refine_keypoints_oracle as rko
from pvnet_b200 import extend_utils as eu
from pvnet_b200 import refine
from pvnet_b200 import ransac_voting_gpu as rv
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf
from tests import refine_keypoint_cases as rkc
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MESH = rf.tool_mesh()
PTS = rkc.tool_keypoints()


def t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def device_mesh():
    return t(MESH[0]), t(MESH[1])


def kof(K, i):
    return K if K.ndim == 2 else K[i]


def scene(b, h, w, seed, per_image_k, f=None, sigma=1.5):
    """True poses, starts 3 degrees and 1 cm away, K ([3,3] or [b,3,3] float32), the truth's coverage masks, and
    keypoints at the true projections plus `sigma` px of noise with covariances sigma^2 s_k I (s_k in 0.5..4)."""
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    f = f if f is not None else 2.5 * max(h, w)
    if per_image_k:
        K = np.stack([rc.camera_for(h, w, f * rng.uniform(0.9, 1.1)) for _ in range(b)])
        K[:, 0, 1] = rng.normal(0, 1.0, b)
        K[:, :2, 2] += rng.normal(0, 2.0, (b, 2))
        K = K.astype(np.float32)
    else:
        K = rc.camera_for(h, w, f)
    v, fc = device_mesh()
    depth = render_mesh(v, fc, t(K), t(Pt, torch.float32), h, w, rf.NEAR, rf.FAR)
    kp, cov = rkc.keypoint_votes(Pt, K, PTS, sigma, rng)
    cov = cov * rng.uniform(0.5, 4.0, (b, len(PTS), 1, 1)).astype(np.float32)
    return Pt, P0, K, (depth > 0).to(torch.uint8), kp, cov


def weights_of(cov):
    """The float32 weights the kernel reads: `covariance_to_weights` on the device."""
    return eu.covariance_to_weights(t(cov)).cpu().numpy()


def oracle_round_results(tr, P):
    """The oracle's result with rounds = k, for every k, from one trace of the full run: the pose evaluation k
    started from while the run went on past k, else the run's result."""
    return lambda k: tr[k]["pose"] if k < len(tr) - 1 else P


@pytest.mark.parametrize("per_image_k", [False, True])
def test_full_size_rounds_match_the_oracle(per_image_k):
    b, h, w, R, lam = 16, 480, 640, 8, 0.5
    Pt, P0, K, mask, kp, cov = scene(b, h, w, 3 + per_image_k, per_image_k, f=600.0)
    v, f = device_mesh()
    wts = weights_of(cov)
    args = (mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR)
    kw = dict(keypoints=t(kp), points_3d=t(PTS), cov=t(cov), keypoint_weight=lam)
    out, info, tr = refine.refine_poses(*args, rounds=R, return_info=True, trace=True, **kw)
    per_k = [refine.refine_poses(*args, rounds=k, **kw).cpu().numpy() for k in range(R)] + [out.cpu().numpy()]
    info = {x: y.cpu().numpy() for x, y in info.items()}
    tr = {x: y.cpu().numpy() for x, y in tr.items()}
    m = mask.cpu().numpy()
    render = rf.device_depth(DEV)
    statuses = set()
    for i in range(b):
        otr = []
        P, oi = rko.refine_image(m[i], P0[i], kof(K, i), *MESH, rf.NEAR, rf.FAR, rounds=R, trace=otr, render=render,
                                 keypoints=kp[i], points_3d=PTS, weights=wts[i], keypoint_weight=lam)
        # first round: the pair sums and the keypoint sums separately
        for key, (A, g) in (("normal_eq", otr[0]["normal_eq"][0]), ("keypoint_eq", otr[0]["kp_eq"][0])):
            ne = tr[key][i]
            Ad = np.zeros((6, 6))
            Ad[np.triu_indices(6)] = ne[:21]
            Ad = Ad + np.triu(Ad, 1).T
            assert np.abs(Ad - A).max() <= 1e-12 * np.abs(A).max(), (i, key)
            assert np.abs(ne[21:] - g).max() <= 1e-12 * np.abs(g).max(), (i, key)
        # every round's pose; the same decisions (an undo moves the pose by far more than 1e-9)
        at = oracle_round_results(otr, P)
        for k in range(R + 1):
            assert np.abs(per_k[k][i] - at(k)).max() <= 1e-9, (i, k)
        assert int(info["status"][i]) == oi["status"] and int(info["pairs"][i]) == oi["pairs"], i
        assert info["dist_before"][i] == oi["dist_before"] and info["cost_before"][i] == oi["cost_before"], i
        for key in ("dist_after", "cost_after"):
            assert abs(info[key][i] - oi[key]) <= 1e-9 * max(1.0, abs(oi[key])), (i, key)
        assert info["cost_after"][i] <= info["cost_before"][i]
        statuses.add(oi["status"])
    assert statuses <= {0, refine.REJECTED}, statuses


def test_a_large_keypoint_weight_gives_uncertainty_pnp():
    """lambda = 1e6: the uncertainty-PnP pose for the same float32 weights and the fp32-rounded K as float64 (no skew,
    which PnP does not read), to the oracle's bound (tests/test_refine_keypoints_cpu.py says why 1e-5)."""
    b, h, w = 8, 480, 640
    Pt, P0, K, mask, kp, cov = scene(b, h, w, 5, False, f=600.0)
    v, f = device_mesh()
    wts = eu.covariance_to_weights(t(cov))
    out, info = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, keypoints=t(kp), points_3d=t(PTS),
                                    weights_2d=wts, keypoint_weight=1e6, return_info=True)
    ref = eu.uncertainty_pnp_batched(t(kp), t(PTS), t(K).double(), weights_2d=wts)
    assert (info["status"] & ~refine.REJECTED == 0).all()
    assert (out - ref).abs().max().item() <= 1e-5
    assert (t(P0) - ref).abs().amax((1, 2)).min().item() > 1e-2


def test_degenerate_images_keep_their_input_and_leave_the_others_alone():
    b, h, w = 5, 96, 128
    Pt, P0, K, mask, kp, cov = scene(b, h, w, 7, True, f=150.0)            # a small object, far from the corner
    v, f = device_mesh()
    mask = mask.clone()
    mask[1] = 0                                                                 # empty mask
    mask[2] = 0
    mask[2, :8, :8] = 1                                                         # a mask far from the render
    P0 = P0.copy()
    P0[3, 2, 3] = -1.0                                                          # the render covers nothing
    kw = dict(keypoints=t(kp), points_3d=t(PTS), cov=t(cov))
    out, info = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, gate=10.0, return_info=True, **kw)
    st = info["status"].cpu().tolist()
    assert st[1] == refine.NO_CONTOUR and st[2] == refine.FEW_PAIRS and st[3] == refine.NO_SILHOUETTE
    assert st[0] & ~refine.REJECTED == 0 and st[4] & ~refine.REJECTED == 0
    assert torch.equal(out[1:4].cpu(), torch.from_numpy(P0[1:4]))
    assert torch.isnan(info["cost_before"][1:4]).all()
    for i in range(b):
        one = refine.refine_poses(mask[i:i + 1], t(P0[i:i + 1]), t(K[i]), v, f, rf.NEAR, rf.FAR, gate=10.0,
                                  keypoints=t(kp[i:i + 1]), points_3d=t(PTS), cov=t(cov[i:i + 1]))
        assert torch.equal(one[0], out[i]), i


def test_no_host_synchronisation_run_to_run_identical_and_graph_replay():
    b, h, w = 4, 96, 128
    PtA, P0A, K, maskA, kpA, covA = scene(b, h, w, 9, True)
    _, P0B, _, _, kpB, covB = scene(b, h, w, 10, True)
    maskB = (render_mesh(*device_mesh(), t(K), t(rf.perturb(P0B, np.random.default_rng(1), 1.0, 0.003), torch.float32),
                         h, w, rf.NEAR, rf.FAR) > 0).to(torch.uint8)
    v, f = device_mesh()
    p3 = t(PTS)
    p, k, kpt, ct = t(P0A), t(K), t(kpA), t(covA)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a, ia = refine.refine_poses(maskA, p, k, v, f, rf.NEAR, rf.FAR, return_info=True, keypoints=kpt, points_3d=p3,
                                    cov=ct)
        b_, ib = refine.refine_poses(maskA, p, k, v, f, rf.NEAR, rf.FAR, return_info=True, keypoints=kpt,
                                     points_3d=p3, cov=ct)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a, b_) and all(torch.equal(ia[x], ib[x]) for x in ia)
    sm, sp, skp, sc = maskA.clone(), t(P0A), t(kpA), t(covA)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        refine.refine_poses(sm, sp, k, v, f, rf.NEAR, rf.FAR, rounds=4, keypoints=skp, points_3d=p3, cov=sc)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, info = refine.refine_poses(sm, sp, k, v, f, rf.NEAR, rf.FAR, rounds=4, return_info=True, keypoints=skp,
                                        points_3d=p3, cov=sc)
    for mk, P, kp, cov in ((maskA, P0A, kpA, covA), (maskB, P0B, kpB, covB)):
        sm.copy_(mk)
        sp.copy_(t(P))
        skp.copy_(t(kp))
        sc.copy_(t(cov))
        g.replay()
        eager, ie = refine.refine_poses(mk, t(P), k, v, f, rf.NEAR, rf.FAR, rounds=4, return_info=True,
                                        keypoints=t(kp), points_3d=p3, cov=t(cov))
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and all(torch.equal(info[x], ie[x]) for x in ie)


# Keypoint-less refine_poses on this batch, computed with the parent commit's library (before the keypoint term):
# the float64 poses' bytes, status, pairs and the (dist_before, dist_after) bytes.
PARENT = dict(
    poses=("2881040b0e4ea93faf0ce91e6423e3bf9c4d4354ee98e9bfcf04ed018f9aa3bfa3c01087b849ccbf247a140bf733e9bf3010e022"
           "0b68e23fe2c85e8516939fbf7900c58a2d2befbfaa43406c3dfdc23f9493486293e6c5bf569b1e31f60edc3fc59fbf6ad0ef92bf"
           "a5a936ba23dcac3f9dd4f59092f1ef3f6170d00586738cbfed4507e70d49efbf054ad6c18ca0ca3f033de77c2a939ebf81bf3809"
           "bb3e91bfc83725abb1cbcabfc40817ee783fefbf632719e1e93eaa3f7252196adc8ee23f9ce2ce4ba3e5ed3f0851e0b26b12d23f"
           "2686978ebddccbbfe2f02c696f4c7ebfe29605c6c7f5a53fb93d9daf513ee6bf851d8288c9f6e6bf92f4800f5061463f02c12f08"
           "0ca7d6bf3d2ae073f627e53fccee1ba6502be5bf8ab001e58467dd3f3d0871efaf78debff65ff9fac471e43fdd0275ac2256e3bf"
           "db354fb52a2597bf19334f478350883fd7c61eb755d6e5bfdaf4ea864863e7bf40bde81ad33a95bf10cc7a783e23ecbf47d9c8e9"
           "d2bad6bfe362660c064fd43f02677ce1b872e03ffee01340f6d5bc3fae2d51f6101bedbf0c434d7c169ad93f187b4c6c921ea53f"
           "6bf1e93b3010eb3fefb92dcd92a2bfbf0abe67968f9ce0bfd6d753a7907e973f9851717ce4b0e03fb5213c80fa64d93f468c509f"
           "882be83f642dd3423a52e33fdb5a9c1367d6e7bfbc58ee3cc502ccbf3b5216eaec2ae43f53f5fc999240ab3f479fce2834e0e13f"
           "8f9379b3ed12e7bfbda69f2ec73bda3f02758602817b8f3f6b20498beb57d73f12003fed7809e53f4d320137a219e53fd0ac9e5c"
           "1b23df3f"),
    dist=("4769ff97ee9cf83fe6d59c111526e33f1faaf42b4ea40b40c49e956143fbbd3fb77af7a43cea0b40b6d65a6badb5b63ff3ebea56"
          "09c70b4028c459f90971c63f000000000000f87f000000000000f87f940b9bc7c66000400117752d0d59dd3f"),
    status=[16, 16, 0, 0, 1, 16], pairs=[161, 212, 248, 155, 0, 200])


def test_without_keypoints_the_parent_commits_poses():
    b, h, w = 6, 96, 128
    rng = np.random.default_rng(97)
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    K = np.stack([rc.camera_for(h, w, 320.0 * rng.uniform(0.9, 1.1)) for _ in range(b)]).astype(np.float32)
    v, f = device_mesh()
    mask = (render_mesh(v, f, t(K), t(Pt, torch.float32), h, w, rf.NEAR, rf.FAR) > 0).to(torch.uint8)
    mask[4] = 0
    out, info = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, return_info=True)
    want = torch.from_numpy(np.frombuffer(bytes.fromhex(PARENT["poses"]), np.float64).reshape(b, 3, 4).copy())
    dist = torch.from_numpy(np.frombuffer(bytes.fromhex(PARENT["dist"]), np.float64).reshape(b, 2).copy())
    assert torch.equal(out.cpu(), want)
    assert info["status"].cpu().tolist() == PARENT["status"] and info["pairs"].cpu().tolist() == PARENT["pairs"]
    got = torch.stack([info["dist_before"], info["dist_after"]], 1).cpu()
    assert torch.equal(torch.nan_to_num(got), torch.nan_to_num(dist))
    assert set(info) == {"status", "pairs", "dist_before", "dist_after"}


def test_bad_arguments_raise():
    Pt, P0, K, mask, kp, cov = scene(2, 32, 40, 11, False)
    v, f = device_mesh()
    p, k = t(P0), t(K)
    ok = dict(near=rf.NEAR, far=rf.FAR)
    kpt, p3, ct = t(kp), t(PTS), t(cov)
    wts = eu.covariance_to_weights(ct)
    refine.refine_poses(mask, p, k, v, f, **ok, keypoints=kpt, points_3d=p3, cov=ct)
    refine.refine_poses(mask, p, k, v, f, **ok, keypoints=kpt, points_3d=p3, weights_2d=wts, keypoint_weight=0.0)
    bad = [dict(keypoints=kpt),                                                  # no points_3d
           dict(keypoints=kpt, points_3d=p3),                                    # neither cov nor weights
           dict(keypoints=kpt, points_3d=p3, cov=ct, weights_2d=wts),            # both
           dict(points_3d=p3, cov=ct),                                           # no keypoints
           dict(keypoints=kpt[:1], points_3d=p3, cov=ct),                        # batch mismatch
           dict(keypoints=kpt[:, :3], points_3d=p3[:3], cov=ct[:, :3]),          # 3 keypoints
           dict(keypoints=torch.zeros(2, 33, 2, device=DEV), points_3d=torch.zeros(33, 3, device=DEV),
                cov=torch.eye(2, device=DEV).expand(2, 33, 2, 2)),               # 33 keypoints
           dict(keypoints=kpt, points_3d=p3[:5], cov=ct),
           dict(keypoints=kpt, points_3d=p3, cov=ct[..., 0]),
           dict(keypoints=kpt, points_3d=p3, weights_2d=wts[..., :2]),
           dict(keypoints=kpt.cpu(), points_3d=p3, cov=ct),                      # another device
           dict(keypoints=kpt, points_3d=p3.cpu(), cov=ct),
           dict(keypoints=kpt.long(), points_3d=p3, cov=ct),                     # integer keypoints
           dict(keypoints=kp, points_3d=p3, cov=ct),                             # numpy
           dict(keypoints=kpt, points_3d=p3, cov=ct, keypoint_weight=-1.0),
           dict(keypoints=kpt, points_3d=p3, cov=ct, keypoint_weight=float("inf")),
           dict(keypoints=kpt, points_3d=p3, cov=ct, keypoint_weight=float("nan"))]
    for kw in bad:
        with pytest.raises(ValueError):
            refine.refine_poses(mask, p, k, v, f, **ok, **kw)


# ------------------------------------------------------------------ pipeline
def _pipeline_setup(graph, refine_cfg=True, per_batch_k=False):
    from pvnet_b200.model_repository import Resnet18_8s
    from pvnet_b200.pipeline import PoseKeypointPipeline
    from tests.helpers import seeded_state_dict
    net = Resnet18_8s(18, 2)
    net.load_state_dict(seeded_state_dict(net, 3))
    net = net.to(DEV).eval()
    pts3d = np.random.default_rng(8).uniform(-0.06, 0.06, (9, 3)).astype(np.float32)
    K = rc.camera_for(96, 128, 300.0).astype(np.float64)
    cfg = dict(vertices=MESH[0], faces=MESH[1], near=rf.NEAR, far=rf.FAR, rounds=3) if refine_cfg else None
    pipe = PoseKeypointPipeline(net, round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64,
                                cov_min_hyp_num=128, points_3d=pts3d, camera_matrix=None if per_batch_k else K,
                                graph=graph, refine=cfg)
    return net, pipe, pts3d, K


def _host_batches(n=3, b=2, seed=4):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy(rng.integers(0, 256, (b, 96, 128, 3), dtype=np.uint8)).pin_memory() for _ in range(n)]


def _run(pipe, hosts):
    b = hosts[0].shape[0]
    kp = [torch.empty([b, 9, 2]).pin_memory() for _ in hosts]
    cov = [torch.empty([b, 9, 2, 2]).pin_memory() for _ in hosts]
    pose = [torch.empty([b, 3, 4], dtype=torch.float64).pin_memory() for _ in hosts]
    rv.reset_device_rng(DEV)
    pipe.run(hosts, out_host=kp, cov_host=cov, pose_host=pose)
    return kp, cov, pose


def test_pipeline_refines_its_own_outputs_eagerly_and_in_its_graph():
    hosts = _host_batches()
    net, eager, pts3d, K = _pipeline_setup(False)
    _, graphed, _, _ = _pipeline_setup(True)
    e = _run(eager, hosts)
    _run(graphed, hosts)                                          # the first run captures
    g = _run(graphed, hosts)                                      # pure replays
    for a, b_ in zip(e, g):
        for x, y in zip(a, b_):
            assert torch.equal(torch.nan_to_num(x), torch.nan_to_num(y))
    # step's poses are refine_poses on the same step's mask, PnP poses, keypoints and covariances
    p3, kd = t(pts3d), t(K)
    v, f = device_mesh()
    with torch.no_grad():
        for x in hosts:
            x = x.to(DEV)
            kp, cov, pose = eager.step(x)
            _, mask = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, mean=eager.mean, std=eager.std,
                                         pixel_major=True)
            pnp = eu.uncertainty_pnp_batched(kp, p3, K, cov=cov)
            want = refine.refine_poses(mask, pnp, kd, v, f, rf.NEAR, rf.FAR, rounds=3, keypoints=kp, points_3d=p3,
                                       cov=cov)
            assert torch.equal(torch.nan_to_num(pose), torch.nan_to_num(want))
            # per-batch cameras reach the refinement too
            ks = t(np.stack([K, K * np.array([[1.05], [1.0], [1.0]])]))
            kp2, cov2, pose2 = eager.step(x, camera_matrix=ks)
            pnp2 = eu.uncertainty_pnp_batched(kp2, p3, ks, cov=cov2)
            want2 = refine.refine_poses(mask, pnp2, ks, v, f, rf.NEAR, rf.FAR, rounds=3, keypoints=kp2, points_3d=p3,
                                        cov=cov2)
            assert torch.equal(torch.nan_to_num(pose2), torch.nan_to_num(want2))


def test_pipeline_without_refine_is_unchanged():
    hosts = _host_batches(n=2, seed=5)
    _, pipe, pts3d, K = _pipeline_setup(False, refine_cfg=False)
    kp, cov, pose = _run(pipe, hosts)
    for i in range(len(hosts)):
        want = eu.uncertainty_pnp_batched(kp[i].to(DEV), pts3d, K, cov=cov[i].to(DEV)).cpu()
        assert torch.equal(torch.nan_to_num(pose[i]), torch.nan_to_num(want))


def test_pipeline_refine_arguments():
    from pvnet_b200.pipeline import PoseKeypointPipeline
    cfg = dict(vertices=MESH[0], faces=MESH[1], near=rf.NEAR, far=rf.FAR)
    with pytest.raises(ValueError):
        PoseKeypointPipeline(None, with_covariance=False, points_3d=PTS, refine=cfg)
    with pytest.raises(ValueError):
        PoseKeypointPipeline(None, with_covariance=True, refine=cfg)
    with pytest.raises(ValueError):
        PoseKeypointPipeline(None, with_covariance=True, points_3d=PTS, refine=dict(cfg, lamda=1.0))
    with pytest.raises(ValueError):
        PoseKeypointPipeline(None, with_covariance=True, points_3d=PTS, refine=dict(vertices=MESH[0]))
