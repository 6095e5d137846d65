"""GPU: depth-anchored refinement (`refine_poses_depth`, `pvnet_refine_poses_depth`, DESIGN.md §28) against
oracle/refine_depth_oracle.py -- the first round's pairs, X, Y and n bit for bit, the normal equations to 1e-12,
every round's pose to 1e-9 and the same accept / undo decisions -- uint16 input, degenerate images, batch
independence, no host synchronisation, graph replay, argument errors and `PoseKeypointPipeline(refine=dict(depth=))`."""
import numpy as np
import pytest
import torch

from oracle import refine_depth_oracle as rdo
from pvnet_b200 import ransac_voting_gpu as rv
from pvnet_b200 import refine
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MESH = rf.tool_mesh()
GATE = rdc.GATE


def t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def device_mesh():
    return t(MESH[0]), t(MESH[1])


def kof(K, i):
    return K if K.ndim == 2 else K[i]


def scene(b, h, w, seed, per_image_k, f=None):
    """True poses, starts 3 degrees and 1 cm away, K, and the observed depth and mask: the truth's render and its
    coverage, with the variants of tests/refine_depth_cases.py in turn (clean, 1 mm noise, a block without readings,
    an occluder with the mask cut out)."""
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
    depth = render_mesh(*device_mesh(), t(K), t(Pt, torch.float32), h, w, rf.NEAR, rf.FAR).cpu().numpy()
    mask = depth > 0
    obs = depth.copy()
    for i in range(b):
        rows, cols = np.nonzero(mask[i])
        if not len(rows):
            continue
        r0, c0 = int(rows.mean()), int(cols.mean())
        if i % 4 == 1:
            obs[i] = rdc.noisy(depth[i], 1e-3, np.random.default_rng(seed * 100 + i))
        elif i % 4 == 2:
            obs[i] = rdc.holed(depth[i], r0 - h // 40, c0 - w // 40, max(2, h // 20))
        elif i % 4 == 3:
            obs[i], mask[i] = rdc.occluded(depth[i], mask[i], r0, c0, max(2, h // 16))
    return Pt, P0, K, mask.astype(np.uint8), obs


def oracle_round_results(tr, P):
    """The oracle's result with rounds = k, for every k, from one trace of the full run."""
    return lambda k: tr[k]["pose"] if k < len(tr) - 1 else P


@pytest.mark.parametrize("per_image_k", [False, True])
def test_full_size_rounds_match_the_oracle(per_image_k):
    b, h, w, R = 16, 480, 640, 8
    Pt, P0, K, mask, obs = scene(b, h, w, 3 + per_image_k, per_image_k, f=600.0)
    v, f = device_mesh()
    args = (t(mask), t(obs), t(P0), t(K), v, f, rf.NEAR, rf.FAR, GATE)
    out, info, tr = refine.refine_poses_depth(*args, rounds=R, return_info=True, trace=True)
    per_k = [refine.refine_poses_depth(*args, rounds=k).cpu().numpy() for k in range(R)] + [out.cpu().numpy()]
    info = {x: y.cpu().numpy() for x, y in info.items()}
    tr = {x: y.cpu().numpy() for x, y in tr.items()}
    render = rf.device_depth(DEV)
    statuses = set()
    for i in range(b):
        otr = []
        P, oi = rdo.refine_image(mask[i], obs[i], P0[i], kof(K, i), *MESH, rf.NEAR, rf.FAR, GATE, rounds=R, trace=otr,
                                 render=render)
        o = otr[0]
        m = len(o["idx"])
        assert tr["counts"][i].tolist() == [m, o["count"], o["mask_pixels"], o["covered_pixels"]], i
        assert np.array_equal(tr["pair_idx"][i, :m], o["idx"]), i
        for key in ("X", "Y", "n"):
            assert np.array_equal(tr[key][i, :m].view(np.uint64), o[key].view(np.uint64)), (i, key)
        A, g = o["normal_eq"][0]
        ne = tr["normal_eq"][i]
        Ad = np.zeros((6, 6))
        Ad[np.triu_indices(6)] = ne[:21]
        Ad = Ad + np.triu(Ad, 1).T
        assert np.abs(Ad - A).max() <= 1e-12 * np.abs(A).max(), i
        assert np.abs(ne[21:] - g).max() <= 1e-12 * np.abs(g).max(), i
        at = oracle_round_results(otr, P)
        for k in range(R + 1):
            assert np.abs(per_k[k][i] - at(k)).max() <= 1e-9, (i, k)
        # the round's decision is the kernel's by construction while its pose is the oracle's bit for bit; a
        # converged round's pose agrees only to rounding, so there an undo may differ, when the two means it compares
        # are within rounding of each other
        st = int(info["status"][i])
        if st != oi["status"]:
            assert st ^ oi["status"] == refine.REJECTED and len(otr) == R + 1, i
            assert abs(otr[-1]["mean"] - otr[-2]["mean"]) <= 1e-9 * oi["dist_before"], i
        assert int(info["pairs"][i]) == oi["pairs"], i
        assert info["dist_before"][i] == oi["dist_before"], i
        assert abs(info["dist_after"][i] - oi["dist_after"]) <= 1e-9 * max(1.0, abs(oi["dist_after"])), i
        assert info["dist_after"][i] <= info["dist_before"][i]
        statuses.add(oi["status"])
    assert statuses <= {0, refine.REJECTED}, statuses


def test_uint16_equals_float32_built_from_it():
    b, h, w = 4, 120, 160
    Pt, P0, K, mask, obs = scene(b, h, w, 5, True, f=300.0)
    d16 = rdc.as_u16_mm(obs)
    scale = 1e-3
    d32 = d16.astype(np.float32) * np.float32(scale)
    v, f = device_mesh()
    args = (t(mask),)
    rest = (t(P0), t(K), v, f, rf.NEAR, rf.FAR, GATE)
    a, ia, ta = refine.refine_poses_depth(*args, t(d16), *rest, depth_scale=scale, return_info=True, trace=True)
    b_, ib, tb = refine.refine_poses_depth(*args, t(d32), *rest, return_info=True, trace=True)
    assert torch.equal(a, b_)
    assert all(torch.equal(torch.nan_to_num(ia[x]), torch.nan_to_num(ib[x])) for x in ia)
    assert torch.equal(ta["counts"], tb["counts"]) and torch.equal(ta["normal_eq"], tb["normal_eq"])
    for i, m in enumerate(ta["counts"][:, 0].tolist()):                        # entries past the count are not written
        assert all(torch.equal(ta[x][i, :m], tb[x][i, :m]) for x in ("pair_idx", "X", "Y", "n")), i
    assert (ia["pairs"] > 0).all()


def test_degenerate_images_keep_their_input_and_leave_the_others_alone():
    b, h, w = 6, 96, 128
    Pt, P0, K, mask, obs = scene(b, h, w, 7, True, f=150.0)
    v, f = device_mesh()
    mask, obs, P0 = mask.copy(), obs.copy(), P0.copy()
    mask[1] = 0                                                                 # empty mask
    obs[2] = 0                                                                  # no readings
    P0[3, 2, 3] = -1.0                                                          # the render covers nothing
    obs[4, :, :] = np.nan                                                       # readings that are not numbers
    out, info = refine.refine_poses_depth(t(mask), t(obs), t(P0), t(K), v, f, rf.NEAR, rf.FAR, GATE,
                                          return_info=True)
    st = info["status"].cpu().tolist()
    assert st[1] == refine.NO_CONTOUR and st[2] == refine.FEW_PAIRS and st[3] == refine.NO_SILHOUETTE
    assert st[4] == refine.FEW_PAIRS
    assert st[0] & ~refine.REJECTED == 0 and st[5] & ~refine.REJECTED == 0
    assert torch.equal(out[1:5].cpu(), torch.from_numpy(P0[1:5]))
    assert torch.isnan(info["dist_before"][1:5]).all()
    for i in range(b):
        one = refine.refine_poses_depth(t(mask[i:i + 1]), t(obs[i:i + 1]), t(P0[i:i + 1]), t(K[i]), v, f, rf.NEAR,
                                        rf.FAR, GATE)
        assert torch.equal(one[0], out[i]), i
    zero = refine.refine_poses_depth(t(mask), t(obs), t(P0), t(K), v, f, rf.NEAR, rf.FAR, GATE, rounds=0)
    assert torch.equal(zero.cpu(), torch.from_numpy(P0))


def test_no_host_synchronisation_run_to_run_identical_and_graph_replay():
    b, h, w = 4, 96, 128
    _, P0A, K, maskA, obsA = scene(b, h, w, 9, True)
    _, P0B, _, maskB, obsB = scene(b, h, w, 10, True)
    v, f = device_mesh()
    k = t(K)
    m, d, p = t(maskA), t(obsA), t(P0A)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a, ia = refine.refine_poses_depth(m, d, p, k, v, f, rf.NEAR, rf.FAR, GATE, return_info=True)
        b_, ib = refine.refine_poses_depth(m, d, p, k, v, f, rf.NEAR, rf.FAR, GATE, return_info=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a, b_) and all(torch.equal(torch.nan_to_num(ia[x]), torch.nan_to_num(ib[x])) for x in ia)
    sm, sd, sp = m.clone(), d.clone(), p.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        refine.refine_poses_depth(sm, sd, sp, k, v, f, rf.NEAR, rf.FAR, GATE, rounds=4)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, info = refine.refine_poses_depth(sm, sd, sp, k, v, f, rf.NEAR, rf.FAR, GATE, rounds=4, return_info=True)
    for mk, ob, P in ((maskA, obsA, P0A), (maskB, obsB, P0B)):
        sm.copy_(t(mk))
        sd.copy_(t(ob))
        sp.copy_(t(P))
        g.replay()
        eager, ie = refine.refine_poses_depth(t(mk), t(ob), t(P), k, v, f, rf.NEAR, rf.FAR, GATE, rounds=4,
                                              return_info=True)
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
        assert all(torch.equal(torch.nan_to_num(info[x]), torch.nan_to_num(ie[x])) for x in ie)


def test_bad_arguments_raise():
    _, P0, K, mask, obs = scene(2, 32, 40, 11, False)
    v, f = device_mesh()
    m, d, p, k = t(mask), t(obs), t(P0), t(K)
    ok = dict(near=rf.NEAR, far=rf.FAR, gate=GATE)
    refine.refine_poses_depth(m, d, p, k, v, f, **ok)
    bad = [((m, d[:1], p, k, v, f), ok),                                        # batch mismatch
           ((m, d[:, :, :-1], p, k, v, f), ok),                                 # size mismatch
           ((m, d.double(), p, k, v, f), ok),                                   # float64 depth
           ((m, d.to(torch.int32), p, k, v, f), ok),                            # int32 depth
           ((m, d.cpu(), p, k, v, f), ok),                                      # another device
           ((m, obs, p, k, v, f), ok),                                          # numpy
           ((m, d, p, k, v, f), dict(ok, gate=0.0)),
           ((m, d, p, k, v, f), dict(ok, gate=float("inf"))),
           ((m, d, p, k, v, f), dict(ok, gate=float("nan"))),
           ((m, d, p, k, v, f), dict(ok, rounds=-1)),
           ((m, d, p, k, v, f), dict(ok, max_points=0)),
           ((m, d, p, k, v, f), dict(ok, depth_scale=0.0)),
           ((m, d, p, k, v, f), dict(ok, depth_scale=float("inf"))),
           ((m.float(), d, p, k, v, f), ok),                                    # float mask
           ((m, d, p, k, v, f), dict(ok, near=1.0, far=0.5))]
    for args, kw in bad:
        with pytest.raises(ValueError):
            refine.refine_poses_depth(*args, **kw)
    with pytest.raises(TypeError):
        refine.refine_poses_depth(m, d, p, k, v, f, rf.NEAR, rf.FAR)          # no gate


# ------------------------------------------------------------------ pipeline
def _pipeline(graph, per_batch_k=False, depth_cfg=True):
    from pvnet_b200.model_repository import Resnet18_8s
    from pvnet_b200.pipeline import PoseKeypointPipeline
    from tests.helpers import seeded_state_dict
    net = Resnet18_8s(18, 2)
    net.load_state_dict(seeded_state_dict(net, 3))
    net = net.to(DEV).eval()
    pts3d = np.random.default_rng(8).uniform(-0.06, 0.06, (9, 3)).astype(np.float32)
    K = rc.camera_for(96, 128, 300.0).astype(np.float64)
    cfg = dict(vertices=MESH[0], faces=MESH[1], near=rf.NEAR, far=rf.FAR, rounds=2)
    if depth_cfg:
        cfg["depth"] = dict(gate=0.2, rounds=3)
    pipe = PoseKeypointPipeline(net, round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64,
                                cov_min_hyp_num=128, points_3d=pts3d, camera_matrix=None if per_batch_k else K,
                                graph=graph, refine=cfg)
    return net, pipe, pts3d, K


def _hosts(n=3, b=2, seed=4):
    rng = np.random.default_rng(seed)
    imgs = [torch.from_numpy(rng.integers(0, 256, (b, 96, 128, 3), dtype=np.uint8)).pin_memory() for _ in range(n)]
    deps = [torch.from_numpy(rng.uniform(0.3, 0.6, (b, 96, 128)).astype(np.float32)).pin_memory() for _ in range(n)]
    return imgs, deps


def _run(pipe, imgs, deps, cams=None):
    b = imgs[0].shape[0]
    pose = [torch.empty([b, 3, 4], dtype=torch.float64).pin_memory() for _ in imgs]
    rv.reset_device_rng(DEV)
    pipe.run(imgs, pose_host=pose, depths=deps, camera_matrices=cams)
    return pose


@pytest.mark.parametrize("per_batch_k", [False, True])
def test_pipeline_refines_against_depth_eagerly_and_in_its_graph(per_batch_k):
    imgs, deps = _hosts()
    net, eager, pts3d, K = _pipeline(False, per_batch_k)
    _, graphed, _, _ = _pipeline(True, per_batch_k)
    cams = None
    if per_batch_k:
        cams = [torch.from_numpy(np.stack([K, K * np.array([[1.0 + 0.02 * i], [1.0], [1.0]])])).pin_memory()
                for i in range(len(imgs))]
    e = _run(eager, imgs, deps, cams)
    _run(graphed, imgs, deps, cams)                                # the first run captures
    g = _run(graphed, imgs, deps, cams)                            # pure replays
    for x, y in zip(e, g):
        assert torch.equal(torch.nan_to_num(x), torch.nan_to_num(y))
    # step's poses are refine_poses_depth on the same step's mask and keypoint-anchored poses
    _, plain, _, _ = _pipeline(False, per_batch_k, depth_cfg=False)
    v, f = device_mesh()
    with torch.no_grad():
        for i, x in enumerate(imgs):
            x, dd = x.to(DEV), deps[i].to(DEV)
            k = t(K) if cams is None else cams[i].to(DEV)
            kcall = None if cams is None else k
            rv.reset_device_rng(DEV)
            _, _, pose = eager.step(x, kcall, dd)
            rv.reset_device_rng(DEV)
            _, _, anchored = plain.step(x, kcall)
            _, mask = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, mean=eager.mean, std=eager.std,
                                         pixel_major=True)
            want = refine.refine_poses_depth(mask, dd, anchored, k, v, f, rf.NEAR, rf.FAR, gate=0.2, rounds=3)
            assert torch.equal(torch.nan_to_num(pose), torch.nan_to_num(want)), i


def test_pipeline_depth_arguments():
    from pvnet_b200.pipeline import PoseKeypointPipeline
    pts = np.zeros((9, 3), np.float32)
    cfg = dict(vertices=MESH[0], faces=MESH[1], near=rf.NEAR, far=rf.FAR)
    for d in (dict(), dict(rounds=2), dict(gate=0.1, gamma=1.0)):
        with pytest.raises(ValueError):
            PoseKeypointPipeline(None, with_covariance=True, points_3d=pts, refine=dict(cfg, depth=d))
    _, with_depth, _, _ = _pipeline(False)
    _, without, _, _ = _pipeline(False, depth_cfg=False)
    x = torch.zeros(2, 96, 128, 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        with_depth.step(x)                                                     # depth missing
    with pytest.raises(ValueError):
        without.step(x, depth=torch.zeros(2, 96, 128, device=DEV))             # depth without refine['depth']
    imgs, deps = _hosts(n=1)
    with pytest.raises(ValueError):
        with_depth.run(imgs)
    with pytest.raises(ValueError):
        without.run(imgs, depths=deps)
