"""GPU: `pvnet_b200.refine.refine_poses` (csrc/refine.cu) against oracle/refine_oracle.py on the same inputs -- the
boundary sets, back-projection and pairs bit for bit, the normal equations to 1e-12, every round's pose to 1e-9 --
and end to end: convergence on a known answer, batch independence, status bits, no host synchronisation, graph
replay and argument errors."""
import numpy as np
import pytest
import torch

from oracle import refine_oracle as rfo
from pvnet_b200 import refine
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MESH = rf.tool_mesh()


def t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def device_mesh():
    return t(MESH[0]), t(MESH[1])


def scene(b, h, w, seed, per_image_k, f=None):
    """True poses, starts 3 degrees and 1 cm away, K ([3,3] or [b,3,3] float32) and the truth's coverage masks."""
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
    return Pt, P0, K, (depth > 0).to(torch.uint8)


def proj_error(P, Pt, K):
    v = MESH[0].astype(np.float64)
    a, b = np.stack(rfo.project(v, P, K), -1), np.stack(rfo.project(v, Pt, K), -1)
    return float(np.linalg.norm(a - b, axis=1).mean())


def kof(K, i):
    return K if K.ndim == 2 else K[i]


@pytest.mark.parametrize("per_image_k", [False, True])
def test_first_round_stages_match_the_oracle(per_image_k):
    b, h, w, mp = 4, 96, 128, 200                    # max_points below the boundary counts: the stride rule runs
    Pt, P0, K, mask = scene(b, h, w, 11 + per_image_k, per_image_k)
    v, f = device_mesh()
    _, info, tr = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, rounds=1, max_points=mp,
                                      return_info=True, trace=True)
    tr = {k: x.cpu().numpy() for k, x in tr.items()}
    m = mask.cpu().numpy()
    for i in range(b):
        orec = []
        rfo.refine_image(m[i], P0[i], kof(K, i), *MESH, rf.NEAR, rf.FAR, rounds=1, max_points=mp, trace=orec)
        o = orec[0]
        ns, nc = tr["counts"][i]
        assert ns == len(o["sil"]) and nc == len(o["con"]) and ns > 0 and nc > 0
        assert np.array_equal(tr["sil_idx"][i, :ns], o["sil"])
        assert np.array_equal(tr["con_idx"][i, :nc], o["con"])
        assert np.array_equal(tr["sil_obj"][i, :ns], o["X"])                    # bit for bit
        assert np.array_equal(tr["pair_idx"][i, :ns], o["pair"])
        A, g = o["normal_eq"][0]
        ne = tr["normal_eq"][i]
        Ad = np.zeros((6, 6))
        Ad[np.triu_indices(6)] = ne[:21]
        Ad = Ad + np.triu(Ad, 1).T
        assert np.abs(Ad - A).max() <= 1e-12 * np.abs(A).max()
        assert np.abs(ne[21:] - g).max() <= 1e-12 * np.abs(g).max()


def test_every_rounds_pose_matches_the_oracle():
    b, h, w, R = 3, 96, 128, 5
    Pt, P0, K, mask = scene(b, h, w, 21, True)
    v, f = device_mesh()
    m = mask.cpu().numpy()
    for k in range(R + 1):
        out, info = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, rounds=k, return_info=True)
        out = out.cpu().numpy()
        for i in range(b):
            P, oi = rfo.refine_image(m[i], P0[i], K[i], *MESH, rf.NEAR, rf.FAR, rounds=k)
            assert np.abs(out[i] - P).max() <= 1e-9, (k, i)
            assert int(info["status"][i]) == oi["status"] and int(info["pairs"][i]) == oi["pairs"]
            for key in ("dist_before", "dist_after"):
                assert abs(float(info[key][i]) - oi[key]) <= 1e-12 * max(1.0, abs(oi[key])), (k, i, key)


@pytest.mark.parametrize("per_image_k", [False, True])
def test_batch_of_16_converges_and_never_ends_farther(per_image_k):
    b, h, w = 16, 480, 640
    Pt, P0, K, mask = scene(b, h, w, 31 + per_image_k, per_image_k, f=600.0)
    v, f = device_mesh()
    out, info = refine.refine_poses(mask, t(P0, torch.float32), t(K), v, f, rf.NEAR, rf.FAR, return_info=True)
    out = out.cpu().numpy()
    st = info["status"].cpu().numpy()
    d0, d1 = info["dist_before"].cpu().numpy(), info["dist_after"].cpu().numpy()
    assert (st & ~refine.REJECTED == 0).all(), st
    assert (d1 <= d0).all() and (d1 < d0).all()
    P0f = P0.astype(np.float32).astype(np.float64)                                  # the input the call received
    before = [proj_error(P0f[i], Pt[i], kof(K, i)) for i in range(b)]
    after = [proj_error(out[i], Pt[i], kof(K, i)) for i in range(b)]
    assert np.mean(after) < 0.5 * np.mean(before), (before, after)
    assert sum(a < bb for a, bb in zip(after, before)) >= b - 1, (before, after)
    # image i of the batch is the batch-of-one call on it, bit for bit
    for i in (0, 7, 15):
        one = refine.refine_poses(mask[i:i + 1], t(P0[i:i + 1], torch.float32), t(kof(K, i)), v, f, rf.NEAR, rf.FAR)
        assert torch.equal(one[0].cpu(), torch.from_numpy(out[i]))


def test_degenerate_images_set_their_bits_and_leave_the_others_alone():
    b, h, w = 4, 96, 128
    Pt, P0, K, mask = scene(b, h, w, 41, True)
    v, f = device_mesh()
    mask = mask.clone()
    mask[1] = 0                                                                 # empty mask
    mask[2] = 0
    mask[2, :8, :8] = 1                                                         # a mask far from the render
    P0 = P0.copy()
    P0[3, 2, 3] = -1.0                                                          # the render covers nothing
    out, info = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, gate=10.0, return_info=True)
    st = info["status"].cpu().tolist()
    assert st[1] == refine.NO_CONTOUR and st[2] == refine.FEW_PAIRS and st[3] == refine.NO_SILHOUETTE
    assert torch.equal(out[1:].cpu(), torch.from_numpy(P0[1:]))
    one = refine.refine_poses(mask[:1], t(P0[:1]), t(K[:1]), v, f, rf.NEAR, rf.FAR, gate=10.0)
    assert torch.equal(one[0], out[0])
    zero, info0 = refine.refine_poses(mask, t(P0), t(K), v, f, rf.NEAR, rf.FAR, gate=10.0, rounds=0,
                                      return_info=True)
    assert torch.equal(zero.cpu(), torch.from_numpy(P0))
    assert info0["status"].cpu().tolist()[1:] == st[1:]
    assert info0["status"][0] == 0 and info0["dist_before"][0] == info0["dist_after"][0]


def test_no_host_synchronisation_and_run_to_run_identical():
    Pt, P0, K, mask = scene(4, 96, 128, 51, True)
    v, f = device_mesh()
    p, k = t(P0), t(K)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a, ia = refine.refine_poses(mask, p, k, v, f, rf.NEAR, rf.FAR, return_info=True)
        b_, ib = refine.refine_poses(mask, p, k, v, f, rf.NEAR, rf.FAR, return_info=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a, b_) and all(torch.equal(ia[x], ib[x]) for x in ("status", "pairs"))


def test_graph_replay_with_new_masks_and_poses_gives_the_eager_result():
    b, h, w = 4, 96, 128
    PtA, P0A, K, maskA = scene(b, h, w, 61, True)
    _, P0B, _, _ = scene(b, h, w, 62, True)
    vB = render_mesh(*device_mesh(), t(K), t(rf.perturb(P0B, np.random.default_rng(1), 1.0, 0.003), torch.float32),
                     h, w, rf.NEAR, rf.FAR)
    maskB = (vB > 0).to(torch.uint8)
    v, f = device_mesh()
    sm, sp, sk = maskA.clone(), t(P0A), t(K)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        refine.refine_poses(sm, sp, sk, v, f, rf.NEAR, rf.FAR, rounds=4)     # warm-up
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out, info = refine.refine_poses(sm, sp, sk, v, f, rf.NEAR, rf.FAR, rounds=4, return_info=True)
    for mk, P in ((maskA, P0A), (maskB, P0B)):
        sm.copy_(mk)
        sp.copy_(t(P))
        g.replay()
        eager, ie = refine.refine_poses(mk, t(P), sk, v, f, rf.NEAR, rf.FAR, rounds=4, return_info=True)
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and torch.equal(info["status"], ie["status"])


def test_bad_arguments_raise():
    Pt, P0, K, mask = scene(2, 32, 40, 71, False)
    v, f = device_mesh()
    p, k = t(P0), t(K)
    ok = dict(near=rf.NEAR, far=rf.FAR)
    refine.refine_poses(mask, p, k, v, f, **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask[:1], p, k, v, f, **ok)                          # batch mismatch
    with pytest.raises(ValueError):
        refine.refine_poses(mask.float(), p, k, v, f, **ok)                      # float mask
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p.half(), k, v, f, **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p[:, :, :3], k, v, f, **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p, k[None].expand(3, 3, 3), v, f, **ok)        # 3 cameras for 2 images
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p, k, v[:, :2], f, **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p, k, v, f.float(), **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p, k, v, f, near=1.0, far=0.5)
    for bad in (dict(rounds=-1), dict(gate=0.0), dict(gate=float("inf")), dict(max_points=0)):
        with pytest.raises(ValueError):
            refine.refine_poses(mask, p, k, v, f, **ok, **bad)
    with pytest.raises(RuntimeError):
        refine.refine_poses(mask.cpu(), p, k, v, f, **ok)
    with pytest.raises(ValueError):
        refine.refine_poses(mask, p, k.cpu().numpy(), v, f, **ok)
    bool_mask = refine.refine_poses(mask.bool(), p, k, v, f, **ok)
    int_mask = refine.refine_poses(mask.long() * 3, p, k, v, f, **ok)
    assert torch.equal(bool_mask, refine.refine_poses(mask, p, k, v, f, **ok)) and torch.equal(bool_mask, int_mask)
