"""GPU: `refine_poses_instances` (DESIGN.md §30) against `refine_poses` and oracle/refine_instances_oracle.py.

- L = 1 on a {0,1} map is bit for bit `refine_poses` on that mask, with and without keypoints, for uint8, int32 and
  int64 labels.
- A scene of three overlapping lumpy meshes, composited by depth into a label map: the first round's silhouette,
  contour and pair sets match the oracle bit for bit, the first step's sums to 1e-12, every pose to 1e-9, and the
  absent row returns its input with status 32.
- The pose errors of the start, of `refine_poses` on `labels == j+1` and of `refine_poses_instances` are printed."""
import numpy as np
import pytest
import torch

from oracle import refine_instances_oracle as rio
from pvnet_b200 import refine as rfn
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 240, 320
MESH = rf.lumpy_mesh()
K = np.array([[572.4114, 0.0, 160.0], [0.0, 573.57043, 120.0], [0.0, 0.0, 1.0]], np.float32)


def t(a, dt=None):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV, dtype=dt)


def _scene(xs=(-0.08, 0.0, 0.08), zs=(0.5, 0.52, 0.54), seed=0):
    """Instances at (x, 0, z) with random rotations, composited by depth: -> labels int64 [H,W], true poses [n,3,4]."""
    rng = np.random.default_rng(seed)
    P = np.zeros((len(xs), 3, 4))
    for i, (x, z) in enumerate(zip(xs, zs)):
        P[i, :, :3] = rf.axis_angle(rng.normal(size=3) * 0.3)
        P[i, :, 3] = (x, rng.uniform(-0.01, 0.01), z)
    d = render_mesh(t(MESH[0]), t(MESH[1]), t(K), t(P, torch.float32), H, W, rf.NEAR, rf.FAR).cpu().numpy()
    dd = np.where(d > 0, d, np.inf)
    lab = np.where(np.isfinite(dd).any(0), dd.argmin(0) + 1, 0).astype(np.int64)
    return lab, P


@pytest.mark.parametrize("ldtype", [torch.uint8, torch.int32, torch.int64])
@pytest.mark.parametrize("with_kp", [False, True])
def test_one_instance_equals_refine_poses(ldtype, with_kp):
    lab, P = _scene(xs=(0.0,), zs=(0.5,), seed=1)
    rng = np.random.default_rng(2)
    P0 = rf.perturb(P, rng)
    mask = t(lab[None] != 0, torch.uint8)
    kw = {}
    if with_kp:
        pts = MESH[0][::15][:9]
        kp = np.stack(rf.rfo.project(pts.astype(np.float64), P[0], K), -1) + rng.normal(0, 0.5, (9, 2))
        kw = dict(keypoints=t(kp[None], torch.float32), points_3d=t(pts, torch.float32),
                  weights_2d=t(np.tile([1.0, 0.0, 1.0], (1, 9, 1)), torch.float32))
    a, ia = rfn.refine_poses(mask, t(P0), t(K), t(MESH[0]), t(MESH[1]), rf.NEAR, rf.FAR, return_info=True, **kw)
    kwi = {k: (v[:, None] if k != "points_3d" else v) for k, v in kw.items()}
    b, ib = rfn.refine_poses_instances(t(lab[None]).to(ldtype), t(np.ones(1, np.int32)), t(P0[:, None]), t(K),
                                       t(MESH[0]), t(MESH[1]), rf.NEAR, rf.FAR, return_info=True, **kwi)
    assert torch.equal(a, b[:, 0])
    for k in ia:
        assert torch.equal(torch.nan_to_num(ia[k]), torch.nan_to_num(ib[k][:, 0])), k
    assert int(ia["pairs"][0]) > 100


def test_scene_matches_oracle_and_absent_row_passes_through():
    lab, P = _scene()
    rng = np.random.default_rng(3)
    P0 = np.concatenate([rf.perturb(P, rng, deg=2.0, dist=0.005), np.eye(3, 4)[None] * 7.0])[None]     # [1,4,3,4]
    num = np.array([3], np.int32)
    out, info, tr = rfn.refine_poses_instances(t(lab[None]), t(num), t(P0), t(K), t(MESH[0]), t(MESH[1]), rf.NEAR,
                                               rf.FAR, rounds=4, return_info=True, trace=True)
    traces = {}
    ref, rinfo = rio.refine(lab[None], num, P0, K, MESH[0], MESH[1], rf.NEAR, rf.FAR, rounds=4,
                            render=rf.device_depth(), traces=traces)
    out, st = out.cpu().numpy(), info["status"].cpu().numpy()
    assert np.array_equal(out[0, 3], P0[0, 3]) and st[0, 3] == rio.NO_INSTANCE
    assert np.array_equal(st, rinfo["status"]) and np.array_equal(info["pairs"].cpu().numpy(), rinfo["pairs"])
    np.testing.assert_allclose(out, ref, rtol=0, atol=1e-9)
    cnt = tr["counts"].cpu().numpy()
    for j in range(3):
        r0 = traces[(0, j)][0]
        ns, nc = len(r0["sil"]), len(r0["con"])
        assert (ns, nc) == tuple(cnt[j]) and ns > 100 and nc > 100
        assert np.array_equal(tr["sil_idx"][j, :ns].cpu().numpy(), r0["sil"])
        assert np.array_equal(tr["con_idx"][j, :nc].cpu().numpy(), r0["con"])
        assert np.array_equal(tr["pair_idx"][j, :ns].cpu().numpy(), r0["pair"])
        assert np.array_equal(tr["sil_obj"][j, :ns].cpu().numpy(), r0["X"])
        A, g = r0["normal_eq"][0]
        ne = tr["normal_eq"][j].cpu().numpy()
        want = np.concatenate([A[np.triu_indices(6)], g])
        np.testing.assert_allclose(ne, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
    # the rules bite in this scene: the touching instances lose contour and silhouette points
    full = [len(rf.rfo.boundary(lab == j + 1)) for j in range(3)]
    assert any(c < f for c, f in zip(cnt[:3, 1], full))


def test_accuracy_against_per_mask_refinement():
    """Report-only: mean rotation / translation error of the start, of refine_poses on labels == j+1 and of
    refine_poses_instances over seeded scenes of three overlapping instances."""
    errs = {"start": [], "per_mask": [], "instances": []}
    for seed in range(6):
        lab, P = _scene(seed=10 + seed)
        rng = np.random.default_rng(100 + seed)
        P0 = rf.perturb(P, rng, deg=3.0, dist=0.01)
        a = rfn.refine_poses(t(np.stack([lab == j + 1 for j in range(3)]), torch.uint8), t(P0), t(K), t(MESH[0]),
                             t(MESH[1]), rf.NEAR, rf.FAR).cpu().numpy()
        b = rfn.refine_poses_instances(t(lab[None]), t(np.array([3], np.int32)), t(P0[None]), t(K), t(MESH[0]),
                                       t(MESH[1]), rf.NEAR, rf.FAR)[0].cpu().numpy()
        for name, Q in (("start", P0), ("per_mask", a), ("instances", b)):
            errs[name] += [rf.pose_error(Q[j], P[j]) for j in range(3)]
    for name, e in errs.items():
        e = np.array(e, np.float64)
        print(f"{name}: rotation {e[:, 0].mean():.3f} deg, translation {1e3 * e[:, 1].mean():.2f} mm")
    assert np.isfinite(np.array(errs["instances"], np.float64)).all()
