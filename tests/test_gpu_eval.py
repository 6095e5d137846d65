"""GPU: pose evaluation on the device (pvnet_b200/evaluation.py, pvnet_b200/csrc/eval.cu).
  - pvnet_find_nearest_point_idx: bit-identical indices to the C oracle and to the reference's own kernel
    (stored in tests/golden/ref_nn.npz by tests/golden/make_golden_ref_nn.py), 2-D and 3-D;
  - pose_metrics against the fp64 oracle (oracle/eval_oracle.py) on 64 random pose pairs;
  - a CUDA-graph capture of Evaluator.evaluate_batch equals the eager run;
  - pnp / uncertainty_pnp_v2 on the PnP fixtures; Evaluator's per-image methods against a numpy restatement."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import eval_oracle as eo
from oracle import pnp_oracle as pno
from pvnet_b200 import evaluation as ev
from tests.helpers import RefGolden, same_as_stored

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_gold = RefGolden("ref_nn.npz")


def _nn_case(name):
    """Deterministic inputs [b,pn1,dim], [b,pn2,dim] of every search case."""
    rng = np.random.default_rng(sum(map(ord, name)))
    spec = {"3d_small": (3, 1000, 777, 3), "3d_tile_edge": (2, 513, 1025, 3), "3d_32k": (1, 32768, 32768, 3),
            "3d_dups": (2, 1500, 900, 3), "3d_nan_inf": (2, 1200, 700, 3),
            "2d_small": (3, 1000, 777, 2), "2d_20k": (2, 20000, 9000, 2), "2d_dups": (2, 1500, 900, 2),
            "2d_nan_inf": (2, 1200, 700, 2)}[name]
    b, pn1, pn2, dim = spec
    ref = rng.normal(size=(b, pn1, dim)).astype(np.float32)
    que = rng.normal(size=(b, pn2, dim)).astype(np.float32)
    if name.endswith("dups"):
        ref[:, pn1 // 2:] = ref[:, :pn1 - pn1 // 2]                       # every point (at least) twice
        que[:, :300] = ref[:, rng.integers(0, pn1, 300)]                   # queries exactly on duplicated points
        ref = np.round(ref * 8) / 8                                        # coarse grid: many equal distances
        que = np.round(que * 8) / 8
    if name.endswith("nan_inf"):
        for a in (ref, que):
            k = rng.integers(0, a.shape[1], (b, 40))
            for bi in range(b):
                a[bi, k[bi, :20], rng.integers(0, dim)] = np.nan
                a[bi, k[bi, 20:], rng.integers(0, dim)] = np.inf * rng.choice([-1, 1])
        ref[1, :] = np.nan                                                  # an image with no finite reference
        ref[1, 5] = 0.0
    return ref, que


NN_CASES = ["3d_small", "3d_tile_edge", "3d_32k", "3d_dups", "3d_nan_inf", "2d_small", "2d_20k", "2d_dups", "2d_nan_inf"]


@pytest.mark.parametrize("name", NN_CASES)
def test_nearest_point_idx_bit_exact(name):
    ref, que = _nn_case(name)
    got = ev.find_nearest_point_idx(torch.from_numpy(ref).to(DEV), torch.from_numpy(que).to(DEV)).cpu().numpy()
    want = eo.find_nearest_point_idx(ref, que)
    assert np.array_equal(got, want), (name, int((got != want).sum()))
    stored = _gold.get(name, lambda: {"idxs": eo.ref_find_nearest_point_idx(ref, que)}, exact=["idxs"])
    assert same_as_stored(got, stored["idxs"]), name
    # the reference call shape: numpy [pn,dim] in, numpy int32 [pn2] out
    one = ev.find_nearest_point_idx(ref[0], que[0])
    assert isinstance(one, np.ndarray) and one.dtype == np.int32 and np.array_equal(one, want[0])


def teardown_module(module):
    _gold.save()


def _random_pose(rng, scale):
    R = pno.rodrigues(rng.normal(0, 1.0, 3))
    t = np.array([rng.uniform(-.1, .1), rng.uniform(-.1, .1), rng.uniform(0.5, 1.2)])
    dR = pno.rodrigues(rng.normal(0, scale, 3))
    dt = rng.normal(0, scale * 0.3, 3)
    return np.concatenate([R, t[:, None]], 1), np.concatenate([dR @ R, (t + dt)[:, None]], 1)


def _pose_batch(b=64, seed=5):
    rng = np.random.default_rng(seed)
    gt, pred = zip(*[_random_pose(rng, s) for s in np.geomspace(1e-3, 0.3, b)])
    Ks = np.stack([np.array([[rng.uniform(500, 600), rng.uniform(-5, 5), rng.uniform(300, 340)],
                             [0, rng.uniform(500, 600), rng.uniform(220, 260)], [0, 0, 1]]) for _ in range(b)])
    model = rng.uniform(-0.06, 0.06, (2999, 3)).astype(np.float32)
    return np.stack(pred), np.stack(gt), model, Ks


@pytest.mark.parametrize("symmetric,sym_proj,per_image_K", [(False, False, False), (True, False, False),
                                                            (False, True, True), (True, True, True)])
def test_pose_metrics_match_oracle(symmetric, sym_proj, per_image_K):
    pred, gt, model, Ks = _pose_batch()
    K = torch.from_numpy(Ks).to(DEV) if per_image_K else Ks[0]
    got = ev.pose_metrics(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV), torch.from_numpy(model).to(DEV),
                          K, symmetric, sym_proj).cpu().numpy()
    want = np.stack([eo.pose_metrics_one(pred[i], gt[i], model, Ks[i] if per_image_K else Ks[0], symmetric,
                                         sym_proj)[0] for i in range(len(pred))])
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-300)
    assert (rel[:, :3] < 1e-12).all(), rel[:, :3].max()
    assert (np.abs(got[:, 3] - want[:, 3]) <= 1e-12 * np.maximum(want[:, 3], 1e-3)).all()
    diameter = 0.15
    for a, b in zip(eo.passes(got, diameter), eo.passes(want, diameter)):
        assert np.array_equal(a, b)
    assert 0 < eo.passes(want, diameter)[0].sum() < len(pred)                # both outcomes occur
    # the ADD-S / 2-D searches run on the same fp32 roundings: the public search gives the oracle's indices there
    for i in (0, 31, 63):
        P, G = eo.transform(pred[i], model), eo.transform(gt[i], model)
        if symmetric:
            idx = ev.find_nearest_point_idx(P.astype(np.float32), G.astype(np.float32))
            assert np.array_equal(idx, eo.pose_metrics_one(pred[i], gt[i], model, Ks[0], True)[1]["add"])
    # run to run: bit-identical
    again = ev.pose_metrics(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV),
                            torch.from_numpy(model).to(DEV), K, symmetric, sym_proj).cpu().numpy()
    assert np.array_equal(got, again)


class _ModelDB:
    def __init__(self, model, diameter):
        self.model, self.diameter = model, diameter

    def get_ply_model(self, class_type):
        return self.model

    def get_diameter(self, class_type):
        return self.diameter


class _Projector:
    def __init__(self, K):
        self.intrinsic_matrix = {"linemod": K, "blender": K}


def test_evaluate_batch_graph_capture_equals_eager():
    pred, gt, model, Ks = _pose_batch(16, seed=7)
    pp, pg, m = (torch.from_numpy(x).to(DEV) for x in (pred, gt, model))
    eager = ev.Evaluator(model_db=_ModelDB(model, 0.15), projector=_Projector(Ks[0]))
    for _ in range(4):
        out_eager = eager.evaluate_batch(pp, pg, m, 0.15, Ks[0], symmetric=True)
    graphed = ev.Evaluator(model_db=_ModelDB(model, 0.15), projector=_Projector(Ks[0]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graphed.evaluate_batch(pp, pg, m, 0.15, Ks[0], symmetric=True)          # warm-up, allocates the totals
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out_graph = graphed.evaluate_batch(pp, pg, m, 0.15, Ks[0], symmetric=True)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_graph, out_eager)
    assert torch.equal(graphed.batch_totals, eager.batch_totals)
    assert eager.batch_totals[0].item() == 64
    assert graphed.average_precision(verbose=False) == eager.average_precision(verbose=False)
    want = eo.passes(eo.pose_metrics(pred, gt, model, Ks[0], symmetric=True), 0.15)
    assert eager.average_precision(verbose=False) == tuple(float(np.mean(w)) for w in (want[1], want[0], want[2]))


def test_pnp_fixtures():
    z = np.load(os.path.join(GOLDEN, "pnp_cases.npz"))
    rt = ev.pnp(z["points_3d"], z["demo_iso_kp"], z["K"])
    assert isinstance(rt, np.ndarray) and rt.shape == (3, 4) and rt.dtype == np.float64
    assert np.abs(rt - z["demo_iso_pose"]).max() < 2e-6
    names = sorted(k[:-len("_cv2iter")] for k in z.files if k.endswith("_cv2iter"))
    assert names
    batch = ev.pnp(z["points_3d"], torch.from_numpy(np.stack([z[n + "_kp"] for n in names])).to(DEV), z["K"])
    assert batch.is_cuda and batch.dtype == torch.float64
    for i, n in enumerate(names):
        one = ev.pnp(z["points_3d"], z[n + "_kp"], z["K"])
        assert np.abs(one - z[n + "_cv2iter"]).max() < 1e-6, (n, np.abs(one - z[n + "_cv2iter"]).max())
        assert np.abs(batch[i].cpu().numpy() - one).max() < 1e-12
    with pytest.raises(ValueError):
        ev.pnp(z["points_3d"], z["demo_iso_kp"], z["K"], method=1)


def test_uncertainty_pnp_v2_matches_oracle_minimiser():
    z = np.load(os.path.join(GOLDEN, "pnp_cases.npz"))
    pts = z["points_3d"].astype(np.float32)
    for n in ("noisy_1", "noisy_4", "demo_aniso"):
        cov = z[n + "_cov"].astype(np.float64)
        lam = np.array([np.max(np.linalg.eigvals(c)).real for c in cov])
        w = np.where(cov[:, 0, 0] < 1e-5, 0.0, 1.0 / lam)
        want = pno.uncertainty_pnp(z[n + "_kp"], np.stack([w, 0 * w, w], 1).astype(np.float32), pts, z["K"])
        got = ev.uncertainty_pnp_v2(z[n + "_kp"], z[n + "_cov"], z["points_3d"], z["K"])
        assert np.abs(got - want).max() < 1e-8, n
        dev = ev.uncertainty_pnp_v2(torch.from_numpy(z[n + "_kp"][None]).to(DEV),
                                    torch.from_numpy(z[n + "_cov"][None]).to(DEV), pts, z["K"])
        assert np.abs(dev[0].cpu().numpy() - got).max() < 1e-12


def _numpy_metrics(pose_pred, pose_targets, model, K, diameter, sym):
    """The reference's formulas (evaluation_utils.py:75-141) in plain numpy, on the vertices in float64 as the
    kernel reads them (np.dot of a float32 model with a float64 pose can come back in float32)."""
    model = model.astype(np.float64)
    def proj(RT):
        p = np.matmul(np.matmul(model, RT[:, :3].T) + RT[:, 3:].T, K.T)
        return p[:, :2] / p[:, 2:]
    mp = np.dot(model, pose_pred[:, :3].T) + pose_pred[:, 3]
    mt = np.dot(model, pose_targets[:, :3].T) + pose_targets[:, 3]
    if sym:
        idx = eo.find_nearest_point_idx(mp.astype(np.float32), mt.astype(np.float32))
        add = np.mean(np.linalg.norm(mp[idx] - mt, 2, 1))
    else:
        add = np.mean(np.linalg.norm(mp - mt, axis=-1))
    pd = np.mean(np.linalg.norm(proj(pose_pred) - proj(pose_targets), axis=-1))
    td = np.linalg.norm(pose_pred[:, 3] - pose_targets[:, 3]) * 100
    tr = min(np.trace(np.dot(pose_pred[:, :3], pose_targets[:, :3].T)), 3)
    ang = np.rad2deg(np.arccos((tr - 1.) / 2.))
    return pd, add, td, ang


@pytest.mark.parametrize("class_type", ["cat", "glue"])
def test_evaluator_per_image_methods(monkeypatch, class_type):
    z = np.load(os.path.join(GOLDEN, "pnp_cases.npz"))
    pts3d = z["points_3d"]
    vt = types.ModuleType("lib.datasets.linemod_dataset")

    class VotingType:
        BB8 = 0

        @staticmethod
        def get_pts_3d(vote_type, class_type):
            assert vote_type == VotingType.BB8
            return pts3d
    vt.VotingType = VotingType
    monkeypatch.setitem(sys.modules, "lib.datasets", types.ModuleType("lib.datasets"))
    monkeypatch.setitem(sys.modules, "lib.datasets.linemod_dataset", vt)
    model = np.random.default_rng(2).uniform(-0.05, 0.05, (1234, 3)).astype(np.float32)
    diameter = 0.12
    e = ev.Evaluator(model_db=_ModelDB(model, diameter), projector=_Projector(z["K"]))
    names = ["demo_iso", "noisy_0", "noisy_1", "noisy_2", "noisy_5"]
    for n in names:
        e.evaluate(z[n + "_kp"], z[n + "_pose"], class_type, intri_type="linemod")
        e.evaluate_uncertainty(z[n + "_kp"], z[n + "_cov"], z[n + "_pose"], class_type, intri_type="linemod")
    assert len(e.uncertainty_pnp_cost) == len(names)
    k = 0
    for n in names:
        w = ev.covariance_to_weights(torch.from_numpy(z[n + "_cov"]).to(DEV)).cpu().numpy()
        for pose_pred in (ev.pnp(pts3d, z[n + "_kp"], z["K"]), ev.uncertainty_pnp(z[n + "_kp"], w, pts3d, z["K"])):
            pd, add, td, ang = _numpy_metrics(pose_pred, z[n + "_pose"], model, z["K"], diameter, class_type == "glue")
            # numpy's BLAS order is not the kernel's: values agree far below the thresholds' resolution
            assert abs(e.proj_mean_diffs[k] - pd) < 1e-9 and abs(e.add_dists[k] - add) < 1e-9
            assert e.projection_2d_recorder[k] == (pd < 5) and e.add_recorder[k] == (add < diameter * 0.1)
            assert e.cm_degree_5_recorder[k] == (td < 5 and ang < 5)
            k += 1
    p, a, c = e.average_precision(verbose=False)
    assert p == np.mean(e.projection_2d_recorder) and a == np.mean(e.add_recorder)
    assert c == np.mean(e.cm_degree_5_recorder)
