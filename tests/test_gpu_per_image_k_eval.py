"""GPU: per-image camera matrices from keypoints to poses to metrics.

- PoseKeypointPipeline with per-batch cameras (`run(..., camera_matrices=)`, `step(x, camera_matrix=)`): its poses
  are what uncertainty_pnp_batched gives on the pipeline's own keypoints and covariances with those cameras, eagerly
  and with graph=True (one captured graph per input buffer serving batches with different cameras).
- Evaluator.evaluate_keypoints_batch: the poses and metric records of the per-image evaluate / evaluate_uncertainty
  with intri_matrix, bit for bit, without a host synchronisation."""
import sys
import types

import numpy as np
import pytest
import torch

from pvnet_b200 import evaluation as ev
from pvnet_b200 import extend_utils as eu
from pvnet_b200.model_repository import Resnet18_8s
from pvnet_b200.pipeline import PoseKeypointPipeline
from tests import pnp_cases as pc
from tests.helpers import seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _cameras(rng, n):
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = rng.uniform(450, 700, n), rng.uniform(450, 700, n)
    K[:, 0, 2], K[:, 1, 2] = rng.uniform(0, 128, n), rng.uniform(0, 96, n)
    K[:, 2, 2] = 1.0
    return K


# ------------------------------------------------------------------ pipeline
@pytest.mark.parametrize("graph", [False, True])
def test_pipeline_per_batch_cameras_equal_separate_pnp(graph):
    net = Resnet18_8s(18, 2)
    net.load_state_dict(seeded_state_dict(net, 3))
    net = net.to(DEV).eval()
    rng = np.random.default_rng(8)
    pts3d = rng.uniform(-0.1, 0.1, (9, 3)).astype(np.float32)
    pipe = PoseKeypointPipeline(net, round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=128,
                                points_3d=pts3d, graph=graph)
    n, b = 4, 3
    hosts = [torch.from_numpy(rng.integers(0, 256, (b, 96, 128, 3), dtype=np.uint8)).pin_memory() for _ in range(n)]
    cams = [torch.from_numpy(_cameras(rng, b)).pin_memory() for _ in range(n)]

    def run():
        kp = [torch.empty([b, 9, 2]).pin_memory() for _ in range(n)]
        cov = [torch.empty([b, 9, 2, 2]).pin_memory() for _ in range(n)]
        pose = [torch.empty([b, 3, 4], dtype=torch.float64).pin_memory() for _ in range(n)]
        pipe.run(hosts, out_host=kp, cov_host=cov, pose_host=pose, camera_matrices=cams)
        return kp, cov, pose
    torch.manual_seed(17)
    for _ in range(2 if graph else 1):                      # with graph=True: capture, then pure replays
        kp, cov, pose = run()
    p3 = torch.from_numpy(pts3d).to(DEV)
    for i in range(n):
        want = eu.uncertainty_pnp_batched(kp[i].to(DEV), p3, cams[i].to(DEV), cov=cov[i].to(DEV)).cpu()
        assert torch.equal(torch.nan_to_num(pose[i]), torch.nan_to_num(want)), i
    # the cameras do reach the solver: other cameras, other poses
    other = eu.uncertainty_pnp_batched(kp[0].to(DEV), p3, cams[1].to(DEV), cov=cov[0].to(DEV)).cpu()
    assert not torch.equal(torch.nan_to_num(pose[0]), torch.nan_to_num(other))
    # step() with a CUDA [b,3,3]: the same as the separate call on its own keypoints
    with torch.no_grad():
        k, c, p = pipe.step(hosts[0].to(DEV), camera_matrix=cams[2].to(DEV))
        assert torch.equal(torch.nan_to_num(p), torch.nan_to_num(eu.uncertainty_pnp_batched(k, p3, cams[2].to(DEV),
                                                                                             cov=c)))
    with pytest.raises(ValueError):
        pipe.run(hosts, camera_matrices=cams[:2])
    with pytest.raises(ValueError):
        pipe.run(hosts, camera_matrices=[torch.ones(b + 1, 3, 3, dtype=torch.float64)] * n)


# ------------------------------------------------------------------ Evaluator
class _ModelDB:
    def __init__(self, model, diameter):
        self.model, self.diameter = model, diameter

    def get_ply_model(self, class_type):
        return self.model

    def get_diameter(self, class_type):
        return self.diameter


class _Projector:
    intrinsic_matrix = {"linemod": pc.K_LINEMOD}


def _truncated_batch(b=16, seed=0):
    """A batch of the LINEMOD cat's 9 keypoints seen through per-image cameras: float32 keypoints, covariances,
    ground-truth poses [b,3,4] (float32, as the loader gives them) and float32 cameras [b,3,3]."""
    rng = np.random.default_rng(seed)
    P = np.load(pc.GOLDEN)["points_3d"]
    K = np.stack([pc.K_LINEMOD] * b)
    K[:, 0, 2] -= rng.uniform(-200, 200, b)                # crop offsets move the principal point
    K[:, 1, 2] -= rng.uniform(-150, 150, b)
    K = K.astype(np.float32)
    R, t = pc.poses("cat", b, rng)
    cov = pc.random_cov(rng, (b, 9))
    cov[:, 2] *= 40.0                                       # one keypoint per image far less certain
    uv = np.stack([pc.project(P, R[i:i + 1], t[i:i + 1], K[i].astype(np.float64))[0] for i in range(b)])
    pose = np.concatenate([R, t[:, :, None]], 2).astype(np.float32)
    return P, K, pc.noisy(rng, uv, cov), cov.astype(np.float32), pose


@pytest.mark.parametrize("class_type", ["cat", "glue"])
def test_evaluate_keypoints_batch_equals_per_image_records(monkeypatch, class_type):
    P, K, kp, cov, pose = _truncated_batch()
    vt = types.ModuleType("lib.datasets.linemod_dataset")

    class VotingType:
        BB8 = 0

        @staticmethod
        def get_pts_3d(vote_type, class_type):
            return P
    vt.VotingType = VotingType
    monkeypatch.setitem(sys.modules, "lib.datasets", types.ModuleType("lib.datasets"))
    monkeypatch.setitem(sys.modules, "lib.datasets.linemod_dataset", vt)
    model = np.random.default_rng(2).uniform(-0.05, 0.05, (1500, 3)).astype(np.float32)
    diameter = 0.12

    def evaluator():
        return ev.Evaluator(model_db=_ModelDB(model, diameter), projector=_Projector())
    kp_d, cov_d, pose_d, K_d = (torch.from_numpy(x).to(DEV) for x in (kp, cov, pose, K))
    for uncertain in (False, True):
        one = evaluator()
        poses_one = []
        for i in range(len(kp)):                            # tools/train_linemod.py:199-205, truncated branch
            if uncertain:
                poses_one.append(one.evaluate_uncertainty(kp[i], cov[i], pose[i], class_type, "use_intrinsic",
                                                          intri_matrix=K[i]))
            else:
                poses_one.append(one.evaluate(kp[i], pose[i], class_type, "use_intrinsic", intri_matrix=K[i]))
        batch = evaluator()
        covar = cov_d if uncertain else None
        batch.evaluate_keypoints_batch(kp_d, pose_d, class_type, K_d, covar=covar)      # first call: points copied
        batch.batch_totals = None
        torch.cuda.synchronize()
        prev = torch.cuda.get_sync_debug_mode()
        torch.cuda.set_sync_debug_mode("error")
        try:
            pose_pred, m = batch.evaluate_keypoints_batch(kp_d, pose_d, class_type, K_d, covar=covar)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
        pose_pred, m = pose_pred.cpu().numpy(), m.cpu().numpy()
        assert np.array_equal(pose_pred, np.stack(poses_one))
        assert np.array_equal(m[:, 0], np.array(one.add_dists))
        assert np.array_equal(m[:, 1], np.array(one.proj_mean_diffs))
        assert np.array_equal((m[:, 2] < 5) & (m[:, 3] < 5), np.array(one.cm_degree_5_recorder))
        assert np.array_equal(m[:, 0] < diameter * 0.1, np.array(one.add_recorder))
        assert np.isfinite(m).all()
        assert batch.average_precision(verbose=False) == one.average_precision(verbose=False)
