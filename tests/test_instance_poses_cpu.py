"""CPU: the per-instance pose layer's host checks and the planted scenes of tests/instance_pose_cases.py.

- `uncertainty_pnp_instances` refuses CPU tensors; `PoseKeypointPipeline(max_instances=)` refuses what it cannot run.
- Each planted scene is what its test needs: the projected centre is the disc's centre, touching layouts touch, and
  the planted field points at the instance's own projected model points."""
import numpy as np
import pytest
import torch
from torch import nn

from pvnet_b200 import extend_utils as eu
from pvnet_b200.pipeline import PoseKeypointPipeline
from tests import instance_pose_cases as ipc


def test_pnp_instances_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        eu.uncertainty_pnp_instances(torch.zeros(1, 2, 9, 2), torch.ones(1, dtype=torch.int32), ipc.POINTS_3D,
                                     ipc.K_LINEMOD, weights_2d=torch.zeros(1, 2, 9, 3))


@pytest.mark.parametrize("kw", [dict(max_instances=0), dict(max_instances=33), dict(max_instances=2.5),
                                dict(max_instances=True), dict(max_instances=4, points_3d=None),
                                dict(max_instances=4, with_covariance=False), dict(max_instances=4, rng="batched"),
                                dict(max_instances=4, refine=dict(vertices=0, faces=0, near=0.1, far=2.0, depth=dict(gate=0.02)))])
def test_pipeline_max_instances_refusals(kw):
    args = dict(with_covariance=True, points_3d=ipc.POINTS_3D, camera_matrix=ipc.K_LINEMOD)
    args.update(kw)
    with pytest.raises(ValueError):
        PoseKeypointPipeline(nn.Linear(1, 1), **args)


def test_pipeline_max_instances_with_refine_and_snapshotted_camera():
    K = ipc.K_LINEMOD.copy()
    pipe = PoseKeypointPipeline(nn.Linear(1, 1), with_covariance=True, points_3d=ipc.POINTS_3D, camera_matrix=K,
                                max_instances=4, refine=dict(vertices=0, faces=0, near=0.1, far=2.0))
    K[0, 0] = 1.0                                     # the constructor's camera is a snapshot
    assert pipe.refine is not None and float(pipe._k_host[0, 0]) == ipc.K_LINEMOD[0, 0]


def test_pipeline_without_max_instances_unchanged():
    pipe = PoseKeypointPipeline(nn.Linear(1, 1), with_covariance=True, points_3d=ipc.POINTS_3D,
                                camera_matrix=ipc.K_LINEMOD)
    assert pipe.max_instances is None


@pytest.mark.parametrize("n,touching,seed", [(1, False, 1), (3, False, 2), (2, True, 3), (4, True, 4)])
def test_pose_scenes(n, touching, seed):
    s = ipc.pose_scene(n, seed, touching=touching)
    assert sorted(np.unique(s["gt"]).tolist()) == list(range(n + 1))
    for i in range(n):
        c = ipc.project(ipc.POINTS_3D[-1:], s["R"][i], s["t"][i], ipc.K_LINEMOD)[0]
        assert np.allclose(c, s["centers"][i], atol=1e-9)
        assert np.allclose(s["keypoints"][i], ipc.project(ipc.POINTS_3D, s["R"][i], s["t"][i], ipc.K_LINEMOD))
        assert 0.9 <= s["t"][i, 2] <= 1.1
        # a pixel of instance i points at instance i's keypoints
        ys, xs = np.nonzero(s["gt"] == i + 1)
        p = np.array([xs[0], ys[0]], np.float64)
        d = s["keypoints"][i] - p
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        assert np.allclose(s["field"][ys[0], xs[0]], d, atol=1e-5)
    assert bool(ipc.touching_pairs(s["gt"])) == touching
