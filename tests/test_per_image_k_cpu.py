"""CPU: the host-side shape rules of per-image camera matrices (extend_utils.check_cameras, and
PoseKeypointPipeline.run / step refusing per-batch cameras it cannot use before anything reaches a device)."""
import numpy as np
import pytest
import torch
from torch import nn

from pvnet_b200 import extend_utils as eu
from pvnet_b200.pipeline import PoseKeypointPipeline


@pytest.mark.parametrize("shape", [(3, 3), (5, 3, 3)])
def test_check_cameras_accepts_one_or_one_per_image(shape):
    eu.check_cameras(shape, 5)
    eu.check_cameras(torch.empty(shape).shape, 5)


@pytest.mark.parametrize("shape, match", [((4, 3, 3), "4 cameras for a batch of 5"), ((6, 3, 3), "6 cameras"),
                                          ((1, 3, 3), "1 cameras"), ((9,), r"\[3,3\] or \[5,3,3\]"),
                                          ((5, 3, 4), r"\[3,3\] or \[5,3,3\]"), ((5, 9), r"\[3,3\] or \[5,3,3\]"),
                                          ((1, 5, 3, 3), r"\[3,3\] or \[5,3,3\]"), ((), r"\[3,3\] or \[5,3,3\]")])
def test_check_cameras_refuses_other_shapes(shape, match):
    with pytest.raises(ValueError, match=match):
        eu.check_cameras(shape, 5)


def test_uncertainty_pnp_batched_refuses_cpu_points():
    with pytest.raises(RuntimeError, match="CUDA"):
        eu.uncertainty_pnp_batched(torch.zeros(2, 9, 2), np.zeros((9, 3)), torch.eye(3).expand(2, 3, 3),
                                   cov=torch.zeros(2, 9, 2, 2))


def _pipe(**kw):
    return PoseKeypointPipeline(nn.Linear(1, 1), with_covariance=kw.pop("with_covariance", True), **kw)


def test_pipeline_refuses_unusable_per_batch_cameras():
    batches = [torch.zeros(2, 8, 8, 3, dtype=torch.uint8)] * 3
    pts = np.zeros((9, 3), np.float32)
    with pytest.raises(ValueError, match="2 camera batches for 3 image batches"):
        _pipe(points_3d=pts).run(batches, camera_matrices=[np.eye(3)] * 2)
    with pytest.raises(ValueError, match="3 cameras for a batch of 2"):
        _pipe(points_3d=pts).run(batches, camera_matrices=[np.stack([np.eye(3)] * 3)] * 3)
    with pytest.raises(ValueError, match="points_3d"):
        _pipe().run(batches, camera_matrices=[np.stack([np.eye(3)] * 2)] * 3)
    with pytest.raises(ValueError, match="with_covariance"):
        _pipe(points_3d=pts, with_covariance=False).run(batches, camera_matrices=[np.eye(3)] * 3)
    with pytest.raises(ValueError, match="points_3d"):
        _pipe().step(batches[0], camera_matrix=torch.eye(3))
