"""`lib.utils.evaluation_utils` as tools/demo.py:9 (`pnp`) and tools/train_linemod.py:18 (`Evaluator`) import it:
the PnP and the pose metrics served by pvnet_b200's device kernels (pvnet_b200/evaluation.py).  Unlike the
reference module, importing it needs neither cv2, scipy nor plyfile; the dataset classes `Evaluator` uses are
imported from this tree when an Evaluator is built."""
from pvnet_b200.evaluation import (Evaluator, find_nearest_point_distance, find_nearest_point_idx,  # noqa: F401
                                   pnp, pose_metrics, uncertainty_pnp_v2)
from pvnet_b200.extend_utils import uncertainty_pnp  # noqa: F401

__all__ = ["pnp", "find_nearest_point_distance", "Evaluator", "pose_metrics", "find_nearest_point_idx",
           "uncertainty_pnp", "uncertainty_pnp_v2"]
