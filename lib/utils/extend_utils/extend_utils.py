"""`lib.utils.extend_utils.extend_utils` as lib/utils/evaluation_utils.py:16 imports it
(`from lib.utils.extend_utils.extend_utils import uncertainty_pnp, find_nearest_point_idx, uncertainty_pnp_v2`):
the uncertainty-driven PnP and the nearest-point search served by pvnet_b200's device kernels.  The module's other
functions (mesh rasterisation, farthest point sampling) are dataset tooling outside the inference and evaluation
paths and are not provided."""
from pvnet_b200.evaluation import find_nearest_point_idx, uncertainty_pnp_v2  # noqa: F401
from pvnet_b200.extend_utils import covariance_to_weights, uncertainty_pnp, uncertainty_pnp_batched  # noqa: F401

__all__ = ["uncertainty_pnp", "uncertainty_pnp_batched", "covariance_to_weights", "find_nearest_point_idx",
           "uncertainty_pnp_v2"]
