"""`lib.utils.extend_utils.extend_utils` with the reference module's eight public names, served by pvnet_b200's
device kernels where the reference has native code:

  - uncertainty_pnp, uncertainty_pnp_v2, find_nearest_point_idx: as lib/utils/evaluation_utils.py:16 imports them;
  - farthest_point_sampling, mesh_binary_rasterization: as lib/utils/data_utils.py:18 imports the first (the
    keypoints of `LineModModelDB.compute_farthest_surface_point_3d[_num]`), bit-identical to the reference's code;
  - post_refinement: the reference's body is `pass`, so it returns None;
  - render_mesh_depth, render_mesh_rgb: raise NotImplementedError -- their native code is commented out of the
    reference's own extension (src/utils_python_binding.h, build_extend_utils_cffi.py:32), so they cannot run there
    either.

Importing this module loads neither cv2 nor plyfile."""
from pvnet_b200.evaluation import find_nearest_point_idx, uncertainty_pnp_v2  # noqa: F401
from pvnet_b200.extend_utils import (covariance_to_weights, farthest_point_sampling,  # noqa: F401
                                     mesh_binary_rasterization, uncertainty_pnp, uncertainty_pnp_batched)

__all__ = ["uncertainty_pnp", "uncertainty_pnp_batched", "covariance_to_weights", "find_nearest_point_idx",
           "uncertainty_pnp_v2", "farthest_point_sampling", "mesh_binary_rasterization", "post_refinement",
           "render_mesh_depth", "render_mesh_rgb"]


def post_refinement(mask, pose, K, pts):
    """The reference's post_refinement is a stub (`pass`): it returns None."""
    return None


def _not_built(name):
    raise NotImplementedError(
        f"{name}: the reference's renderer (render_depth_cffi / render_rgb_cffi) is commented out of its own "
        "extension build (src/utils_python_binding.h, build_extend_utils_cffi.py:32), so this function cannot run "
        "there either; mesh rendering is not provided")


def render_mesh_depth(RT, K, vert, face, h, w, init):
    _not_built("render_mesh_depth")


def render_mesh_rgb(RT, K, vert, colors, face, h, w, init):
    _not_built("render_mesh_rgb")
