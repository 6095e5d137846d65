"""The reference's lib/utils/extend_utils on the device.

Farthest point sampling and binary mesh rasterisation (`farthest_point_sampling`, `mesh_binary_rasterization`,
extend_utils.py:7-37) run over `pvnet_farthest_point_sampling` / `pvnet_mesh_binary_rasterization` (csrc/extend.cu)
and return what the reference's compiled code returns, bit for bit (DESIGN.md §11).

Device-side uncertainty-driven PnP: the reference's `uncertainty_pnp`
(zju3dv/pvnet lib/utils/extend_utils/extend_utils.py:63-114) and the covariance -> weight step of
`Evaluator.evaluate_uncertainty` (lib/utils/evaluation_utils.py:165-201), over the C ABI
(`pvnet_uncertainty_pnp`, `pvnet_covariance_to_weights` in include/pvnet_b200.h).

    uncertainty_pnp(points_2d [pn,2], weights_2d [pn,3], points_3d [pn,3], camera_matrix [3,3]) -> Rt [3,4]

keeps the reference's signature and return type (numpy float64) for numpy inputs -- the arrays are
moved to the current CUDA device; batched CUDA tensors ([b,pn,2], [b,pn,3]) return a float64 CUDA
tensor [b,3,4] with no host synchronisation, which is what `PoseKeypointPipeline(with_pose=True)` uses so
that poses, not keypoints, are what leaves the GPU.  The batched form also takes one camera matrix per image as a
CUDA tensor [b,3,3] (`pvnet_uncertainty_pnp_per_image_k`).  `uncertainty_pnp_instances` solves the [b,L] instance
rows of a label-map vote and leaves the rows past each image's instance count unsolved
(`pvnet_uncertainty_pnp_instances`, DESIGN.md §30).  No CPU path: without the library or a CUDA device these
functions raise.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _native


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _camera(camera_matrix):
    k = np.asarray(camera_matrix.detach().cpu() if isinstance(camera_matrix, torch.Tensor) else camera_matrix,
                   dtype=np.float64).reshape(3, 3)
    return (ctypes.c_double * 9)(*k.ravel().tolist())


def covariance_to_weights(cov: torch.Tensor) -> torch.Tensor:
    """cov [...,2,2] CUDA float32 -> weights [...,3] = (wxx, wxy, wyy) of inv(sqrtm(cov))
    (evaluation_utils.py:170-181; zeros where the reference skips the point)."""
    if not cov.is_cuda:
        raise RuntimeError("pvnet_b200: `cov` must be a CUDA tensor (there is no CPU path)")
    c = cov.contiguous().float()
    n = c.numel() // 4
    out = torch.empty(tuple(c.shape[:-2]) + (3,), dtype=torch.float32, device=c.device)
    with torch.cuda.device(c.device):
        _native.check(_native.lib().pvnet_covariance_to_weights(c.data_ptr(), n, out.data_ptr(), _stream(c.device)),
                      "pvnet_covariance_to_weights")
    return out


def check_cameras(shape, b: int):
    """Raise ValueError unless `shape` is [3,3] (one camera for the batch) or [b,3,3] (one per image)."""
    shape = tuple(shape)
    if shape == (3, 3) or shape == (b, 3, 3):
        return
    if len(shape) == 3 and shape[1:] == (3, 3):
        raise ValueError(f"camera_matrix holds {shape[0]} cameras for a batch of {b} images")
    raise ValueError(f"camera_matrix must be [3,3] or [{b},3,3], got {shape}")


def uncertainty_pnp_batched(points_2d, points_3d, camera_matrix, weights_2d=None, cov=None, return_info=False):
    """points_2d [b,pn,2] CUDA; weights_2d [b,pn,3] or cov [b,pn,2,2] (exactly one); points_3d [pn,3];
    camera_matrix a host 3x3 (numpy, list, CPU tensor) for every image, or a CUDA tensor [b,3,3] (one camera per
    image, the truncated-LINEMOD form) or [3,3].  A CUDA camera stays on the device (no host synchronisation) and
    goes to `pvnet_uncertainty_pnp_per_image_k` as float64 [b,3,3]; a [3,3] one is expanded to every image, which
    gives bit for bit the poses of the host 3x3.  -> poses float64 [b,3,4] on the device (and info int32 [b,2];
    status bit 4 marks an image whose K has a zero focal length, its pose is NaN)."""
    if not points_2d.is_cuda:
        raise RuntimeError("pvnet_b200: `points_2d` must be a CUDA tensor (there is no CPU path)")
    if (weights_2d is None) == (cov is None):
        raise ValueError("pass exactly one of weights_2d / cov")
    dev = points_2d.device
    p2 = points_2d.contiguous().float()
    b, pn, _ = p2.shape
    p3 = torch.as_tensor(points_3d, dtype=torch.float32, device=dev).contiguous()
    if tuple(p3.shape) != (pn, 3):
        raise ValueError(f"points_3d must be [{pn},3], got {tuple(p3.shape)}")
    w = None if weights_2d is None else weights_2d.to(dev).contiguous().float()
    c = None if cov is None else cov.to(dev).contiguous().float()
    out = torch.empty([b, 3, 4], dtype=torch.float64, device=dev)
    info = torch.empty([b, 2], dtype=torch.int32, device=dev) if return_info else None
    args = (p2.data_ptr(), None if c is None else c.data_ptr(), None if w is None else w.data_ptr(), p3.data_ptr())
    tail = (b, pn, out.data_ptr(), None if info is None else info.data_ptr(), _stream(dev))
    with torch.cuda.device(dev):
        if isinstance(camera_matrix, torch.Tensor) and camera_matrix.is_cuda:
            check_cameras(camera_matrix.shape, b)
            ks = camera_matrix.to(device=dev, dtype=torch.float64).expand(b, 3, 3).contiguous()
            _native.check(_native.lib().pvnet_uncertainty_pnp_per_image_k(*args, ks.data_ptr(), *tail),
                          "pvnet_uncertainty_pnp_per_image_k")
        else:
            _native.check(_native.lib().pvnet_uncertainty_pnp(*args, _camera(camera_matrix), *tail),
                          "pvnet_uncertainty_pnp")
    return (out, info) if return_info else out


def uncertainty_pnp_instances(points_2d, num, points_3d, camera_matrix, weights_2d=None, cov=None, return_info=False):
    """One pose per instance row of a label-map vote (DESIGN.md §30): points_2d [b,L,pn,2] CUDA, as
    `ransac_voting_labels` returns them; weights_2d [b,L,pn,3] or cov [b,L,pn,2,2] (exactly one); num the int32 [b]
    instance count of `ransac_voting_center`, on the device; points_3d [pn,3]; camera_matrix [3,3] or [b,3,3], host or
    CUDA (a host one is copied to the device once, with the call's other inputs).  1 <= L <= 32, b * L <= 1024.
    Row (i, j) with j < num[i] is solved with image i's camera, bit for bit as `uncertainty_pnp_batched` solves that
    row; a row with j >= num[i] is not solved: its pose is NaN and its info (8, 0).  num stays on the device: the call
    does not synchronise.  -> poses float64 [b,L,3,4] on the device (and info int32 [b,L,2])."""
    if not points_2d.is_cuda:
        raise RuntimeError("pvnet_b200: `points_2d` must be a CUDA tensor (there is no CPU path)")
    if (weights_2d is None) == (cov is None):
        raise ValueError("pass exactly one of weights_2d / cov")
    if points_2d.dim() != 4 or points_2d.shape[-1] != 2:
        raise ValueError(f"points_2d must be [b,L,pn,2], got {tuple(points_2d.shape)}")
    dev = points_2d.device
    p2 = points_2d.contiguous().float()
    b, L, pn, _ = p2.shape
    if not 1 <= L <= 32 or b * L > 1024:
        raise ValueError(f"L = {L} instances per image outside 1..32, or b * L = {b * L} above 1024")
    if not 4 <= pn <= 32:
        raise ValueError(f"point count {pn} outside [4,32]")
    if not (isinstance(num, torch.Tensor) and num.device == dev and tuple(num.shape) == (b,)):
        raise ValueError(f"num must be a [{b}] tensor on {dev}")
    n = num.to(torch.int32).contiguous()
    p3 = torch.as_tensor(points_3d, dtype=torch.float32, device=dev).contiguous()
    if tuple(p3.shape) != (pn, 3):
        raise ValueError(f"points_3d must be [{pn},3], got {tuple(p3.shape)}")
    want = (b, L, pn, 3) if cov is None else (b, L, pn, 2, 2)
    given = weights_2d if cov is None else cov
    if tuple(given.shape) != want:
        raise ValueError(f"{'weights_2d' if cov is None else 'cov'} must be {list(want)}, got {tuple(given.shape)}")
    w = None if weights_2d is None else weights_2d.to(dev).contiguous().float()
    c = None if cov is None else cov.to(dev).contiguous().float()
    k = torch.as_tensor(camera_matrix.detach() if isinstance(camera_matrix, torch.Tensor) else
                        np.asarray(camera_matrix, np.float64), dtype=torch.float64)
    check_cameras(k.shape, b)
    ks = k.to(dev).expand(b, 3, 3).contiguous()
    out = torch.empty([b, L, 3, 4], dtype=torch.float64, device=dev)
    info = torch.empty([b, L, 2], dtype=torch.int32, device=dev) if return_info else None
    with torch.cuda.device(dev):
        _native.check(_native.lib().pvnet_uncertainty_pnp_instances(
            p2.data_ptr(), None if c is None else c.data_ptr(), None if w is None else w.data_ptr(), p3.data_ptr(),
            ks.data_ptr(), n.data_ptr(), L, b, pn, out.data_ptr(), None if info is None else info.data_ptr(),
            _stream(dev)), "pvnet_uncertainty_pnp_instances")
    return (out, info) if return_info else out


def uncertainty_pnp(points_2d, weights_2d, points_3d, camera_matrix):
    """Reference signature (extend_utils.py:63): numpy [pn,2], [pn,3] (wxx,wxy,wyy), [pn,3], [3,3] ->
    Rt numpy float64 [3,4].  Batched CUDA tensors are accepted too (see uncertainty_pnp_batched)."""
    if isinstance(points_2d, torch.Tensor) and points_2d.dim() == 3:
        return uncertainty_pnp_batched(points_2d, points_3d, camera_matrix, weights_2d=weights_2d)
    if not torch.cuda.is_available():
        raise RuntimeError("pvnet_b200: uncertainty_pnp needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    p2 = torch.as_tensor(np.asarray(points_2d, np.float32), device=dev)[None]
    w = torch.as_tensor(np.asarray(weights_2d, np.float32), device=dev)[None]
    assert p2.shape[1] == np.asarray(points_3d).shape[0] and p2.shape[1] >= 4          # extend_utils.py:72
    return uncertainty_pnp_batched(p2, np.asarray(points_3d, np.float32), camera_matrix, weights_2d=w)[0].cpu().numpy()


def _default_device():
    if not torch.cuda.is_available():
        raise RuntimeError("pvnet_b200: this function needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


def farthest_point_sampling(pts, sn, init_center=False, *, start=None, return_indices=False):
    """The reference's farthest_point_sampling (extend_utils.py:22-37) over `pvnet_farthest_point_sampling`.

    numpy pts [pn,3] -> float32 numpy [sn,3], the sampled points ``pts[idxs]``, as the reference returns.  A CUDA
    tensor [pn,3] or [b,pn,3] (one cloud per batch entry) gives a float32 CUDA tensor [sn,3] / [b,sn,3] and does
    not synchronise.  return_indices=True returns the int32 indices [sn] / [b,sn] instead of the points.

    init_center=True starts from the point farthest from the bounding-box centre and is deterministic (the mode
    lib/utils/data_utils.py uses for the keypoints).  Otherwise the reference starts at rand() % pn; here `start`
    (an int, or one per cloud) is that first index, taken modulo pn, and when it is None it is drawn uniformly in
    [0, pn) from torch's default generator (the CUDA one for CUDA input).
    """
    as_numpy = not isinstance(pts, torch.Tensor)
    if as_numpy:
        pts = np.asarray(pts)
        pn = pts.shape[0]
        assert pts.shape[1] == 3                                                      # extend_utils.py:24
        dev = _default_device()
        p = torch.as_tensor(np.ascontiguousarray(pts, np.float32), device=dev)[None]
    else:
        if not pts.is_cuda:
            raise RuntimeError("pvnet_b200: `pts` must be a CUDA tensor (there is no CPU path)")
        if pts.dim() not in (2, 3) or pts.shape[-1] != 3:
            raise ValueError(f"pts must be [pn,3] or [b,pn,3], got {tuple(pts.shape)}")
        dev = pts.device
        p = (pts if pts.dim() == 3 else pts[None]).contiguous().float()
    b, pn = int(p.shape[0]), int(p.shape[1])
    if pn < 1:
        raise ValueError("farthest_point_sampling needs at least one point")
    sn = int(sn)
    if sn < 0:
        raise ValueError(f"negative sample count {sn}")
    st = None
    if not init_center:
        if start is None:
            st = torch.randint(0, pn, (b,), dtype=torch.int32, device=dev)
        else:
            st = torch.as_tensor(start, dtype=torch.int32).reshape(-1).to(dev)
            if st.numel() == 1:
                st = st.expand(b)
            if st.numel() != b:
                raise ValueError(f"start has {st.numel()} entries for {b} clouds")
            st = st.contiguous()
    idxs = torch.empty((b, sn), dtype=torch.int32, device=dev)
    L = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(L.pvnet_farthest_point_sampling_workspace_bytes(b, pn, ctypes.byref(need)),
                      "pvnet_farthest_point_sampling_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev) if need.value else None
        _native.check(L.pvnet_farthest_point_sampling(
            p.data_ptr(), None if st is None else st.data_ptr(), b, pn, sn, idxs.data_ptr(),
            None if ws is None else ws.data_ptr(), need.value, _stream(dev)), "pvnet_farthest_point_sampling")
    single = as_numpy or pts.dim() == 2
    if return_indices:
        out = idxs[0] if single else idxs
    else:
        out = torch.gather(p, 1, idxs.long()[..., None].expand(b, sn, 3))
        out = out[0] if single else out
    return out.cpu().numpy() if as_numpy else out


def mesh_binary_rasterization(triangles_2d, h, w):
    """The reference's mesh_binary_rasterization (extend_utils.py:7-20) over `pvnet_mesh_binary_rasterization`.

    numpy triangles [tn,3,2] (pixel x, y) -> uint8 numpy mask [h,w] of 0/1.  A CUDA tensor [tn,3,2] or [b,tn,3,2]
    gives a uint8 CUDA tensor [h,w] / [b,h,w] without synchronising."""
    as_numpy = not isinstance(triangles_2d, torch.Tensor)
    if as_numpy:
        t = np.asarray(triangles_2d)
        assert t.shape[1] == 3                                                        # extend_utils.py:9-10
        assert t.shape[2] == 2
        dev = _default_device()
        tri = torch.as_tensor(np.ascontiguousarray(t, np.float32), device=dev)[None]
    else:
        if not triangles_2d.is_cuda:
            raise RuntimeError("pvnet_b200: `triangles_2d` must be a CUDA tensor (there is no CPU path)")
        if triangles_2d.dim() not in (3, 4) or tuple(triangles_2d.shape[-2:]) != (3, 2):
            raise ValueError(f"triangles_2d must be [tn,3,2] or [b,tn,3,2], got {tuple(triangles_2d.shape)}")
        dev = triangles_2d.device
        tri = (triangles_2d if triangles_2d.dim() == 4 else triangles_2d[None]).contiguous().float()
    b, tn = int(tri.shape[0]), int(tri.shape[1])
    h, w = int(h), int(w)
    if h < 2 or w < 2:
        raise ValueError(f"the mask must be at least 2x2, got {h}x{w}")
    mask = torch.empty((b, h, w), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _native.check(_native.lib().pvnet_mesh_binary_rasterization(tri.data_ptr() if tn else None, b, tn, h, w,
                                                                     mask.data_ptr(), _stream(dev)),
                      "pvnet_mesh_binary_rasterization")
    single = as_numpy or triangles_2d.dim() == 3
    out = mask[0] if single else mask
    return out.cpu().numpy() if as_numpy else out
