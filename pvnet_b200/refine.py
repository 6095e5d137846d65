"""Silhouette pose refinement on the device, over `pvnet_refine_poses` (csrc/refine.cu, DESIGN.md §26).

The reference declares `post_refinement(mask, pose, K, pts)` (lib/utils/extend_utils/extend_utils.py:181-193) with a
four-step docstring -- find the mask's edge, render the silhouette and back-project it, pair it with the edge,
optimise -- and a `pass` body; the `extend_utils` shim keeps returning None for that name.  `refine_poses` is the
device form: each round renders the mesh at the current pose with `render_mesh`'s renderer, pairs its silhouette
with the mask's contour and takes damped Gauss-Newton steps on the pairs' pixel distances.  oracle/refine_oracle.py
restates it.  No CPU path: without the library or a CUDA device it raises.

With `keypoints` (the voted keypoints, their model points and covariances or weights, as `uncertainty_pnp_batched`
takes them) each step also pulls the keypoints' weighted reprojections towards the votes
(`pvnet_refine_poses_keypoints`, DESIGN.md §27): the rotations an outline barely constrains are held by the
keypoints.

`refine_poses_depth` refines the same way against a registered depth image (`pvnet_refine_poses_depth`, DESIGN.md
§28): point-to-plane ICP of the rendered surface against the observed one, which holds the distance along the
viewing ray that the RGB cues barely see.

`refine_poses_instances` refines every instance of a label map (`pvnet_refine_poses_instances`, DESIGN.md §30): each
instance is refined alone, with a contour that leaves out its borders with other instances and a silhouette that
leaves out what another instance may hide.

`refine_poses_depth_instances` refines every instance of a label map against the depth image
(`pvnet_refine_poses_depth_instances`, DESIGN.md §31): each present row is `refine_poses_depth` on the mask of its own
label, in one launch sequence for the whole map, without reading the instance counts on the host."""
from __future__ import annotations

import ctypes
import math

import torch

from . import _native
from .extend_utils import check_cameras, covariance_to_weights

# status bits of info["status"]
NO_CONTOUR = 1          # the mask has no foreground: the input pose is returned
NO_SILHOUETTE = 2       # the render at the input pose covers nothing: the input pose is returned
FEW_PAIRS = 4           # fewer than 6 pairs at the input pose: the input pose is returned
SINGULAR = 8            # a round's normal equations were singular: that round's starting pose is kept
REJECTED = 16           # a round raised the mean pair distance (or lost its pairs) and was undone
NO_INSTANCE = 32        # refine_poses_instances: the row is past its image's instance count; its pose is the input

# lambda of the keypoint-anchored objective: the best of 0.25, 1 and 4 on the synthetic scenes of
# benchmarks/refine_keypoints.py (DESIGN.md §27); real-data accuracy has not been measured
DEFAULT_KEYPOINT_WEIGHT = 0.25


def _cuda_tensor(name, t):
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise RuntimeError(f"pvnet_b200: `{name}` must be a CUDA tensor (there is no CPU path)")


def _keypoint_inputs(b, dev, keypoints, points_3d, cov, weights_2d, keypoint_weight):
    """Check the keypoint arguments -> (keypoints f32 [b,nk,2], points f32 [nk,3], weights f32 [b,nk,3], nk,
    lambda), all contiguous on `dev`."""
    if points_3d is None:
        raise ValueError("keypoints need points_3d")
    if (cov is None) == (weights_2d is None):
        raise ValueError("pass exactly one of weights_2d / cov with keypoints")
    for name, t in (("keypoints", keypoints), ("points_3d", points_3d), ("cov", cov), ("weights_2d", weights_2d)):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
        if t.device != dev:
            raise ValueError(f"{name} must be on the poses' device {dev}, got {t.device}")
        if not t.dtype.is_floating_point:
            raise ValueError(f"{name} must be floating point, got {t.dtype}")
    if keypoints.dim() != 3 or int(keypoints.shape[0]) != b or keypoints.shape[2] != 2:
        raise ValueError(f"keypoints must be [{b},nk,2], got {tuple(keypoints.shape)}")
    nk = int(keypoints.shape[1])
    if not 4 <= nk <= 32:
        raise ValueError(f"keypoint count must lie in 4..32, got {nk}")
    if tuple(points_3d.shape) != (nk, 3):
        raise ValueError(f"points_3d must be [{nk},3], got {tuple(points_3d.shape)}")
    if cov is not None and tuple(cov.shape) != (b, nk, 2, 2):
        raise ValueError(f"cov must be [{b},{nk},2,2], got {tuple(cov.shape)}")
    if weights_2d is not None and tuple(weights_2d.shape) != (b, nk, 3):
        raise ValueError(f"weights_2d must be [{b},{nk},3], got {tuple(weights_2d.shape)}")
    lam = float(keypoint_weight)
    if not 0.0 <= lam < math.inf:
        raise ValueError(f"keypoint_weight must be finite and >= 0, got {keypoint_weight}")
    wgt = covariance_to_weights(cov) if cov is not None else weights_2d.contiguous().float()
    return keypoints.contiguous().float(), points_3d.contiguous().float(), wgt.contiguous(), nk, lam


def _check_common(mask, poses, K, vertices, faces, near, far, rounds, gate, max_points, point_words):
    """refine_poses's checks, shared with refine_poses_depth -> (device, b, h, w, near, far, rounds, gate,
    max_points); point_words: the fp64 words kept per point, which bounds b * max_points."""
    for name, t in (("mask", mask), ("poses", poses), ("K", K), ("vertices", vertices), ("faces", faces)):
        _cuda_tensor(name, t)
    dev = poses.device
    if any(t.device != dev for t in (mask, K, vertices, faces)):
        raise ValueError("mask, poses, K, vertices and faces must be on one device")
    if poses.dim() != 3 or tuple(poses.shape[1:]) != (3, 4):
        raise ValueError(f"poses must be [b,3,4], got {tuple(poses.shape)}")
    if poses.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"poses must be float32 or float64, got {poses.dtype}")
    b = int(poses.shape[0])
    if b < 1:
        raise ValueError("poses holds no pose")
    if mask.dim() != 3 or int(mask.shape[0]) != b:
        raise ValueError(f"mask must be [{b},H,W], got {tuple(mask.shape)}")
    if mask.dtype.is_floating_point or mask.dtype.is_complex:
        raise ValueError(f"mask must be an integer or bool tensor, got {mask.dtype}")
    h, w = int(mask.shape[1]), int(mask.shape[2])
    if h < 1 or w < 1:
        raise ValueError(f"image size must be positive, got {h}x{w}")
    check_cameras(K.shape, b)
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"vertices must be [nv,3], got {tuple(vertices.shape)}")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must be [nf,3], got {tuple(faces.shape)}")
    if faces.dtype.is_floating_point or faces.dtype.is_complex or faces.dtype == torch.bool:
        raise ValueError(f"faces must hold integer indices, got {faces.dtype}")
    near, far = float(near), float(far)
    if not 0 < near < far < math.inf:
        raise ValueError(f"clip planes must satisfy 0 < near < far, got {near}, {far}")
    rounds, max_points, gate = int(rounds), int(max_points), float(gate)
    if rounds < 0:
        raise ValueError(f"rounds must be >= 0, got {rounds}")
    if not 0 < gate < math.inf:
        raise ValueError(f"gate must be positive and finite, got {gate}")
    if not 1 <= max_points <= (2 ** 31 - 1) // point_words // b:
        raise ValueError(f"max_points must lie in 1..{(2 ** 31 - 1) // point_words // b} for b = {b}, got {max_points}")
    return dev, b, h, w, near, far, rounds, gate, max_points


def _device_inputs(mask, poses, K, vertices, faces):
    """-> mask uint8, poses f64, K f32, vertices f32, faces int32, all contiguous, and nv, nf."""
    nv, nf = int(vertices.shape[0]), int(faces.shape[0])
    m = mask.view(torch.uint8) if mask.dtype in (torch.uint8, torch.bool) else (mask != 0).to(torch.uint8)
    # an index beyond int32 is out of range either way; the clamp keeps it so
    f = faces.contiguous() if faces.dtype == torch.int32 else faces.clamp(-1, nv).to(torch.int32).contiguous()
    return (m.contiguous(), poses.contiguous().double(), K.contiguous().float(), vertices.contiguous().float(), f,
            nv, nf)


def refine_poses(mask, poses, K, vertices, faces, near, far, rounds=8, gate=20.0, max_points=4096,
                 return_info=False, trace=False, keypoints=None, points_3d=None, cov=None, weights_2d=None,
                 keypoint_weight=DEFAULT_KEYPOINT_WEIGHT):
    """Refine b poses of one mesh so its rendered silhouette meets each mask's contour.

    mask [b,H,W] (any integer dtype or bool; nonzero is foreground), poses [b,3,4] (float32 or float64, R | t object
    to OpenCV camera), K [3,3] or [b,3,3], vertices [nv,3] and faces [nf,3] (integer): CUDA tensors on one device.
    The mesh is in the poses' translation units, and so are near and far, the render's clip planes.  Each round
    pairs the silhouette with the contour, drops pairs more than `gate` pixels apart, and keeps at most `max_points`
    points of each (every ceil(n / max_points)-th).  `rounds` is a host constant: a call is a fixed sequence of
    launches, with no host synchronisation, and can be captured in a CUDA graph.  rounds = 0 returns the input.

    -> poses float64 [b,3,4] on the device.  return_info: also a dict of [b] tensors, "status" (int32 bits, see the
    module's constants), "pairs" (int32, the pairs of the last round that took its steps), "dist_before" and
    "dist_after" (float64, the mean pair distance in pixels at the input pose and at the returned one, NaN without
    pairs).  trace: also a dict of the first round's intermediates ("sil_idx", "con_idx", "pair_idx" int32
    [b,max_points], "counts" int32 [b,2], "sil_obj" float64 [b,max_points,3], "normal_eq" float64 [b,27]), for
    checking the stages against the oracle.

    keypoints [b,nk,2] (4 <= nk <= 32, pixels as `uncertainty_pnp_batched` reads them), points_3d [nk,3] (their
    model points, in the mesh's units) and exactly one of cov [b,nk,2,2] / weights_2d [b,nk,3] (converted through
    `covariance_to_weights`), floating-point CUDA tensors on the poses' device: each step then minimises
    (1/n) sum |pi(R X_i + t) - c_i|^2 + (keypoint_weight / nk) sum |W_k (pi(R P_k + t) - x_k)|^2, and a round is
    undone when C = mean pair distance + keypoint_weight * mean_k |W_k e_k| rose or is NaN (DESIGN.md §27).
    return_info then adds "cost_before" and "cost_after" (float64, C at the input pose and at the returned one), and
    trace adds "keypoint_eq" (float64 [b,27], the first step's keypoint sums, unscaled)."""
    dev, b, h, w, near, far, rounds, gate, max_points = _check_common(mask, poses, K, vertices, faces, near, far,
                                                                      rounds, gate, max_points, 3)

    kpt = None
    if keypoints is not None:
        kpt = _keypoint_inputs(b, dev, keypoints, points_3d, cov, weights_2d, keypoint_weight)
    elif points_3d is not None or cov is not None or weights_2d is not None:
        raise ValueError("points_3d, cov and weights_2d go with keypoints")

    m, p, k, v, f, nv, nf = _device_inputs(mask, poses, K, vertices, faces)
    out = torch.empty((b, 3, 4), dtype=torch.float64, device=dev)
    info = torch.empty((b, 2), dtype=torch.int32, device=dev) if return_info else None
    dist = torch.empty((b, 2), dtype=torch.float64, device=dev) if return_info else None
    cost = torch.empty((b, 2), dtype=torch.float64, device=dev) if return_info and kpt is not None else None
    tr, tr_struct = None, None
    if trace:
        tr = dict(sil_idx=torch.full((b, max_points), -1, dtype=torch.int32, device=dev),
                  con_idx=torch.full((b, max_points), -1, dtype=torch.int32, device=dev),
                  counts=torch.zeros((b, 2), dtype=torch.int32, device=dev),
                  sil_obj=torch.zeros((b, max_points, 3), dtype=torch.float64, device=dev),
                  pair_idx=torch.full((b, max_points), -1, dtype=torch.int32, device=dev),
                  normal_eq=torch.full((b, 27), math.nan, dtype=torch.float64, device=dev))
        tr_struct = _native.RefineTrace(*(tr[n].data_ptr() for n in ("sil_idx", "con_idx", "counts", "sil_obj",
                                                                      "pair_idx", "normal_eq")))
        if kpt is not None:
            tr["keypoint_eq"] = torch.full((b, 27), math.nan, dtype=torch.float64, device=dev)
    L = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(L.pvnet_refine_workspace_bytes(b, h, w, max_points, ctypes.byref(need)),
                      "pvnet_refine_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        head = (m.data_ptr(), p.data_ptr(), k.data_ptr(), int(k.dim() == 3), v.data_ptr() if nv else None,
                f.data_ptr() if nf else None, nv, nf, b, h, w, near, far, rounds, gate, max_points)
        outs = (out.data_ptr(), None if info is None else info.data_ptr(), None if dist is None else dist.data_ptr())
        trace_p = None if tr_struct is None else ctypes.byref(tr_struct)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        if kpt is None:
            _native.check(L.pvnet_refine_poses(*head, *outs, trace_p, ws.data_ptr(), need.value, stream),
                          "pvnet_refine_poses")
        else:
            kp, pts, wgt, nk, lam = kpt
            _native.check(L.pvnet_refine_poses_keypoints(
                *head, kp.data_ptr(), pts.data_ptr(), wgt.data_ptr(), nk, lam, *outs,
                None if cost is None else cost.data_ptr(), trace_p,
                None if tr is None else tr["keypoint_eq"].data_ptr(), ws.data_ptr(), need.value, stream),
                "pvnet_refine_poses_keypoints")
    res = (out,)
    if return_info:
        res += (dict(status=info[:, 0], pairs=info[:, 1], dist_before=dist[:, 0], dist_after=dist[:, 1]),)
        if cost is not None:
            res[-1].update(cost_before=cost[:, 0], cost_after=cost[:, 1])
    if trace:
        res += (tr,)
    return res[0] if len(res) == 1 else res


_INT_ELEM = {torch.uint8: 1, torch.int8: 1, torch.int16: 2, torch.int32: 4, torch.int64: 8}


def refine_poses_instances(labels, num, poses, K, vertices, faces, near, far, rounds=8, gate=20.0, max_points=4096,
                           return_info=False, trace=False, keypoints=None, points_3d=None, cov=None, weights_2d=None,
                           keypoint_weight=DEFAULT_KEYPOINT_WEIGHT):
    """`refine_poses` for every instance of a label map (DESIGN.md §30).

    labels [b,H,W] integer CUDA tensor (0 background, j+1 instance j, `ransac_voting_center`'s map as it is; values
    above L count as other instances), num int32 [b] instance counts on the device, poses [b,L,3,4] (1 <= L <= 32,
    b * L <= 1024), K [3,3] or [b,3,3]; keypoints [b,L,nk,2] with cov [b,L,nk,2,2] or weights_2d [b,L,nk,3] as
    `ransac_voting_labels` returns them.  Row (i, j) is refined as `refine_poses` refines one image, except for the
    boundary sets: the contour of instance j is its pixels with a 4-neighbour of value 0 or on the image border, and
    a silhouette pixel whose 3x3 neighbourhood holds another instance is left out.  A row with j >= num[i] keeps its
    input pose with status NO_INSTANCE and costs no render.  Without host synchronisation; graph-capturable.

    -> poses float64 [b,L,3,4]; return_info: a dict of [b,L] tensors as `refine_poses` returns; trace: the first
    round's intermediates with one row per virtual image i * L + j."""
    _cuda_tensor("labels", labels)
    _cuda_tensor("num", num)
    _cuda_tensor("poses", poses)
    if labels.dtype not in _INT_ELEM:
        raise ValueError(f"labels must be an integer tensor, got {labels.dtype}")
    if labels.dim() != 3:
        raise ValueError(f"labels must be [b,H,W], got {tuple(labels.shape)}")
    if poses.dim() != 4 or tuple(poses.shape[2:]) != (3, 4):
        raise ValueError(f"poses must be [b,L,3,4], got {tuple(poses.shape)}")
    b, L = int(poses.shape[0]), int(poses.shape[1])
    h, w = int(labels.shape[1]), int(labels.shape[2])
    if int(labels.shape[0]) != b:
        raise ValueError(f"labels holds {labels.shape[0]} images for {b} pose rows")
    if not 1 <= L <= 32 or b * L > 1024:
        raise ValueError(f"L = {L} instances per image outside 1..32, or b * L = {b * L} above 1024")
    if tuple(num.shape) != (b,) or num.device != poses.device:
        raise ValueError(f"num must be a [{b}] tensor on {poses.device}")
    B = b * L
    _cuda_tensor("K", K)
    check_cameras(K.shape, b)
    # the checks refine_poses makes, on the virtual images (a zero-stride stand-in for their masks)
    stand_in = torch.zeros((), dtype=torch.uint8, device=labels.device).expand(B, h, w)
    dev, _, _, _, near, far, rounds, gate, max_points = _check_common(
        stand_in, poses.flatten(0, 1), K.expand(b, 3, 3).repeat_interleave(L, 0), vertices, faces, near, far, rounds,
        gate, max_points, 3)
    kpt = None
    if keypoints is not None:
        if keypoints.dim() != 4 or tuple(keypoints.shape[:2]) != (b, L):
            raise ValueError(f"keypoints must be [{b},{L},nk,2], got {tuple(keypoints.shape)}")
        kpt = _keypoint_inputs(B, dev, keypoints.flatten(0, 1), points_3d, None if cov is None else cov.flatten(0, 1),
                               None if weights_2d is None else weights_2d.flatten(0, 1), keypoint_weight)
    elif points_3d is not None or cov is not None or weights_2d is not None:
        raise ValueError("points_3d, cov and weights_2d go with keypoints")
    lab = labels.contiguous()
    n32 = num.to(torch.int32).contiguous()
    p = poses.flatten(0, 1).contiguous().double()
    k = K.expand(b, 3, 3).float().repeat_interleave(L, 0).contiguous()        # one camera per virtual image
    nv, nf = int(vertices.shape[0]), int(faces.shape[0])
    v = vertices.contiguous().float()
    f = faces.contiguous() if faces.dtype == torch.int32 else faces.clamp(-1, nv).to(torch.int32).contiguous()
    out = torch.empty((B, 3, 4), dtype=torch.float64, device=dev)
    info = torch.empty((B, 2), dtype=torch.int32, device=dev) if return_info else None
    dist = torch.empty((B, 2), dtype=torch.float64, device=dev) if return_info else None
    cost = torch.empty((B, 2), dtype=torch.float64, device=dev) if return_info and kpt is not None else None
    tr, tr_struct = None, None
    if trace:
        tr = dict(sil_idx=torch.full((B, max_points), -1, dtype=torch.int32, device=dev),
                  con_idx=torch.full((B, max_points), -1, dtype=torch.int32, device=dev),
                  counts=torch.zeros((B, 2), dtype=torch.int32, device=dev),
                  sil_obj=torch.zeros((B, max_points, 3), dtype=torch.float64, device=dev),
                  pair_idx=torch.full((B, max_points), -1, dtype=torch.int32, device=dev),
                  normal_eq=torch.full((B, 27), math.nan, dtype=torch.float64, device=dev))
        tr_struct = _native.RefineTrace(*(tr[x].data_ptr() for x in ("sil_idx", "con_idx", "counts", "sil_obj",
                                                                      "pair_idx", "normal_eq")))
        if kpt is not None:
            tr["keypoint_eq"] = torch.full((B, 27), math.nan, dtype=torch.float64, device=dev)
    kp, pts, wgt, nk, lam = kpt if kpt is not None else (None, None, None, 0, 0.0)
    lib = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(lib.pvnet_refine_workspace_bytes(B, h, w, max_points, ctypes.byref(need)),
                      "pvnet_refine_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        ptr = (lambda t: None if t is None else t.data_ptr())
        _native.check(lib.pvnet_refine_poses_instances(
            lab.data_ptr(), _INT_ELEM[lab.dtype], n32.data_ptr(), L, p.data_ptr(), k.data_ptr(), ptr(v) if nv else None,
            ptr(f) if nf else None, nv, nf, b, h, w, near, far, rounds, gate, max_points, ptr(kp), ptr(pts), ptr(wgt),
            nk, lam, out.data_ptr(), ptr(info), ptr(dist), ptr(cost),
            None if tr_struct is None else ctypes.byref(tr_struct), None if tr is None else ptr(tr.get("keypoint_eq")),
            ws.data_ptr(), need.value, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
            "pvnet_refine_poses_instances")
    res = (out.view(b, L, 3, 4),)
    if return_info:
        d = dict(status=info[:, 0], pairs=info[:, 1], dist_before=dist[:, 0], dist_after=dist[:, 1])
        if cost is not None:
            d.update(cost_before=cost[:, 0], cost_after=cost[:, 1])
        res += ({key: t.view(b, L) for key, t in d.items()},)
    if trace:
        res += (tr,)
    return res[0] if len(res) == 1 else res


def refine_poses_depth(mask, depth, poses, K, vertices, faces, near, far, gate, rounds=8, max_points=4096,
                       depth_scale=1.0, return_info=False, trace=False):
    """Refine b poses of one mesh so its rendered surface meets each registered depth image (DESIGN.md §28).

    mask, poses, K, vertices, faces, near, far, rounds and max_points as for `refine_poses`.  depth [b,H,W] on the
    poses' device: float32 in the poses' units, or uint16 (the LINEMOD PNG format) read as fp32(d) * fp32(depth_scale)
    (depth_scale is only read for uint16); a value <= 0 or not finite is no reading.  Each round pairs every pixel
    that the render covers, the mask holds and the sensor read (with its four 4-neighbours in the image, the mask and
    read, for the observed normal), drops pairs whose rendered and observed points lie more than `gate` apart (in the
    poses' units; there is no default, as there is none for near and far), keeps at most `max_points` (every
    ceil(n / max_points)-th) and takes damped Gauss-Newton steps on sum (n . (R X + t - Y))^2.  A call is a fixed
    sequence of launches, with no host synchronisation, and can be captured in a CUDA graph.  rounds = 0 returns the
    input.

    -> poses float64 [b,3,4] on the device.  return_info: also a dict of [b] tensors, "status" (int32 bits, the
    module's constants: NO_CONTOUR is an empty mask, NO_SILHOUETTE a render that covers nothing, FEW_PAIRS fewer than
    6 pairs at the input pose, which includes no readings), "pairs" (int32, the pairs of the last round that took its
    steps), "dist_before" and "dist_after" (float64, the mean |n . (R X + t - Y)| in the poses' units at the input
    pose and at the returned one, NaN without pairs).  trace: also a dict of the first round's pairs ("pair_idx"
    int32 [b,max_points] pixel indices, "counts" int32 [b,4]: pairs kept, pairs before the stride, mask pixels,
    covered pixels; "X", "Y", "n" float64 [b,max_points,3]; "normal_eq" float64 [b,27]), for checking the stages
    against the oracle."""
    dev, b, h, w, near, far, rounds, gate, max_points = _check_common(mask, poses, K, vertices, faces, near, far,
                                                                      rounds, gate, max_points, 9)
    if not isinstance(depth, torch.Tensor):
        raise ValueError(f"depth must be a torch tensor, got {type(depth).__name__}")
    if depth.device != dev:
        raise ValueError(f"depth must be on the poses' device {dev}, got {depth.device}")
    if tuple(depth.shape) != (b, h, w):
        raise ValueError(f"depth must be [{b},{h},{w}], got {tuple(depth.shape)}")
    if depth.dtype not in (torch.float32, torch.uint16):
        raise ValueError(f"depth must be float32 or uint16, got {depth.dtype}")
    is_u16 = depth.dtype == torch.uint16
    scale = float(depth_scale)
    if not 0 < scale < math.inf:
        raise ValueError(f"depth_scale must be positive and finite, got {depth_scale}")
    m, p, k, v, f, nv, nf = _device_inputs(mask, poses, K, vertices, faces)
    d = depth.contiguous()
    out = torch.empty((b, 3, 4), dtype=torch.float64, device=dev)
    info = torch.empty((b, 2), dtype=torch.int32, device=dev) if return_info else None
    dist = torch.empty((b, 2), dtype=torch.float64, device=dev) if return_info else None
    tr, tr_struct = None, None
    if trace:
        tr = dict(pair_idx=torch.full((b, max_points), -1, dtype=torch.int32, device=dev),
                  counts=torch.zeros((b, 4), dtype=torch.int32, device=dev),
                  X=torch.zeros((b, max_points, 3), dtype=torch.float64, device=dev),
                  Y=torch.zeros((b, max_points, 3), dtype=torch.float64, device=dev),
                  n=torch.zeros((b, max_points, 3), dtype=torch.float64, device=dev),
                  normal_eq=torch.full((b, 27), math.nan, dtype=torch.float64, device=dev))
        tr_struct = _native.RefineDepthTrace(*(tr[x].data_ptr() for x in ("pair_idx", "counts", "X", "Y", "n",
                                                                          "normal_eq")))
    L = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(L.pvnet_refine_depth_workspace_bytes(b, h, w, max_points, ctypes.byref(need)),
                      "pvnet_refine_depth_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _native.check(L.pvnet_refine_poses_depth(
            m.data_ptr(), d.data_ptr(), int(is_u16), scale, p.data_ptr(), k.data_ptr(), int(k.dim() == 3),
            v.data_ptr() if nv else None, f.data_ptr() if nf else None, nv, nf, b, h, w, near, far, rounds, gate,
            max_points, out.data_ptr(), None if info is None else info.data_ptr(),
            None if dist is None else dist.data_ptr(), None if tr_struct is None else ctypes.byref(tr_struct),
            ws.data_ptr(), need.value, stream), "pvnet_refine_poses_depth")
    res = (out,)
    if return_info:
        res += (dict(status=info[:, 0], pairs=info[:, 1], dist_before=dist[:, 0], dist_after=dist[:, 1]),)
    if trace:
        res += (tr,)
    return res[0] if len(res) == 1 else res


def refine_poses_depth_instances(labels, num, depth, poses, K, vertices, faces, near, far, gate, rounds=8,
                                 max_points=4096, depth_scale=1.0, return_info=False, trace=False):
    """`refine_poses_depth` for every instance of a label map (DESIGN.md §31).

    labels [b,H,W] (uint8, int8, int16, int32 or int64; 0 background, j+1 instance j, any other nonzero value another
    instance, so `ransac_voting_center`'s map works as it is), num [b] instance counts on the device, depth [b,H,W]
    float32 or uint16 as `refine_poses_depth` reads it, poses [b,L,3,4] (1 <= L <= 32, b * L <= 1024), K [3,3] or
    [b,3,3]: CUDA tensors on one device.  Row (i, j) with j < num[i] is bit for bit
    `refine_poses_depth((labels[i] == j+1)[None], depth[i][None], poses[i, j][None], K[i], ...)`: a pixel pairs only
    when it and its four 4-neighbours carry label j+1, so no pair or observed normal is taken across an instance
    border.  A row with j >= num[i] keeps its input pose with status NO_INSTANCE, pairs 0 and NaN distances, and costs
    no pairs or steps.  Without host synchronisation; graph-capturable.

    -> poses float64 [b,L,3,4]; return_info: a dict of [b,L] tensors as `refine_poses_depth` returns; trace: its
    first-round dict with one row per virtual image i * L + j (pixel indices r * W + c in image i; an absent row's
    counts are 0)."""
    _cuda_tensor("labels", labels)
    _cuda_tensor("num", num)
    _cuda_tensor("depth", depth)
    _cuda_tensor("poses", poses)
    if labels.dtype not in _INT_ELEM:
        raise ValueError(f"labels must be an integer tensor, got {labels.dtype}")
    if labels.dim() != 3:
        raise ValueError(f"labels must be [b,H,W], got {tuple(labels.shape)}")
    if poses.dim() != 4 or tuple(poses.shape[2:]) != (3, 4):
        raise ValueError(f"poses must be [b,L,3,4], got {tuple(poses.shape)}")
    b, L = int(poses.shape[0]), int(poses.shape[1])
    h, w = int(labels.shape[1]), int(labels.shape[2])
    if int(labels.shape[0]) != b:
        raise ValueError(f"labels holds {labels.shape[0]} images for {b} pose rows")
    if not 1 <= L <= 32 or b * L > 1024:
        raise ValueError(f"L = {L} instances per image outside 1..32, or b * L = {b * L} above 1024")
    if tuple(num.shape) != (b,) or num.device != poses.device:
        raise ValueError(f"num must be a [{b}] tensor on {poses.device}")
    B = b * L
    _cuda_tensor("K", K)
    check_cameras(K.shape, b)
    # the checks refine_poses_depth makes, on the virtual images (a zero-stride stand-in for their masks)
    stand_in = torch.zeros((), dtype=torch.uint8, device=labels.device).expand(B, h, w)
    dev, _, _, _, near, far, rounds, gate, max_points = _check_common(
        stand_in, poses.flatten(0, 1), K.expand(b, 3, 3).repeat_interleave(L, 0), vertices, faces, near, far, rounds,
        gate, max_points, 9)
    if depth.device != dev:
        raise ValueError(f"depth must be on the poses' device {dev}, got {depth.device}")
    if tuple(depth.shape) != (b, h, w):
        raise ValueError(f"depth must be [{b},{h},{w}], got {tuple(depth.shape)}")
    if depth.dtype not in (torch.float32, torch.uint16):
        raise ValueError(f"depth must be float32 or uint16, got {depth.dtype}")
    is_u16 = depth.dtype == torch.uint16
    scale = float(depth_scale)
    if not 0 < scale < math.inf:
        raise ValueError(f"depth_scale must be positive and finite, got {depth_scale}")
    lab = labels.contiguous()
    d = depth.contiguous()
    n32 = num.to(torch.int32).contiguous()
    p = poses.flatten(0, 1).contiguous().double()
    k = K.expand(b, 3, 3).float().repeat_interleave(L, 0).contiguous()        # one camera per virtual image
    nv, nf = int(vertices.shape[0]), int(faces.shape[0])
    v = vertices.contiguous().float()
    f = faces.contiguous() if faces.dtype == torch.int32 else faces.clamp(-1, nv).to(torch.int32).contiguous()
    out = torch.empty((B, 3, 4), dtype=torch.float64, device=dev)
    info = torch.empty((B, 2), dtype=torch.int32, device=dev) if return_info else None
    dist = torch.empty((B, 2), dtype=torch.float64, device=dev) if return_info else None
    tr, tr_struct = None, None
    if trace:
        tr = dict(pair_idx=torch.full((B, max_points), -1, dtype=torch.int32, device=dev),
                  counts=torch.zeros((B, 4), dtype=torch.int32, device=dev),
                  X=torch.zeros((B, max_points, 3), dtype=torch.float64, device=dev),
                  Y=torch.zeros((B, max_points, 3), dtype=torch.float64, device=dev),
                  n=torch.zeros((B, max_points, 3), dtype=torch.float64, device=dev),
                  normal_eq=torch.full((B, 27), math.nan, dtype=torch.float64, device=dev))
        tr_struct = _native.RefineDepthTrace(*(tr[x].data_ptr() for x in ("pair_idx", "counts", "X", "Y", "n",
                                                                          "normal_eq")))
    lib = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(lib.pvnet_refine_depth_instances_workspace_bytes(b, L, h, w, max_points, ctypes.byref(need)),
                      "pvnet_refine_depth_instances_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        ptr = (lambda t: None if t is None else t.data_ptr())
        _native.check(lib.pvnet_refine_poses_depth_instances(
            lab.data_ptr(), _INT_ELEM[lab.dtype], n32.data_ptr(), L, d.data_ptr(), int(is_u16), scale, p.data_ptr(),
            k.data_ptr(), ptr(v) if nv else None, ptr(f) if nf else None, nv, nf, b, h, w, near, far, rounds, gate,
            max_points, out.data_ptr(), ptr(info), ptr(dist), None if tr_struct is None else ctypes.byref(tr_struct),
            ws.data_ptr(), need.value, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
            "pvnet_refine_poses_depth_instances")
    res = (out.view(b, L, 3, 4),)
    if return_info:
        fields = dict(status=info[:, 0], pairs=info[:, 1], dist_before=dist[:, 0], dist_after=dist[:, 1])
        res += ({key: x.view(b, L) for key, x in fields.items()},)
    if trace:
        res += (tr,)
    return res[0] if len(res) == 1 else res
