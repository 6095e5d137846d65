"""Mesh rendering on the device: depth and flat-shaded RGB of one mesh at a batch of poses, over `pvnet_render_mesh`
(csrc/render.cu).  The conventions are those of the reference's OpenGL backend (lib/utils/opengl_render_backend.py
`render`, DESIGN.md §24): pixel (r, c) samples the OpenCV image point (c + 0.5, r + 0.5), depth is the camera-space
Z of the nearest face (0 where none), and RGB is the flat-shaded vertex colour with the light at the camera.
oracle/render_oracle.py restates it bit for bit.  No CPU path: without the library or a CUDA device it raises.

Label maps (DESIGN.md §25, over `pvnet_render_label_map`): `MeshSet` packs several meshes once, `render_label_map`
gives each pixel the label of the nearest one in one depth test, and `masks_of_all_objects` /
`get_mask_of_all_objects` compute the reference's Occlusion-LINEMOD label maps (lib/utils/data_utils.py:788-826)
from its own dataset object; oracle/label_map_oracle.py restates them."""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from . import _native
from .extend_utils import check_cameras

MODES = ("depth", "rgb", "rgb+depth")


def render_mesh(vertices, faces, K, poses, h, w, near, far, colors=None, mode="depth", ambient_weight=0.5,
                bg_color=(0.0, 0.0, 0.0)):
    """vertices [nv,3], faces [nf,3] (integer), poses [b,3,4] (R | t, object to OpenCV camera), K [3,3] or [b,3,3]
    and colors [nv,3] in [0, 1] (None: 0.5 grey): CUDA tensors on one device.  near, far: the clip planes
    (0 < near < far); ambient_weight and bg_color[:3] as in the reference's `render`.

    -> depth float32 [b,h,w] ('depth'), rgb uint8 [b,h,w,3] ('rgb') or (rgb, depth) ('rgb+depth'), on the device,
    without a host synchronisation."""
    if mode not in MODES:
        raise ValueError(f"unknown rendering mode {mode!r} (expected one of {MODES})")
    for name, t in (("vertices", vertices), ("faces", faces), ("K", K), ("poses", poses)) + \
            ((("colors", colors),) if colors is not None else ()):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
        if not t.is_cuda:
            raise RuntimeError(f"pvnet_b200: `{name}` must be a CUDA tensor (there is no CPU path)")
    dev = vertices.device
    if vertices.dim() != 2 or vertices.shape[1] != 3:
        raise ValueError(f"vertices must be [nv,3], got {tuple(vertices.shape)}")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must be [nf,3], got {tuple(faces.shape)}")
    if faces.dtype.is_floating_point or faces.dtype.is_complex or faces.dtype == torch.bool:
        raise ValueError(f"faces must hold integer indices, got {faces.dtype}")
    if poses.dim() != 3 or tuple(poses.shape[1:]) != (3, 4):
        raise ValueError(f"poses must be [b,3,4], got {tuple(poses.shape)}")
    b, nv, nf = int(poses.shape[0]), int(vertices.shape[0]), int(faces.shape[0])
    if b < 1:
        raise ValueError("poses holds no pose")
    check_cameras(K.shape, b)
    if colors is not None and tuple(colors.shape) != (nv, 3):
        raise ValueError(f"colors must be [{nv},3], got {tuple(colors.shape)}")
    if any(t.device != dev for t in (faces, K, poses) + ((colors,) if colors is not None else ())):
        raise ValueError("vertices, faces, K, poses and colors must be on one device")
    h, w = int(h), int(w)
    if h < 1 or w < 1:
        raise ValueError(f"image size must be positive, got {h}x{w}")
    near, far = float(near), float(far)
    if not 0 < near < far < float("inf"):
        raise ValueError(f"clip planes must satisfy 0 < near < far, got {near}, {far}")
    bg = [float(v) for v in tuple(bg_color)[:3]]
    if len(bg) != 3:
        raise ValueError(f"bg_color needs three components, got {bg_color!r}")

    v = vertices.contiguous().float()
    # an index beyond int32 is out of range either way; the clamp keeps it so
    f = faces.contiguous() if faces.dtype == torch.int32 else faces.clamp(-1, nv).to(torch.int32).contiguous()
    p = poses.contiguous().float()
    k = K.contiguous().float()
    c = None if colors is None else colors.contiguous().float()
    want_rgb, want_depth = mode != "depth", mode != "rgb"
    depth = torch.empty((b, h, w), dtype=torch.float32, device=dev) if want_depth else None
    rgb = torch.empty((b, h, w, 3), dtype=torch.uint8, device=dev) if want_rgb else None
    L = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(L.pvnet_render_workspace_bytes(b, h, w, ctypes.byref(need)), "pvnet_render_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        _native.check(L.pvnet_render_mesh(
            v.data_ptr() if nv else None, f.data_ptr() if nf else None, None if c is None else c.data_ptr(), nv, nf,
            p.data_ptr(), k.data_ptr(), int(k.dim() == 3), b, h, w, near, far, float(ambient_weight),
            (ctypes.c_float * 3)(*bg), None if depth is None else depth.data_ptr(),
            None if rgb is None else rgb.data_ptr(), ws.data_ptr(), need.value,
            ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "pvnet_render_mesh")
    if mode == "depth":
        return depth
    if mode == "rgb":
        return rgb
    return rgb, depth


def _host_or_device(a):
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(a)))


class MeshSet:
    """M meshes (1 <= M <= 255) with one label each (1..255), packed once into device buffers for
    `render_label_map`: slot m is meshes[m] = (vertices [nv,3], faces [nf,3] with indices into its own vertices),
    numpy arrays or tensors.  A face with an index outside [0, nv) covers nothing, as in `render_mesh`."""

    def __init__(self, meshes, labels, device=None):
        meshes, labels = list(meshes), [int(v) for v in labels]
        M = len(meshes)
        if not 1 <= M <= 255:
            raise ValueError(f"a MeshSet holds 1 to 255 meshes, got {M}")
        if len(labels) != M:
            raise ValueError(f"{M} meshes but {len(labels)} labels")
        if any(not 1 <= v <= 255 for v in labels):
            raise ValueError(f"labels must lie in 1..255 (0 is the background), got {labels}")
        checked, table, vo, fo = [], [], 0, 0
        for m, (v, f) in enumerate(meshes):
            v, f = _host_or_device(v), _host_or_device(f)
            if v.dim() != 2 or v.shape[1] != 3:
                raise ValueError(f"mesh {m}: vertices must be [nv,3], got {tuple(v.shape)}")
            if f.dim() != 2 or f.shape[1] != 3:
                raise ValueError(f"mesh {m}: faces must be [nf,3], got {tuple(f.shape)}")
            if f.dtype.is_floating_point or f.dtype.is_complex or f.dtype == torch.bool:
                raise ValueError(f"mesh {m}: faces must hold integer indices, got {f.dtype}")
            nv, nf = int(v.shape[0]), int(f.shape[0])
            checked.append((v, f, nv))
            table.append((vo, nv, fo, nf))
            vo, fo = vo + nv, fo + nf
        if vo > 2 ** 31 - 1 or fo > 2 ** 31 - 1:
            raise ValueError(f"{vo} vertices and {fo} faces in all: each must fit in int32")
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != "cuda":
            raise RuntimeError("pvnet_b200: a MeshSet lives on a CUDA device (there is no CPU path)")
        verts = [v.to(dev, torch.float32) for v, _, _ in checked]
        # an index beyond int32 is out of range either way; the clamp keeps it so
        faces = [f.to(dev).clamp(-1, nv).to(torch.int32) for _, f, nv in checked]
        self.device, self.labels, self.nf_total = dev, tuple(labels), fo
        self.verts = torch.cat(verts).contiguous()
        self.faces = torch.cat(faces).contiguous()
        self.table = torch.tensor(table, dtype=torch.int32, device=dev)
        self._labels = (ctypes.c_uint8 * M)(*labels)

    def __len__(self):
        return len(self.labels)


def render_label_map(mesh_set, poses, K, h, w, near, far, present=None, depth_divisor=1.0, max_depth=math.inf):
    """The label map of a MeshSet at b images in one depth test.  poses [b,M,3,4] (slot m's R | t in image i), K
    [3,3] or [b,3,3] and present [b,M] (nonzero: the slot is in the image; None: all are): CUDA tensors on the
    MeshSet's device.  near, far: the clip planes (0 < near < far).

    A slot's depth at a pixel is `render_mesh`'s depth of its mesh alone, divided by depth_divisor in fp32 (one IEEE
    division).  -> (label uint8 [b,h,w], depth float32 [b,h,w]): the label of the slot with the smallest depth
    strictly below max_depth, ties to the lower slot, and that depth; 0 and max_depth where there is none.  On the
    device, without a host synchronisation."""
    if not isinstance(mesh_set, MeshSet):
        raise ValueError(f"mesh_set must be a MeshSet, got {type(mesh_set).__name__}")
    dev, M = mesh_set.device, len(mesh_set)
    for name, t in (("poses", poses), ("K", K)) + ((("present", present),) if present is not None else ()):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a torch tensor, got {type(t).__name__}")
        if not t.is_cuda:
            raise RuntimeError(f"pvnet_b200: `{name}` must be a CUDA tensor (there is no CPU path)")
        if t.device != dev:
            raise ValueError(f"{name} is on {t.device}, the MeshSet on {dev}")
    if poses.dim() != 4 or tuple(poses.shape[1:]) != (M, 3, 4):
        raise ValueError(f"poses must be [b,{M},3,4], got {tuple(poses.shape)}")
    b = int(poses.shape[0])
    if b < 1:
        raise ValueError("poses holds no image")
    check_cameras(K.shape, b)
    if present is not None and tuple(present.shape) != (b, M):
        raise ValueError(f"present must be [{b},{M}], got {tuple(present.shape)}")
    h, w = int(h), int(w)
    if h < 1 or w < 1:
        raise ValueError(f"image size must be positive, got {h}x{w}")
    near, far = float(near), float(far)
    if not 0 < near < far < math.inf:
        raise ValueError(f"clip planes must satisfy 0 < near < far, got {near}, {far}")
    depth_divisor, max_depth = float(depth_divisor), float(max_depth)
    if not 0 < depth_divisor < math.inf:
        raise ValueError(f"depth_divisor must be positive and finite, got {depth_divisor}")
    if not np.float32(near) / np.float32(depth_divisor) > 0:
        raise ValueError(f"near / depth_divisor ({near} / {depth_divisor}) underflows to 0 in float32")
    if not max_depth > 0:
        raise ValueError(f"max_depth must be positive (inf allowed), got {max_depth}")

    p = poses.contiguous().float()
    k = K.contiguous().float()
    pr = None if present is None else (present != 0).to(torch.uint8).contiguous()
    label = torch.empty((b, h, w), dtype=torch.uint8, device=dev)
    depth = torch.empty((b, h, w), dtype=torch.float32, device=dev)
    L = _native.lib()
    with torch.cuda.device(dev):
        need = ctypes.c_size_t()
        _native.check(L.pvnet_render_workspace_bytes(b, h, w, ctypes.byref(need)), "pvnet_render_workspace_bytes")
        ws = torch.empty(need.value, dtype=torch.uint8, device=dev)
        nf = mesh_set.nf_total
        _native.check(L.pvnet_render_label_map(
            mesh_set.verts.data_ptr() if nf else None, mesh_set.faces.data_ptr() if nf else None,
            mesh_set.table.data_ptr(), mesh_set._labels, M, nf, p.data_ptr(), None if pr is None else pr.data_ptr(),
            k.data_ptr(), int(k.dim() == 3), b, h, w, near, far, depth_divisor, max_depth, label.data_ptr(),
            depth.data_ptr(), ws.data_ptr(), need.value,
            ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "pvnet_render_label_map")
    return label, depth


# What the reference's get_mask_of_all_objects renders with (data_utils.py:788-826 through OpenGLRenderer.render,
# render_utils.py:510-524): LINEMOD's camera at 640x480, clip planes 10 and 10 000 mm, depth in metres, and a
# depth map that starts at 10.
OCCLUSION_SIZE = (480, 640)
OCCLUSION_CLIP = (10.0, 10000.0)
OCCLUSION_DEPTH_DIVISOR = 1000.0
OCCLUSION_MAX_DEPTH = 10.0
_mesh_cache = []                                  # [(models, labels, device, MeshSet)]: the last one built


def _occlusion_mesh_set(models, labels, dev):
    """The MeshSet of the db's models, packed again only when load_ply returns other arrays."""
    if _mesh_cache:
        cm, cl, cd, ms = _mesh_cache[0]
        if cl == labels and cd == dev and len(cm) == len(models) and \
                all(a["pts"] is b["pts"] and a["faces"] is b["faces"] for a, b in zip(cm, models)):
            return ms
    ms = MeshSet([(np.asarray(m["pts"]), np.asarray(m["faces"]).reshape(-1, 3).astype(np.int64)) for m in models],
                 labels, device=dev)
    _mesh_cache[:] = [(list(models), labels, dev, ms)]
    return ms


def occlusion_poses(db, indices):
    """The poses get_mask_of_all_objects renders, per image and class in `class_type_to_number` order -> poses f32
    [n,M,3,4] (R | t in mm) and present u8 [n,M].  `db.class_type` is set before each `db.read_blender_pose(index)`;
    an empty pose is absent.  As in OpenGLRenderer.render (render_utils.py:519-520), R = pose[:, :3] and
    t = pose[:, 3:] * 1000. are computed in the pose's own dtype, then stored as fp32."""
    classes = list(db.class_type_to_number.keys())
    P = np.zeros((len(indices), len(classes), 3, 4), np.float32)
    present = np.zeros((len(indices), len(classes)), np.uint8)
    for j, index in enumerate(indices):
        for m, c in enumerate(classes):
            db.class_type = c
            pose = db.read_blender_pose(index)
            if len(pose) == 0:
                continue
            pose = np.asarray(pose)
            P[j, m, :, :3] = pose[:, :3]
            P[j, m, :, 3:] = pose[:, 3:] * 1000.
            present[j, m] = 1
    return P, present


def masks_of_all_objects(db, indices, chunk=64):
    """The reference's Occlusion-LINEMOD label maps for a batch of image indices: db is its `OcclusionLineModDB` or
    `OcclusionLineModDBSyn` (duck-typed: `class_type_to_number`, `read_blender_pose`, `opengl_renderer` with
    `load_ply` and `intrinsic_matrix['linemod']`).  -> uint8 [n,480,640] (numpy), image j the map
    `get_mask_of_all_objects(indices[j])` returns, from one device call per `chunk` images.

    As the reference does, `db.class_type` is set to each class before `db.read_blender_pose(index)` (it ends on the
    last class), an empty pose leaves the object out, and each model drawn has `model['colors']` divided by 255 in
    place when its maximum is above 1.  The meshes are uploaded once and reused while `load_ply` returns the same
    arrays; a model's arrays must not be changed in place after that."""
    indices = list(indices)
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError(f"chunk must be positive, got {chunk}")
    classes = list(db.class_type_to_number.keys())
    labels = [int(db.class_type_to_number[c]) for c in classes]
    renderer = db.opengl_renderer
    if not torch.cuda.is_available():
        raise RuntimeError("pvnet_b200: masks_of_all_objects needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    models = [renderer.load_ply(c) for c in classes]
    mesh_set = _occlusion_mesh_set(models, labels, dev)
    K = torch.from_numpy(np.asarray(renderer.intrinsic_matrix["linemod"], np.float64).reshape(3, 3)
                         .astype(np.float32)).to(dev)
    h, w = OCCLUSION_SIZE
    out = np.empty((len(indices), h, w), np.uint8)
    drawn = np.zeros(len(classes), bool)
    for c0 in range(0, len(indices), chunk):
        idx = indices[c0:c0 + chunk]
        P, present = occlusion_poses(db, idx)
        drawn |= present.any(0)
        label, _ = render_label_map(mesh_set, torch.from_numpy(P).to(dev), K, h, w, *OCCLUSION_CLIP,
                                    present=torch.from_numpy(present).to(dev),
                                    depth_divisor=OCCLUSION_DEPTH_DIVISOR, max_depth=OCCLUSION_MAX_DEPTH)
        out[c0:c0 + len(idx)] = label.cpu().numpy()
    for m in np.flatnonzero(drawn):
        model = models[m]
        if "colors" in model.keys() and model["colors"].max() > 1.0:
            model["colors"] /= 255.0
    return out


def get_mask_of_all_objects(self, index):
    """`OcclusionLineModDB.get_mask_of_all_objects` on the device: uint8 [480,640], the reference's label map of image
    `index`.  Bound as `OcclusionLineModDB.get_mask_of_all_objects = pvnet_b200.render.get_mask_of_all_objects`, it
    serves the reference's unchanged `get_mask`, `get_masks` and `run.py --type gen_mask`."""
    return masks_of_all_objects(self, [index])[0]
