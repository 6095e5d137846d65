"""Mesh rendering on the device: depth and flat-shaded RGB of one mesh at a batch of poses, over `pvnet_render_mesh`
(csrc/render.cu).  The conventions are those of the reference's OpenGL backend (lib/utils/opengl_render_backend.py
`render`, DESIGN.md §24): pixel (r, c) samples the OpenCV image point (c + 0.5, r + 0.5), depth is the camera-space
Z of the nearest face (0 where none), and RGB is the flat-shaded vertex colour with the light at the camera.
oracle/render_oracle.py restates it bit for bit.  No CPU path: without the library or a CUDA device it raises."""
from __future__ import annotations

import ctypes

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
