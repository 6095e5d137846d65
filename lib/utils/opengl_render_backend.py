"""`lib.utils.opengl_render_backend` with the reference module's `render`, served by `pvnet_b200.render.render_mesh`
(csrc/render.cu, DESIGN.md §24) instead of an OpenGL context, so `OpenGLRenderer.render` and
`OcclusionLineModDB.get_mask_of_all_objects` run on a headless GPU server.

Depth and flat-shaded RGB follow the reference's conventions: pixel (r, c) samples the OpenCV image point
(c + 0.5, r + 0.5), depth is the camera-space Z (0 where no face covers the pixel) and the light sits at the camera.
Textures and Phong shading are not provided and raise ValueError, as does an unknown mode (where the reference
prints and exits).  Importing this module loads neither glumpy nor cv2."""
import numpy as np
import torch

from pvnet_b200.render import MODES, render_mesh

__all__ = ["render"]


def render(model, im_size, K, R, t, clip_near=100, clip_far=2000,
           texture=None, surf_color=None, bg_color=(0.0, 0.0, 0.0, 0.0),
           ambient_weight=0.5, shading='flat', mode='rgb+depth'):
    """model: {'pts' [nv,3], 'faces' [nf,3], optionally 'colors' [nv,3]}; im_size [w, h]; K [3,3]; R [3,3]; t [3,1]
    or [3] -> float32 depth [h,w] ('depth'), uint8 rgb [h,w,3] ('rgb') or (rgb, depth) ('rgb+depth'), numpy.

    As in the reference (opengl_render_backend.py:315-333), model['colors'] with a maximum above 1 is divided by 255
    in place, in every mode; a caller that keeps the model (OpenGLRenderer does) sees the divided colours from then on."""
    assert {'pts', 'faces'}.issubset(set(model.keys()))
    if texture is not None:
        raise ValueError("render: textures are not supported (flat vertex colours only)")
    if shading != 'flat':
        raise ValueError(f"render: shading {shading!r} is not supported (only 'flat')")
    if mode not in MODES:
        raise ValueError(f"render: unknown rendering mode {mode!r} (expected one of {MODES})")

    nv = model['pts'].shape[0]
    if not surf_color:
        if 'colors' in model.keys():
            assert (model['pts'].shape[0] == model['colors'].shape[0])
            colors = model['colors']
            if colors.max() > 1.0:
                colors /= 255.0  # Color values are expected in range [0, 1]
        else:
            colors = None        # 0.5 grey
    else:
        colors = np.tile(np.asarray(list(surf_color)[:3], np.float32), [nv, 1])

    if not torch.cuda.is_available():
        raise RuntimeError("pvnet_b200: render needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    w, h = int(im_size[0]), int(im_size[1])
    pose = np.zeros((1, 3, 4), np.float32)
    pose[0, :, :3] = np.asarray(R, np.float32).reshape(3, 3)
    pose[0, :, 3] = np.asarray(t, np.float32).reshape(3)

    def dev_tensor(a, dtype):
        return torch.as_tensor(np.ascontiguousarray(a, dtype), device=dev)

    faces = np.asarray(model['faces']).reshape(-1, 3).astype(np.int64)
    out = render_mesh(dev_tensor(model['pts'], np.float32), dev_tensor(faces, np.int64),
                      dev_tensor(np.asarray(K, np.float64).reshape(3, 3), np.float32), dev_tensor(pose, np.float32),
                      h, w, clip_near, clip_far,
                      colors=None if colors is None else dev_tensor(np.asarray(colors)[:, :3], np.float32),
                      mode=mode, ambient_weight=ambient_weight, bg_color=tuple(bg_color)[:3])
    if mode != 'rgb+depth':
        return out[0].cpu().numpy()
    return out[0][0].cpu().numpy(), out[1][0].cpu().numpy()
