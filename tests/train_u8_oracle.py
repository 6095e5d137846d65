"""numpy restatement of the uint8 training input (DESIGN.md §18) -- TEST INFRASTRUCTURE ONLY.

  normalise: torchvision's ToTensor + Normalize as the loader runs them on the CPU, (float(u) / 255 - mean) / std,
    three correctly rounded fp32 operations (numpy rounds each float32 operation once);
  pack_u8: what pvnet_stem_s2d_nhwc's pack writes for a uint8 image -- S, the 2x2 space-to-depth image (channel
    (py*2+px)*3+c, TF32-rounded, 4 zero channels), and, in a caller's channels_last buffer, the normalised image
    unrounded at channels [co, co+3) and zeros at [co+3, co+8), every other channel left as it was;
  mask_weights: the loader's vertex_weights, mask.unsqueeze(0).float() per image (linemod_dataset.py:227).
"""
from __future__ import annotations

import numpy as np

from pvnet_b200.pipeline import IMAGENET_MEAN, IMAGENET_STD  # noqa: F401  (re-exported for the tests)

F32 = np.float32


def normalise(img, mean, std):
    """uint8 [b,H,W,3] -> float32 [b,3,H,W]."""
    x = np.ascontiguousarray(np.asarray(img).transpose(0, 3, 1, 2)).astype(F32) / F32(255)
    return (x - np.asarray(mean, F32).reshape(1, 3, 1, 1)) / np.asarray(std, F32).reshape(1, 3, 1, 1)


def round_tf32(a):
    """Nearest TF32 value, ties away from zero (cvt.rna), kept in float32."""
    i = np.ascontiguousarray(a, F32).view(np.uint32)
    return ((i + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(F32)


def pack_u8(img, mean, std, buf, co):
    """-> (S float32 [b,H/2,W/2,16], buf): buf float32 [b,H,W,cs] is written at channels [co, co+8) and returned."""
    x = normalise(img, mean, std)
    b, _, H, W = x.shape
    xr = round_tf32(x)
    S = np.zeros((b, H // 2, W // 2, 16), F32)
    for py in range(2):
        for px in range(2):
            S[..., (py * 2 + px) * 3:(py * 2 + px) * 3 + 3] = xr[:, :, py::2, px::2].transpose(0, 2, 3, 1)
    buf[..., co:co + 3] = x.transpose(0, 2, 3, 1)
    buf[..., co + 3:co + 8] = 0
    return S, buf


def mask_weights(mask):
    """mask [b,h,w] (int64, int32, uint8 or bool) -> float32 [b,1,h,w], each value converted to the nearest float."""
    return np.asarray(mask).astype(F32)[:, None]
