"""numpy restatement of the keypoint vertex targets (pvnet_vertex_targets, csrc/losses.cu; DESIGN.md §12): the
ground-truth vertex field of the reference's loader, as float32 [b,2K,h,w].

Every step is one correctly rounded fp64 numpy operation in the kernel's order, so the result is bit-identical:
    vx = hx - x*hw, vy = hy - y*hw; unless use_motion: n = sqrt(vx*vx + vy*vy), n < 1e-3 -> n + 1e-3, v = v / n;
    channel 2k = float32(vx), channel 2k+1 = float32(vy) where mask == 1, +0 elsewhere.
"""
import numpy as np


def vertex_targets(mask, hcoords, use_motion=False):
    """mask [b,h,w] (any integer or bool dtype), hcoords [b,K,3] -> float32 [b,2K,h,w]."""
    mask = np.asarray(mask)
    hc = np.asarray(hcoords).astype(np.float64)
    b, h, w = mask.shape
    K = hc.shape[1]
    out = np.zeros((b, 2 * K, h, w), np.float32)
    with np.errstate(all="ignore"):
        for i in range(b):
            ys, xs = np.nonzero(mask[i] == 1)
            x = xs.astype(np.float64)[:, None]                # [n,1] against the K keypoints
            y = ys.astype(np.float64)[:, None]
            hx, hy, hw = hc[i, :, 0][None], hc[i, :, 1][None], hc[i, :, 2][None]
            vx = hx - x * hw
            vy = hy - y * hw
            if not use_motion:
                n = np.sqrt(vx * vx + vy * vy)
                n = np.where(n < 1e-3, n + 1e-3, n)
                vx = vx / n
                vy = vy / n
            ox, oy = out[i, 0::2], out[i, 1::2]                 # views [K,h,w]
            ox[:, ys, xs] = vx.T.astype(np.float32)
            oy[:, ys, xs] = vy.T.astype(np.float32)
    return out
