"""CPU oracle for the training losses' gradients -- TEST INFRASTRUCTURE ONLY.

numpy restatements of what `pvnet_seg_vertex_losses[_keypoints]_backward` (pvnet_b200/csrc/losses.cu, DESIGN.md
§13) computes: the sequences torch's CUDA autograd runs through the reference's smooth_l1_loss (lib/utils/
net_utils.py:54-80, torch.pow(diff, 2), normalize=True) and through nn.CrossEntropyLoss(reduction='none') followed
by the per-image mean (tools/train_linemod.py:83,87-88).  The forward's restatement is oracle/loss_oracle.py.
"""
from __future__ import annotations

import numpy as np

from oracle.loss_oracle import F32, IGNORE_INDEX, smooth_l1_constants


def vertex_denominator(weights, ver_dim):
    """ver_dim * sum(w) + 1e-3 per image as the forward computes it: the fp64 sum rounded to fp32, then fp32 ops."""
    b = np.shape(weights)[0]
    s_w = np.asarray(weights, F32).reshape(b, -1).astype(np.float64).sum(1).astype(F32)
    return F32(ver_dim) * s_w + F32(1e-3)


def smooth_l1_grad(pred, tgt, weights, grad_loss_vertex, sigma=1.0, den=None):
    """d loss_vertex / d pred of the normalised smooth-L1 (net_utils.py:54-80 with torch.pow(diff, 2)), one fp32
    numpy operation per operation torch's autograd runs, in its order:
        gi = gv / den                                 DivBackward0 (tensor / tensor)
        diff = w * (p - t), s = |diff| < c1
        A = ((gi * s) * c2) * (2 * diff)              MulBackward0 (* s), MulBackward1 (* c2), PowBackward0
        B = (gi * (1 - s)) * sgn(diff)                MulBackward0 (* (1 - s)), SubBackward1, AbsBackward0
        grad = (A + B) * w                            PowBackward0 runs before AbsBackward0: B is added to A;
                                                      MulBackward0 (w *), SubBackward0
    sgn is torch.sign: 0 for +-0 and NaN.  den defaults to the forward's (vertex_denominator); pass torch's own
    fp32 denominator to restate torch's sequence where its fp32 sum of the weights is not exact.
    pred, tgt float32 [b,vd,h,w], weights float32 [b,1,h,w], grad_loss_vertex float32 [b] -> float32 [b,vd,h,w]."""
    c1, c2, _ = smooth_l1_constants(sigma)
    pred, tgt, weights = (np.asarray(a, F32) for a in (pred, tgt, weights))
    b, vd = pred.shape[:2]
    if den is None:
        den = vertex_denominator(weights, vd)
    with np.errstate(all="ignore"):
        gi = (np.asarray(grad_loss_vertex, F32) / np.asarray(den, F32))[:, None, None, None]
        diff = weights * (pred - tgt)
        s = (np.abs(diff) < c1).astype(F32)
        sgn = np.where(diff > 0, F32(1), np.where(diff < 0, F32(-1), F32(0)))
        a = ((gi * s) * c2) * (F32(2) * diff)
        bb = (gi * (F32(1) - s)) * sgn
        return (a + bb) * weights


def cross_entropy_grad(seg, mask, grad_loss_seg):
    """d loss_seg / d seg of the per-image mean cross-entropy, from the fp32 logits in fp32 as torch's CUDA autograd
    computes it: g = gs * (1 / N) (MeanBackward as ATen runs a CUDA tensor divided by a scalar), lp = (x - m) -
    log(s) as the forward, S = 0 + sum_c gO_c with gO_t = -g at the target, grad_c = fma(-exp(lp_c), S, gO_c) (the
    product exact in fp64, then one fp64 addition and the rounding to fp32, which can differ from a single rounding
    in rare halfway cases).  Target -100 gives gO = 0; an image with any other target outside [0,C) is all NaN.
    seg float32 [b,C,h,w], mask integer [b,h,w], grad_loss_seg float32 [b] -> float32 [b,C,h,w]."""
    x = np.asarray(seg, F32)
    t = np.asarray(mask).astype(np.int64)
    b, C, h, w = x.shape
    with np.errstate(all="ignore"):
        g = (np.asarray(grad_loss_seg, F32) * (F32(1) / F32(h * w)))[:, None, None]
        m = np.fmax.reduce(x, axis=1)
        s = np.zeros((b, h, w), F32)
        for c in range(C):
            s = s + np.exp(x[:, c] - m)
        lp = (x - m[:, None]) - np.log(s)[:, None]
        valid = (t >= 0) & (t < C)
        go = np.where((np.arange(C)[None, :, None, None] == t[:, None]) & valid[:, None], -g[:, None], F32(0))
        S = np.where(valid, F32(0) + (-g), F32(0))
        e = np.exp(lp)
        out = (-e.astype(np.float64) * S[:, None].astype(np.float64) + go.astype(np.float64)).astype(F32)
    bad = (~valid & (t != IGNORE_INDEX)).reshape(b, -1).any(1)
    out[bad] = np.nan
    return out
