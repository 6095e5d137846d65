"""CPU oracle for the validation losses -- TEST INFRASTRUCTURE ONLY.

A numpy restatement of what `pvnet_seg_vertex_losses` (pvnet_b200/csrc/losses.cu) computes, written from the
semantics of the reference's smooth_l1_loss / compute_precision_recall (lib/utils/net_utils.py:54-80, 329-348) and
of nn.CrossEntropyLoss with its default ignore_index -100:

  - the elementwise smooth-L1 in fp32, one numpy operation per torch operation (numpy rounds each float32 operation
    once and never fuses), so it is bit-equal to the kernel and to torch;
  - the cross-entropy per pixel in fp64 from the fp32 logits (log-sum-exp minus the target logit);
  - the precision / recall counts exactly in int64;
  - every sum in fp64, then the final fp32 operations in the reference's order.
"""
from __future__ import annotations

import numpy as np

IGNORE_INDEX = -100
F32 = np.float32


def smooth_l1_constants(sigma):
    """c1 = 1/sigma^2, c2 = sigma^2/2, c3 = 0.5/sigma^2: derived in double as Python does, rounded to float32 as
    they reach torch's fp32 kernels."""
    s2 = float(sigma) ** 2
    return F32(1.0 / s2), F32(s2 / 2.0), F32(0.5 / s2)


def smooth_l1_elementwise(pred, tgt, weights, sigma=1.0):
    """pred, tgt float32 [b,vd,h,w], weights float32 [b,1,h,w] -> float32 [b,vd,h,w]."""
    c1, c2, c3 = smooth_l1_constants(sigma)
    pred, tgt, weights = (np.asarray(a, F32) for a in (pred, tgt, weights))
    with np.errstate(all="ignore"):
        diff = weights * (pred - tgt)
        ad = np.abs(diff)
        s = (ad < c1).astype(F32)
        return ((diff * diff) * c2) * s + (ad - c3) * (F32(1) - s)


def smooth_l1_normalized(pred, tgt, weights, sigma=1.0):
    """sum(in) / (ver_dim * sum(w) + 1e-3) per image: fp64 sums, fp32 final ops -> float32 [b]."""
    b, vd = np.shape(pred)[:2]
    el = smooth_l1_elementwise(pred, tgt, weights, sigma)
    s_in = el.reshape(b, -1).astype(np.float64).sum(1).astype(F32)
    s_w = np.asarray(weights, F32).reshape(b, -1).astype(np.float64).sum(1).astype(F32)
    with np.errstate(all="ignore"):
        return s_in / (F32(vd) * s_w + F32(1e-3))


def cross_entropy(seg, mask):
    """Per-image mean over all pixels of -log_softmax(seg)[target]: seg float32 [b,C,h,w], mask integer [b,h,w] ->
    float32 [b].  Target -100 adds 0 (and counts); an image with any other target outside [0,C) gives NaN."""
    x = np.asarray(seg, F32).astype(np.float64)
    t = np.asarray(mask).astype(np.int64)
    b, C = x.shape[:2]
    with np.errstate(all="ignore"):
        m = x.max(1, keepdims=True)
        lse = (m + np.log(np.exp(x - m).sum(1, keepdims=True)))[:, 0]
        xt = np.take_along_axis(x, np.clip(t, 0, C - 1)[:, None], 1)[:, 0]
        valid = (t >= 0) & (t < C)
        term = np.where(valid, lse - xt, 0.0)
        out = term.reshape(b, -1).sum(1) / term[0].size
    bad = (~valid & (t != IGNORE_INDEX)).reshape(b, -1).any(1)
    out[bad] = np.nan
    return out.astype(F32)


def argmax(seg):
    """torch.argmax over dim 1 as on CUDA: the first maximum; a NaN wins, the first NaN when there are several."""
    seg = np.asarray(seg, F32)
    nan = np.isnan(seg)
    with np.errstate(all="ignore"):
        first_max = np.argmax(np.where(nan, -np.inf, seg), 1)
    return np.where(nan.any(1), np.argmax(nan, 1), first_max).astype(np.int64)


def precision_recall_counts(seg, mask):
    """Exact tp, fp, fn int64 [b] of compute_precision_recall's float arithmetic (p = argmax, t = target)."""
    b = np.shape(seg)[0]
    p = argmax(seg).reshape(b, -1)
    t = np.asarray(mask).astype(np.int64).reshape(b, -1)
    return (p * t).sum(1), (p * (1 - t)).sum(1), ((1 - p) * t).sum(1)


def precision_recall(seg, mask):
    """(tp+1)/(tp+fp+1), (tp+1)/(tp+fn+1) in fp32 from the exact counts -> float32 [b] each."""
    tp, fp, fn = (c.astype(F32) for c in precision_recall_counts(seg, mask))
    num = tp + F32(1)
    return num / ((tp + fp) + F32(1)), num / ((tp + fn) + F32(1))
