"""CPU restatement of the voting layer's device-side sampler (``rng="device"``) -- TEST INFRASTRUCTURE ONLY.

numpy, no torch.  Written from the sampler's specification (include/pvnet_b200.h, DESIGN.md section 3),
not from the CUDA source, so that a test comparing the two holds the kernels to that specification:

  generator  Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11), multipliers 0xD2511F53 / 0xCD9E8D57,
             key increments 0x9E3779B9 / 0xBB67AE85
  key        (seed & 0xffffffff, seed >> 32); seed = torch.initial_seed() & (2^63 - 1)
  counter    (item, image | stream << 28, offset & 0xffffffff, offset >> 32)
  stream 0   selection: item = y*w + x; sel = (x & 0xffffff) * 2^-24; a foreground pixel of an image with
             fg > max_num is kept iff sel < subsample_probability(max_num, fg)
  stream 1   v3 samples: item = h*vn + k (h < hn); the pair is (x, y) % tn into the row-major list of kept pixels
  stream 2   covariance samples: as stream 1, h < cov_round_hyp_num * rounds
  tn == 0    (an image below min_num, or every pixel dropped by the subsampling): nothing is drawn

One call draws all three streams at the call's {seed, offset}; the call then advances the offset by one.
"""
from __future__ import annotations

import numpy as np

from . import pvnet_oracle as po

PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85
STREAM_SELECTION, STREAM_V3, STREAM_COV = 0, 1, 2
_M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """Philox4x32-10 on broadcastable arrays: counter [..., 4], key [..., 2] (32-bit words) -> uint32 [..., 4].
    Every word is carried in uint64, so each 32x32-bit product is exact."""
    counter = np.asarray(counter, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    c0, c1, c2, c3 = (counter[..., i] & _M32 for i in range(4))
    k0, k1 = key[..., 0] & _M32, key[..., 1] & _M32
    m0, m1 = np.uint64(PHILOX_M0), np.uint64(PHILOX_M1)
    w0, w1 = np.uint64(PHILOX_W0), np.uint64(PHILOX_W1)
    for r in range(10):
        if r:                                     # the key schedule advances between rounds
            k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
    return np.stack(np.broadcast_arrays(c0, c1, c2, c3), -1).astype(np.uint32)


def draw(seed, offset, image, stream, items):
    """The four 32-bit words the sampler draws for `items` (int array) of `image` in `stream` at {seed, offset}."""
    seed, offset = int(seed), int(offset)
    items = np.asarray(items, dtype=np.uint64)
    ctr = np.zeros(items.shape + (4,), np.uint64)
    ctr[..., 0] = items
    ctr[..., 1] = np.asarray(image, dtype=np.uint64) | np.uint64(stream << 28)
    ctr[..., 2] = offset & 0xFFFFFFFF
    ctr[..., 3] = (offset >> 32) & 0xFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint64)
    return philox4x32_10(ctr, key)


def selection_values(seed, offset, image, npx):
    """float32 [npx]: the uniform value of every pixel of `image` (24 random bits times 2^-24, exact)."""
    x = draw(seed, offset, image, STREAM_SELECTION, np.arange(npx))[..., 0]
    return (x & np.uint32(0xFFFFFF)).astype(np.float32) * np.float32(2.0 ** -24)


def foreground(mask_img, mode):
    """The foreground of one image: "nonzero" = `.byte()` nonzero (v3's reading), "equals_one" = value == 1."""
    if mode == "nonzero":
        return po._byte_mask(mask_img) != 0
    if mode == "equals_one":
        return np.asarray(mask_img) == 1
    raise ValueError(f"unknown mask mode {mode!r}")


def _pairs(seed, offset, image, stream, nh, vn):
    """int32 [nh, vn, 2]: words x, y of items h*vn + k, as the int32 bit patterns the injection path takes."""
    r = draw(seed, offset, image, stream, np.arange(nh * vn))
    return r[:, :2].reshape(nh, vn, 2).view(np.int32)


def device_samples(mask, mode, seed, offset, hn, vn, cov_hn_total, min_num, max_num):
    """What one `rng="device"` call at {seed, offset} draws for mask [b,h,w] read with `mode`.

    Returns a dict of
      idxs       int32 [b, hn, vn, 2]: the raw 32-bit words (zeros where the image has tn == 0)
      cov_idxs   int32 [b, cov_hn_total, vn, 2], or None when cov_hn_total == 0
      selection  float32 [b, h, w]: the uniform field of every pixel (consulted only where fg > max_num)
      tn         int32 [b]: kept pixels per image
    Fed back as injected idxs / cov_idxs / selection, these reproduce the device draw; the kernels reduce
    the words modulo tn themselves (see `reduce` for the CPU oracle's form)."""
    mask = np.asarray(mask)
    b, h, w = mask.shape
    npx = h * w
    idxs = np.zeros((b, hn, vn, 2), np.int32)
    cov_idxs = np.zeros((b, cov_hn_total, vn, 2), np.int32) if cov_hn_total else None
    selection = np.empty((b, h, w), np.float32)
    tn = np.zeros(b, np.int32)
    for bi in range(b):
        sel = selection_values(seed, offset, bi, npx).reshape(h, w)
        selection[bi] = sel
        fg_mask = foreground(mask[bi], mode)
        fg = int(fg_mask.sum())
        if fg < min_num:
            continue
        if fg > max_num:
            fg_mask = fg_mask & (sel < po.subsample_probability(max_num, fg))
        tn[bi] = int(fg_mask.sum())
        if tn[bi] == 0:
            continue
        idxs[bi] = _pairs(seed, offset, bi, STREAM_V3, hn, vn)
        if cov_hn_total:
            cov_idxs[bi] = _pairs(seed, offset, bi, STREAM_COV, cov_hn_total, vn)
    return dict(idxs=idxs, cov_idxs=cov_idxs, selection=selection, tn=tn)


def reduce(idxs, tn):
    """Raw words [b, n, vn, 2] -> per-image int32 indices into the kept-pixel list, `(unsigned)word % tn`
    (the form pvnet_oracle's layers take); None for an image with tn == 0."""
    words = np.asarray(idxs, np.int32).view(np.uint32)
    return [None if int(t) == 0 else (words[i] % np.uint32(t)).astype(np.int32) for i, t in enumerate(tn)]
