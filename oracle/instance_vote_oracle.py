"""CPU restatement of `pvnet_ransac_voting_center` (DESIGN.md section 29) -- TEST INFRASTRUCTURE ONLY.

numpy/fp64 on the v3 oracle pieces of `pvnet_oracle`: `compact`, `generate_hypothesis_kernel`, `vote_counts`,
`voting_for_hypothesis_kernel` and `refit`.  The instance assignment needs the reference's cosine value `ang`
bit for bit; numpy has every correctly rounded fp32 operation it uses except fmaf, so `fmaf` below restates
that one exactly in fp64 (the product of two floats is exact in fp64; the sum's rounding error is recovered
with TwoSum and breaks the one case where rounding to fp32 twice could differ, an fp64 sum that lies exactly
half-way between two floats).

Device samples (rng="device"): Philox4x32-10 as `philox_oracle` states it, stream 3, item i*hn + m of image b
for round i; the two words are the pair before the reduction modulo |R_i|.
"""
from __future__ import annotations

import numpy as np

from . import philox_oracle as px
from . import pvnet_oracle as po

STREAM_CENTER = 3
_F32 = np.float32


def fmaf(a, b, c):
    """float32 fma(a, b, c), correctly rounded once, on broadcastable float32 arrays."""
    a, b, c = (np.asarray(v, _F32).astype(np.float64) for v in (a, b, c))
    p = a * b                                       # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                 # TwoSum: s + err == p + c exactly
    bits = s.view(np.uint64)
    half = (bits & np.uint64((1 << 29) - 1)) == np.uint64(1 << 28)    # s half-way between two floats
    fix = half & (err != 0)
    s = np.where(fix, np.nextafter(s, np.copysign(np.inf, err)), s)
    return s.astype(_F32)


def exact_cosine(nx, ny, cx, cy, hx, hy):
    """(valid, ang): the reference's inlier test (ransac_voting_kernel.cu:107-125) up to its comparison;
    valid is False where the norm test rejects the pair."""
    nx, ny, cx, cy, hx, hy = (np.asarray(v, _F32) for v in (nx, ny, cx, cy, hx, hy))
    dx = (hx - cx).astype(_F32)
    dy = (hy - cy).astype(_F32)
    norm1 = np.sqrt(fmaf(nx, nx, (ny * ny).astype(_F32)))
    norm2 = np.sqrt(fmaf(dx, dx, (dy * dy).astype(_F32)))
    valid = ~((norm1.astype(np.float64) < 1e-6) | (norm2.astype(np.float64) < 1e-6))
    num = fmaf(dx, nx, (dy * ny).astype(_F32))
    den = (norm1 * norm2).astype(_F32)
    with np.errstate(all="ignore"):
        ang = (num / den).astype(_F32)
    return valid, ang


def device_center_idxs(seed, offset, b, max_instances, hn):
    """int32 [b, I, hn, 2]: the raw words an rng="device" call at {seed, offset} draws (fed back as idxs,
    they reproduce the call)."""
    out = np.empty((b, max_instances, hn, 2), np.int32)
    for bi in range(b):
        r = px.draw(seed, offset, bi, STREAM_CENTER, np.arange(max_instances * hn))
        out[bi] = r[:, :2].reshape(max_instances, hn, 2).view(np.int32)
    return out


def assign(mask_img, field_img, centers, num, thresh):
    """int32 [h,w]: 1 + argmax_j ang over the centres j < num the pixel is an inlier of (lowest j on ties),
    0 for background and for pixels that are inliers of none."""
    fg = po._byte_mask(mask_img) != 0
    ys, xs = np.nonzero(fg)
    field = np.asarray(field_img, _F32)
    nx, ny = field[ys, xs, 0], field[ys, xs, 1]
    best = np.zeros(ys.shape, _F32)
    label = np.zeros(ys.shape, np.int32)
    for j in range(int(num)):
        valid, ang = exact_cosine(nx, ny, xs.astype(_F32), ys.astype(_F32), centers[j, 0], centers[j, 1])
        take = valid & (ang > _F32(thresh)) & ((label == 0) | (ang > best))
        best = np.where(take, ang, best)
        label = np.where(take, j + 1, label)
    out = np.zeros(fg.shape, np.int32)
    out[ys, xs] = label
    return out


def center_search(mask_img, field_img, idxs, thresh, min_num, centers_for_assign=None):
    """One image.  mask_img [h,w]; field_img [h,w,2] f32; idxs int32 [I,hn,2] raw words.

    Returns a dict of num, centers [I,2] f32 (zeros beyond num), labels [h,w] int32 and the per-round
    counts [I,hn], hyp [I,hn,2], tn [I], win_counts [I], win_idx [I] and inliers (the list of S_i as
    indices into R_0).  `centers_for_assign` assigns with other centres (the kernel's own) instead."""
    idxs = np.asarray(idxs, np.int32)
    I, hn, _ = idxs.shape
    field = np.asarray(field_img, _F32)
    coords, direct = po.compact(po._byte_mask(mask_img), field[:, :, None, :])   # R_0, row-major
    alive = np.arange(coords.shape[0])             # R_i as indices into R_0
    out = dict(counts=np.zeros((I, hn), np.int32), hyp=np.zeros((I, hn, 2), _F32), tn=np.zeros(I, np.int32),
               win_counts=np.zeros(I, np.int32), win_idx=np.full(I, -1), centers=np.zeros((I, 2), _F32),
               inliers=[], num=0)
    for i in range(I):
        t = alive.size
        out["tn"][i] = t
        if t == 0 or t < min_num:
            break
        c, d = coords[alive], direct[alive]
        pairs = (idxs[i].view(np.uint32) % np.uint32(t)).astype(np.int32)[:, None, :]
        hyp = po.generate_hypothesis_kernel(d, c, pairs)[:, 0]
        counts = po.vote_counts(d, c, hyp[:, None], thresh)[:, 0]
        win = int(counts.argmax())
        out["hyp"][i], out["counts"][i], out["win_counts"][i], out["win_idx"][i] = hyp, counts, counts[win], win
        if counts[win] < min_num:
            break
        pts, inl = po.refit(d, c, hyp[win][None], thresh)
        centre = pts[0] if np.all(np.isfinite(pts[0])) else hyp[win]
        out["centers"][i] = centre
        out["inliers"].append(alive[inl[0] != 0])
        alive = alive[inl[0] == 0]
        out["num"] = i + 1
    cen = out["centers"] if centers_for_assign is None else np.asarray(centers_for_assign, _F32)
    out["labels"] = assign(mask_img, field, cen, out["num"], thresh)
    return out


def ransac_voting_center(mask, field, idxs, thresh, min_num, centers_for_assign=None):
    """Batch form: mask [b,h,w], field [b,h,w,2], idxs [b,I,hn,2] -> list of `center_search` dicts."""
    return [center_search(mask[bi], field[bi], idxs[bi], thresh, min_num,
                          None if centers_for_assign is None else centers_for_assign[bi])
            for bi in range(len(mask))]
