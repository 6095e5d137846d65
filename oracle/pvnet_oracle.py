"""CPU oracle for PVNet's RANSAC voting layer -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module, and only as the checker or the
timed CPU baseline.  Nothing under ``pvnet_b200/`` imports it; the product path
fails loudly when its CUDA library is missing.

It restates, in numpy + the C kernels of ``pvnet_oracle.c``, what these reference
functions compute (paths relative to the reference project):

  ransac_voting_layer_v3                    lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:514-598
  estimate_voting_distribution_with_mean    lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:333-406
  ransac_voting_layer_v5                    lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:763-858
  generate_hypothesis (python, per batch)   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:983-1034
  b_inv (2x2 inverse via LU)                lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:503-512
  the two CUDA kernels                      lib/ransac_voting_gpu_layer/src/ransac_voting_kernel.cu:11-49, 88-126

Randomness.  The reference draws ``idxs`` (and, when subsampling, a uniform field)
from torch's CUDA generator.  The oracle never draws: callers pass ``idxs`` (and
``selection`` fields) explicitly, so both sides of a parity test see the same
samples.

Parity pin.  The reference has no test suite and no golden vectors (SURVEY.md §4).
The oracle is pinned two ways: (1) the analytic known-answer fixture derived from
the reference's ``data/demo`` (tests/golden/demo_cat.npz, made by
tests/golden/make_golden.py): voting on the exact vector field must return the
projected keypoints; (2) on the GPU the reference's own CUDA kernels, compiled
verbatim into ``oracle/_ref``, are run against the C kernels here bit for bit
(tests/test_gpu_reference_layer.py).
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libpvnet_oracle.so")
_lib = None

_F32P = ctypes.POINTER(ctypes.c_float)
_I32P = ctypes.POINTER(ctypes.c_int32)
_U8P = ctypes.POINTER(ctypes.c_uint8)


def build(force: bool = False) -> str:
    """Compile pvnet_oracle.c (gcc, OpenMP) if the .so is missing or stale."""
    src = os.path.join(_HERE, "pvnet_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "oracle"])
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        L.pvo_generate_hypothesis.argtypes = [_F32P, _F32P, _I32P, _F32P, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.pvo_generate_hypothesis.restype = None
        L.pvo_voting_for_hypothesis.argtypes = [_F32P, _F32P, _F32P, _U8P, ctypes.c_int, ctypes.c_int,
                                                ctypes.c_int, ctypes.c_float]
        L.pvo_voting_for_hypothesis.restype = None
        L.pvo_vote_counts.argtypes = [_F32P, _F32P, _F32P, _I32P, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                      ctypes.c_float]
        L.pvo_vote_counts.restype = None
        L.pvo_generate_hypothesis_vp.argtypes = [_F32P, _F32P, _I32P, _F32P, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.pvo_generate_hypothesis_vp.restype = None
        L.pvo_voting_for_hypothesis_vp.argtypes = [_F32P, _F32P, _F32P, _U8P, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                   ctypes.c_float]
        L.pvo_voting_for_hypothesis_vp.restype = None
        L.pvo_num_threads.restype = ctypes.c_int
        L.pvo_set_num_threads.argtypes = [ctypes.c_int]
        _lib = L
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _ptr(a, t):
    return a.ctypes.data_as(t)


# --------------------------------------------------------------------------- kernels
def generate_hypothesis_kernel(direct, coords, idxs):
    """ransac_voting_kernel.cu:11-86.  direct [tn,vn,2] f32, coords [tn,2] f32 (x,y),
    idxs [hn,vn,2] i32 -> hypo [hn,vn,2] f32 (degenerate pairs stay (0,0))."""
    direct, coords = _f32(direct), _f32(coords)
    idxs = np.ascontiguousarray(idxs, dtype=np.int32)
    tn, vn, _ = direct.shape
    hn = idxs.shape[0]
    assert coords.shape == (tn, 2) and idxs.shape == (hn, vn, 2)
    if hn and (idxs.min() < 0 or idxs.max() >= tn):
        raise ValueError("idxs out of range")
    hypo = np.empty((hn, vn, 2), np.float32)
    lib().pvo_generate_hypothesis(_ptr(direct, _F32P), _ptr(coords, _F32P), _ptr(idxs, _I32P),
                                  _ptr(hypo, _F32P), tn, vn, hn)
    return hypo


def voting_for_hypothesis_kernel(direct, coords, hypo, thresh):
    """ransac_voting_kernel.cu:88-167 -> inliers [hn,vn,tn] u8 (zero-filled first,
    as ransac_voting_gpu.py:557 does)."""
    direct, coords, hypo = _f32(direct), _f32(coords), _f32(hypo)
    tn, vn, _ = direct.shape
    hn = hypo.shape[0]
    inl = np.zeros((hn, vn, tn), np.uint8)
    lib().pvo_voting_for_hypothesis(_ptr(direct, _F32P), _ptr(coords, _F32P), _ptr(hypo, _F32P),
                                    _ptr(inl, _U8P), tn, vn, hn, np.float32(thresh))
    return inl


def vote_counts(direct, coords, hypo, thresh):
    """sum over pixels of the inlier predicate -> int32 [hn,vn]
    (== torch.sum(cur_inlier, 2), ransac_voting_gpu.py:561)."""
    direct, coords, hypo = _f32(direct), _f32(coords), _f32(hypo)
    tn, vn, _ = direct.shape
    hn = hypo.shape[0]
    counts = np.zeros((hn, vn), np.int32)
    lib().pvo_vote_counts(_ptr(direct, _F32P), _ptr(coords, _F32P), _ptr(hypo, _F32P),
                          _ptr(counts, _I32P), tn, vn, hn, np.float32(thresh))
    return counts


# ----------------------------------------------------------------- mask / compaction
def generate_hypothesis_vanishing_point_kernel(direct, coords, idxs):
    """ransac_voting_kernel.cu:170-230 -> hypo [hn,vn,3] f32 (homogeneous)."""
    direct, coords = _f32(direct), _f32(coords)
    idxs = np.ascontiguousarray(idxs, dtype=np.int32)
    tn, vn, _ = direct.shape
    hn = idxs.shape[0]
    hypo = np.empty((hn, vn, 3), np.float32)
    lib().pvo_generate_hypothesis_vp(_ptr(direct, _F32P), _ptr(coords, _F32P), _ptr(idxs, _I32P), _ptr(hypo, _F32P),
                                     tn, vn, hn)
    return hypo


def voting_for_hypothesis_vanishing_point_kernel(direct, coords, hypo, thresh):
    """ransac_voting_kernel.cu:263-305 -> inliers [hn,vn,tn] u8."""
    direct, coords, hypo = _f32(direct), _f32(coords), _f32(hypo)
    tn, vn, _ = direct.shape
    hn = hypo.shape[0]
    inl = np.zeros((hn, vn, tn), np.uint8)
    lib().pvo_voting_for_hypothesis_vp(_ptr(direct, _F32P), _ptr(coords, _F32P), _ptr(hypo, _F32P), _ptr(inl, _U8P),
                                       tn, vn, hn, float(thresh))
    return inl


def _byte_mask(mask_img):
    """`.byte()` of ransac_voting_gpu.py:527: integer masks keep their low 8 bits."""
    m = np.asarray(mask_img)
    if m.dtype == np.bool_:
        return m.astype(np.uint8)
    if np.issubdtype(m.dtype, np.integer):
        return (m.astype(np.int64) & 0xFF).astype(np.uint8)
    return m.astype(np.uint8)


def subsample_probability(max_num, foreground):
    """`max_num / foreground_num.float()` (ransac_voting_gpu.py:539).  torch evaluates
    int / tensor as tensor.reciprocal() * int, both in float32."""
    r = np.float32(1.0) / np.float32(foreground)
    return np.float32(r * np.float32(max_num))


def compact(cur_mask_u8, vertex_img):
    """ransac_voting_gpu.py:542-546.  cur_mask [h,w] (nonzero = keep), vertex [h,w,vn,2]
    -> coords [tn,2] f32 as (x,y) in row-major pixel order, direct [tn,vn,2] f32."""
    ys, xs = np.nonzero(cur_mask_u8)
    coords = np.stack([xs, ys], 1).astype(np.float32)
    direct = np.ascontiguousarray(np.asarray(vertex_img)[ys, xs], dtype=np.float32)
    return coords, direct


def refit(direct, coords, win_pts, thresh):
    """ransac_voting_gpu.py:578-595: inliers of the winning hypothesis, then the
    least-squares intersection  (sum n n^T) p = sum n (n.c),  n = (d_y, -d_x).
    Sums are carried in float64 (the reference's fp32 cuBLAS order is unspecified;
    tolerance 1e-4, see DESIGN.md).  Returns (pts [vn,2] f32, inlier [vn,tn] u8)."""
    tn, vn, _ = direct.shape
    inl = voting_for_hypothesis_kernel(direct, coords, win_pts[None], thresh)[0]  # [vn,tn]
    nx = direct[:, :, 1].T.astype(np.float64)      # [vn,tn]
    ny = (-direct[:, :, 0]).T.astype(np.float64)
    w = inl.astype(np.float64)
    nx, ny = nx * w, ny * w
    bb = nx * coords[None, :, 0].astype(np.float64) + ny * coords[None, :, 1].astype(np.float64)
    a00, a01, a11 = (nx * nx).sum(1), (nx * ny).sum(1), (ny * ny).sum(1)
    b0, b1 = (nx * bb).sum(1), (ny * bb).sum(1)
    det = a00 * a11 - a01 * a01
    with np.errstate(all="ignore"):
        px = (a11 * b0 - a01 * b1) / det
        py = (a00 * b1 - a01 * b0) / det
    pts = np.stack([px, py], 1).astype(np.float32)
    return pts, inl


# ------------------------------------------------------------------------ the layer
def ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=30000, idxs=None, selection=None, return_debug=False):
    """ransac_voting_gpu.py:514-598.

    mask [b,h,w] integer (nonzero = foreground after `.byte()`), vertex [b,h,w,vn,2] f32.
    idxs: sequence of b arrays [round_hyp_num,vn,2] int32 (entries for skipped images
    are ignored; may be None there).  selection: sequence of b float32 [h,w] uniform
    fields, consulted only for images with foreground > max_num (:537-540).

    The reference's `while True` loop (:552-576) re-evaluates the SAME idxs every
    round (they are drawn once at :547), so every round gives identical counts and
    the strict `<` update (:567) makes rounds 2.. no-ops: one evaluation is the
    whole result.  confidence / max_iter therefore do not influence the output.
    """
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    out = np.zeros((b, vn, 2), np.float32)
    debug = []
    for bi in range(b):
        cur_mask = _byte_mask(mask[bi])
        fg = int(cur_mask.astype(np.int64).sum())          # torch.sum(uint8) -> int64
        if fg < min_num:                                   # :531-534
            debug.append(None)
            continue
        if fg > max_num:                                   # :537-540
            p = subsample_probability(max_num, fg)
            sel = np.asarray(selection[bi], dtype=np.float32)
            cur_mask = cur_mask * (sel < p).astype(np.uint8)
        coords, direct = compact(cur_mask, vertex[bi])     # :542-546
        tn = coords.shape[0]
        cur_idxs = np.ascontiguousarray(idxs[bi], dtype=np.int32)
        assert cur_idxs.shape == (round_hyp_num, vn, 2)
        hyp = generate_hypothesis_kernel(direct, coords, cur_idxs)        # :554
        counts = vote_counts(direct, coords, hyp, inlier_thresh)          # :557-561
        win_idx = counts.argmax(0)                         # first max on ties (:562)
        win_counts = counts[win_idx, np.arange(vn)]
        win_pts = hyp[win_idx, np.arange(vn)]
        ratio = win_counts.astype(np.float32) / np.float32(tn)
        all_win_pts = np.zeros((vn, 2), np.float32)
        larger = np.float32(0) < ratio                     # :567 (all_win_ratio starts at 0)
        all_win_pts[larger] = win_pts[larger]
        pts, inl = refit(direct, coords, all_win_pts, inlier_thresh)      # :578-595
        out[bi] = pts
        debug.append(dict(tn=tn, coords=coords, direct=direct, hyp=hyp, counts=counts,
                          win_idx=win_idx, win_pts=all_win_pts, refit_inliers=inl))
    return (out, debug) if return_debug else out


def ransac_voting_layer_v5(mask, vertex, round_hyp_num, inlier_thresh=0.999, min_num=5, max_num=100, idxs=None,
                           selection=None):
    """ransac_voting_gpu.py:763-858: v3 plus confidence = inliers of the refitted point at
    threshold 0.999 (:850), divided by tn (:851); zeros for skipped images (:788-793)."""
    kp, dbg = ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=inlier_thresh, min_num=min_num,
                                     max_num=max_num, idxs=idxs, selection=selection, return_debug=True)
    conf = np.zeros(kp.shape[:2], np.float32)
    for bi, d in enumerate(dbg):
        if d is None:
            continue
        cnt = vote_counts(d["direct"], d["coords"], kp[bi][None], 0.999)[0]
        conf[bi] = cnt.astype(np.float32) / np.float32(d["tn"])
    return kp, conf


def generate_hypothesis(mask, vertex, round_hyp_num, inlier_thresh=0.999, min_num=5, max_num=30000,
                        idxs=None, selection=None):
    """ransac_voting_gpu.py:983-1034 (python-level `generate_hypothesis`): per image the
    hypotheses [hn,vn,2] and their inlier counts [hn,vn] (int64 there).  The reference's
    skip branch is broken (`batch_win_pts` undefined, :1003); here a skipped image
    raises, like the NameError it would hit."""
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    hyps, cnts = [], []
    for bi in range(b):
        cur_mask = _byte_mask(mask[bi])
        fg = int(cur_mask.astype(np.int64).sum())
        if fg < min_num:
            raise NameError("batch_win_pts")  # reference behaviour at :1003
        if fg > max_num:
            p = subsample_probability(max_num, fg)
            cur_mask = cur_mask * (np.asarray(selection[bi], np.float32) < p).astype(np.uint8)
        coords, direct = compact(cur_mask, vertex[bi])
        hyp = generate_hypothesis_kernel(direct, coords, np.asarray(idxs[bi], np.int32))
        hyps.append(hyp)
        cnts.append(vote_counts(direct, coords, hyp, inlier_thresh).astype(np.int64))
    return np.stack(hyps), np.stack(cnts)


def estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, topk=128,
                                           inlier_thresh=0.99, min_num=5, max_num=30000, idxs=None,
                                           selection=None, return_debug=False):
    """ransac_voting_gpu.py:333-406.

    mask [b,h,w] (foreground = value == 1, :339), vertex [b,h,w,vn,2], mean [b,vn,2].
    idxs: sequence of b arrays [rounds,round_hyp_num,vn,2] int32 with
    rounds = ceil(min_hyp_num/round_hyp_num) (fresh draw per round, :367).
    Returns (mean, cov [b,vn,2,2] f32).  `topk` is unused by the reference here.
    """
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    mean = np.asarray(mean, dtype=np.float32)
    b, h, w, vn, _ = vertex.shape
    rounds = int(np.ceil(min_hyp_num / round_hyp_num))
    all_hyp, all_ratio, debug = [], [], []
    for bi in range(b):
        cur_mask = (mask[bi] == 1)
        fg = int(cur_mask.sum())
        if fg < min_num:                                   # :343-348
            all_hyp.append(np.zeros((min_hyp_num, vn, 2), np.float32))
            all_ratio.append(np.ones((min_hyp_num, vn), np.float32))
            debug.append(None)
            continue
        if fg > max_num:                                   # :351-355
            p = subsample_probability(max_num, fg)
            cur_mask = cur_mask & (np.asarray(selection[bi], np.float32) < p)
            fg = int(cur_mask.sum())
        coords, direct = compact(cur_mask.astype(np.uint8), vertex[bi])
        hyps, ratios, cnts = [], [], []
        for r in range(rounds):                            # :363-378
            hyp = generate_hypothesis_kernel(direct, coords, np.asarray(idxs[bi][r], np.int32))
            c = vote_counts(direct, coords, hyp, inlier_thresh)
            hyps.append(hyp)
            cnts.append(c)
            ratios.append(c.astype(np.float32) / np.float32(fg))
        all_hyp.append(np.concatenate(hyps, 0))
        all_ratio.append(np.concatenate(ratios, 0))
        debug.append(dict(tn=coords.shape[0], hyp=np.concatenate(hyps, 0), counts=np.concatenate(cnts, 0)))
    lens = {a.shape[0] for a in all_hyp}
    if len(lens) != 1:
        # torch.cat at :389 fails when a skipped image (min_hyp_num rows) meets a
        # normal one (rounds*round_hyp_num rows) of a different length (SURVEY App. C.4)
        raise RuntimeError("Sizes of tensors must match except in dimension 0")
    hyp = np.stack(all_hyp).transpose(0, 2, 1, 3)          # [b,vn,hn,2]  :392
    ratio = np.stack(all_ratio).transpose(0, 2, 1).copy()  # [b,vn,hn]    :393
    thresh = (ratio.max(2) - np.float32(0.1)).astype(np.float32)          # :394
    ratio[ratio < thresh[:, :, None]] = 0.0                               # :395
    diff = (hyp - mean[:, :, None, :]).astype(np.float32)                 # :398
    wdiff = (diff * ratio[..., None]).astype(np.float32)                  # :399
    cov = np.einsum("bvhi,bvhj->bvij", diff.astype(np.float64), wdiff.astype(np.float64))  # :400
    wsum = ratio.astype(np.float64).sum(2).astype(np.float32)
    cov = (cov.astype(np.float32) / (wsum + np.float32(1e-3))[:, :, None, None]).astype(np.float32)  # :401
    return (mean, cov, debug) if return_debug else (mean, cov)


# ------------------------------------------------------------ remaining layer variants
def ransac_motion_voting(mask, vertex):
    """ransac_voting_gpu.py:960-981: per image and keypoint the mean over the foreground
    pixels (`.byte()` nonzero) of vertex + (x, y); zeros when the mask is empty (:971-973).
    Sums in float64 (the reference's torch.mean is fp32 with library-defined order)."""
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    out = np.zeros((b, vn, 2), np.float32)
    for bi in range(b):
        coords, direct = compact(_byte_mask(mask[bi]), vertex[bi])
        if coords.shape[0] < 1:
            continue
        out[bi] = (direct.astype(np.float64) + coords[:, None, :].astype(np.float64)).mean(0).astype(np.float32)
    return out


def ransac_voting_layer(mask, vertex, class_num, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                        min_num=5, max_num=30000, idxs=None, selection=None):
    """ransac_voting_gpu.py:10-97 (the first layer): for every class k+1 in 1..class_num-1 the
    pixels with mask == k+1 vote; the result is the WINNING HYPOTHESIS itself (no refit),
    [b, class_num-1, vn, 2].  idxs[bi][k] is the [hn,vn,2] draw of (image, class); as in v3 the
    extra rounds re-score the same draw, so one evaluation is the result."""
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    out = np.zeros((b, class_num - 1, vn, 2), np.float32)
    for bi in range(b):
        for k in range(class_num - 1):
            cur_mask = (mask[bi] == k + 1)
            fg = int(cur_mask.sum())
            if fg < min_num:                               # :28-31
                continue
            if fg > max_num:                               # :34-37
                p = subsample_probability(max_num, fg)
                cur_mask = cur_mask & (np.asarray(selection[bi][k], np.float32) < p)
            coords, direct = compact(cur_mask.astype(np.uint8), vertex[bi])
            tn = coords.shape[0]
            hyp = generate_hypothesis_kernel(direct, coords, np.ascontiguousarray(idxs[bi][k], np.int32))
            counts = vote_counts(direct, coords, hyp, inlier_thresh)
            win_idx = counts.argmax(0)
            win_counts = counts[win_idx, np.arange(vn)]
            ratio = win_counts.astype(np.float32) / np.float32(tn)
            larger = np.float32(0) < ratio                 # :74
            out[bi, k][larger] = hyp[win_idx, np.arange(vn)][larger]
    return out


def ransac_voting_layer_v4(mask, vertex, round_hyp_num, inlier_thresh=0.99, confidence=0.999, max_iter=20,
                           min_num=5, max_num=30000, idxs=None, selection=None):
    """ransac_voting_gpu.py:669-760: v3 plus var[b,vn] = sum over the winner's inliers of
    (n.p - n.c)^2 / #inliers, n = (d_y,-d_x), p the refitted point (:750-752); skipped images
    give zeros and var = 1 (:685-689).  float64 sums."""
    kp, dbg = ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=inlier_thresh, min_num=min_num,
                                     max_num=max_num, idxs=idxs, selection=selection, return_debug=True)
    var = np.ones(kp.shape[:2], np.float32)
    for bi, d in enumerate(dbg):
        if d is None:
            continue
        direct, coords, inl = d["direct"], d["coords"], d["refit_inliers"]     # inl [vn,tn]
        nx = direct[:, :, 1].T.astype(np.float64)
        ny = (-direct[:, :, 0]).T.astype(np.float64)
        bb = nx * coords[None, :, 0] + ny * coords[None, :, 1]
        res = nx * kp[bi][:, 0:1].astype(np.float64) + ny * kp[bi][:, 1:2].astype(np.float64) - bb
        w = inl.astype(np.float64)
        with np.errstate(all="ignore"):
            var[bi] = ((res * res * w).sum(1) / w.sum(1)).astype(np.float32)
    return kp, var


def ransac_voting_hypothesis(mask, vertex, round_hyp_num, inlier_thresh=0.999, min_num=5, max_num=30000,
                             idxs=None, selection=None):
    """ransac_voting_gpu.py:218-261: hypotheses [b,hn,vn,2] and inlier counts [b,hn,vn] (int64)
    of the pixels with mask == 1; a skipped image gives zero hypotheses and counts of ONE (:228-233)."""
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    hyps = np.zeros((b, round_hyp_num, vn, 2), np.float32)
    cnts = np.ones((b, round_hyp_num, vn), np.int64)
    for bi in range(b):
        cur_mask = (mask[bi] == 1)
        fg = int(cur_mask.sum())
        if fg < min_num:
            continue
        if fg > max_num:
            p = subsample_probability(max_num, fg)
            cur_mask = cur_mask & (np.asarray(selection[bi], np.float32) < p)
        coords, direct = compact(cur_mask.astype(np.uint8), vertex[bi])
        hyps[bi] = generate_hypothesis_kernel(direct, coords, np.ascontiguousarray(idxs[bi], np.int32))
        cnts[bi] = vote_counts(direct, coords, hyps[bi], inlier_thresh)
    return hyps, cnts


def estimate_voting_distribution(mask, vertex, round_hyp_num=256, min_hyp_num=4096, topk=128, inlier_thresh=0.99,
                                 min_num=5, max_num=30000, idxs=None, selection=None, return_ratio=False):
    """ransac_voting_gpu.py:263-331: ratio-weighted mean and covariance of the top-k hypotheses
    per keypoint.  idxs as in estimate_voting_distribution_with_mean.  When several ratios tie at
    the k-th place torch.topk's choice among them is unspecified; this restatement keeps the
    lowest hypothesis indices (tests avoid ties).  float64 sums."""
    mask = np.asarray(mask)
    vertex = np.asarray(vertex)
    b, h, w, vn, _ = vertex.shape
    rounds = int(np.ceil(min_hyp_num / round_hyp_num))
    hn = rounds * round_hyp_num
    hyp = np.zeros((b, hn, vn, 2), np.float32)
    ratio = np.ones((b, hn, vn), np.float32)
    for bi in range(b):
        cur_mask = (mask[bi] == 1)
        fg = int(cur_mask.sum())
        if fg < min_num:                                   # :271-277 (the reference's shapes only fit hn == round_hyp_num)
            continue
        if fg > max_num:
            p = subsample_probability(max_num, fg)
            cur_mask = cur_mask & (np.asarray(selection[bi], np.float32) < p)
            fg = int(cur_mask.sum())
        coords, direct = compact(cur_mask.astype(np.uint8), vertex[bi])
        for r in range(rounds):
            hp = generate_hypothesis_kernel(direct, coords, np.asarray(idxs[bi][r], np.int32))
            c = vote_counts(direct, coords, hp, inlier_thresh)
            hyp[bi, r * round_hyp_num:(r + 1) * round_hyp_num] = hp
            ratio[bi, r * round_hyp_num:(r + 1) * round_hyp_num] = c.astype(np.float32) / np.float32(fg)
    hyp = hyp.transpose(0, 2, 1, 3)                        # [b,vn,hn,2]
    ratio = ratio.transpose(0, 2, 1)                       # [b,vn,hn]
    order = np.argsort(-ratio, axis=2, kind="stable")[:, :, :topk]
    kept = np.zeros_like(ratio)
    np.put_along_axis(kept, order, np.take_along_axis(ratio, order, 2), 2)   # :316-317
    w64 = kept.astype(np.float64)
    wsum = w64.sum(2)
    with np.errstate(all="ignore"):
        mean = (w64[..., None] * hyp.astype(np.float64)).sum(2) / wsum[..., None]              # :319-320
        diff = hyp.astype(np.float64) - mean[:, :, None, :]
        cov = np.einsum("bvhi,bvhj->bvij", diff, diff * w64[..., None]) / wsum[..., None, None]  # :322-325
    if return_ratio:       # [b,vn,hn] ratios before the top-k cut (tests use them to find ties at the cut)
        return mean.astype(np.float32), cov.astype(np.float32), ratio
    return mean.astype(np.float32), cov.astype(np.float32)


def num_threads():
    return int(lib().pvo_num_threads())


def set_num_threads(n):
    lib().pvo_set_num_threads(int(n))
