"""Host side of the H100 voting layer: the reference's Python API over libpvnet_b200.so.

Same names, argument meaning and defaults as zju3dv/pvnet's
``lib/ransac_voting_gpu_layer/ransac_voting_gpu.py`` for the functions on the
inference hot path:

    ransac_voting_layer_v3                   (reference :514-598)
    ransac_voting_layer_v5                   (reference :763-858)
    estimate_voting_distribution_with_mean   (reference :333-406)
    generate_hypothesis                      (reference :983-1034)
    ransac_motion_voting                     (reference :960-981)
    ransac_voting_layer_v4                   (reference :669-760)
    ransac_voting_layer                      (reference :10-97)
    ransac_voting_layer_v2                   (reference :99-216)
    ransac_voting_vanish_point_layer         (reference :408-501)
    ransac_voting_hypothesis                 (reference :218-261)
    estimate_voting_distribution             (reference :263-331)

so ``tools/demo.py`` / ``tools/train_linemod.py --test_model`` keep working when
``lib/ransac_voting_gpu_layer/ransac_voting_gpu.py`` is this module (the shim under
``lib/`` re-exports it).  Tensors in, tensors out; the work happens in hand-written
sm_90a kernels behind the C ABI of ``include/pvnet_b200.h``.  There is no CPU or
PyTorch fallback: without the library or a CUDA device these functions raise.

Randomness (``rng=``):
  "reference" (default)  replays the reference's torch RNG calls in the reference's
        order -- per image, ``uniform_`` only when subsampling (:538), then
        ``random_(0, tn)`` for idxs (:547; once per round at :367) -- so under a fixed
        ``torch.manual_seed`` the samples are the ones the reference would draw.  This
        needs the per-image foreground counts on the host: ONE device->host copy per
        call (the reference does >= 3 blocking syncs per image).
  "batched"  one ``random_`` (and, if subsampling is possible, one ``uniform_``) call
        for the whole batch, no host sync at all; statistically equivalent, different
        stream.
  "device"   (``ransac_voting_layer_v3`` and ``ransac_voting_pipeline`` only) nothing is drawn by
        torch at all: the kernels sample with a counter-based Philox generator whose
        {seed, offset} live in a small device tensor (seeded from ``torch.initial_seed()``),
        so the call has no RNG launches, no host sync, and a captured CUDA graph draws fresh
        samples on every replay.
  explicit ``idxs=`` / ``selection=`` tensors override all of them (used by the parity tests).

``ransac_voting_pipeline`` is the fused form of what ``UncertaintyEvalWrapper``
(tools/train_linemod.py:119-130) runs per batch -- v3, then
estimate_voting_distribution_with_mean on its result -- with one compaction / gather of the
mask and field for both layers.
"""
from __future__ import annotations

import ctypes
import math

import torch

from . import _native

_MASK_NONZERO_BYTE = 0
_MASK_EQUALS_ONE = 1

_INT_DTYPES = {torch.uint8: 1, torch.int8: 1, torch.bool: 1, torch.int16: 2, torch.int32: 4, torch.int64: 8}


def _require_cuda(t: torch.Tensor, name: str):
    if not t.is_cuda:
        raise RuntimeError(f"pvnet_b200: `{name}` must be a CUDA tensor (there is no CPU path)")


def _prep_mask(mask: torch.Tensor, mode: int):
    """-> (tensor kept alive, element size).  Integer/bool masks are used in place."""
    if mask.dtype not in _INT_DTYPES:
        # float masks: `.byte()` (v3) / `== 1` (with_mean) semantics, evaluated by torch once
        mask = mask.byte() if mode == _MASK_NONZERO_BYTE else (mask == 1).to(torch.uint8)
    if not mask.is_contiguous():
        mask = mask.contiguous()
    return mask, _INT_DTYPES[mask.dtype]


def _prep_vertex(vertex: torch.Tensor):
    if vertex.dtype != torch.float32:
        vertex = vertex.float()
    if vertex.dim() != 5 or vertex.shape[-1] != 2:
        raise ValueError(f"vertex must be [b,h,w,vn,2], got {tuple(vertex.shape)}")
    strides = (ctypes.c_int64 * 5)(*vertex.stride())
    return vertex, strides


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


_WS_CACHE = {}       # (device, stream) -> grow-only uint8 workspace; stream-ordered reuse is safe
_RNG_STATE = {}      # device -> (seed the state was made from, int64[2] device tensor {seed, offset})


def _workspace(b, h, w, vn, hn_total, device):
    """The caller-owned workspace of the C ABI.  One grow-only buffer per (device, stream): calls on a
    stream are ordered, so reusing the address is safe, costs no allocation per call and keeps the
    launch sequence capturable in a CUDA graph (the reference allocates per call, :557)."""
    n = ctypes.c_size_t()
    _native.check(_native.lib().pvnet_vote_workspace_bytes(b, h, w, vn, hn_total, ctypes.byref(n)),
                  "pvnet_vote_workspace_bytes")
    device = torch.device(device)
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < n.value:
        ws = torch.empty(n.value, dtype=torch.uint8, device=device)
        _WS_CACHE[key] = ws
    return ws, ws.numel()


def reset_device_rng(device=None):
    """Rewind the device-side sampler of `device` to {torch.initial_seed(), offset 0}, in place."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = device.index if device.index is not None else torch.cuda.current_device()
    seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
    cur = _RNG_STATE.get(key)
    if cur is None:
        _rng_state(device)
    else:
        cur[1].copy_(torch.tensor([seed, 0], dtype=torch.int64))
        cur[0] = seed


def _rng_state(device):
    """{seed, offset} of the device-side Philox generator; re-made when torch.manual_seed changed."""
    device = torch.device(device)
    key = device.index if device.index is not None else torch.cuda.current_device()
    seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
    cur = _RNG_STATE.get(key)
    if cur is None:
        cur = [seed, torch.tensor([seed, 0], dtype=torch.int64, device=device)]
        _RNG_STATE[key] = cur
    elif cur[0] != seed:       # re-seed IN PLACE: captured CUDA graphs hold this tensor's address
        cur[1].copy_(torch.tensor([seed, 0], dtype=torch.int64))
        cur[0] = seed
    return cur[1]


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def foreground_counts(mask: torch.Tensor, mode: int = _MASK_NONZERO_BYTE) -> torch.Tensor:
    """int32 [b] foreground pixels per image, on the device (no sync)."""
    _require_cuda(mask, "mask")
    m, esz = _prep_mask(mask, mode)
    b, h, w = m.shape
    with torch.cuda.device(m.device):
        out = torch.empty(b, dtype=torch.int32, device=m.device)
        nchunk = (h * w + 2047) // 2048
        ws = torch.empty(b * nchunk * 4, dtype=torch.uint8, device=m.device)
        _native.check(_native.lib().pvnet_mask_foreground_count(_ptr(m), esz, mode, b, h, w, _ptr(out), _ptr(ws),
                                                                ws.numel(), _stream(m.device)),
                      "pvnet_mask_foreground_count")
    return out


def _draw_reference(mask, mode, b, h, w, vn, hn, rounds, min_num, max_num):
    """Replays the reference's RNG calls (see module docstring).  Returns
    (idxs [b,rounds*hn,vn,2] int32, selection [b,h,w] f32 or None, fg list)."""
    dev = mask.device
    fg = foreground_counts(mask, mode).cpu().tolist()          # the one host sync
    idxs = torch.zeros([b, rounds * hn, vn, 2], dtype=torch.int32, device=dev)
    selection = None
    for bi in range(b):
        if fg[bi] < min_num:
            continue
        tn = fg[bi]
        if fg[bi] > max_num:
            if selection is None:
                selection = torch.empty([b, h, w], dtype=torch.float32, device=dev)
            sel = torch.zeros([h, w], dtype=torch.float32, device=dev).uniform_(0, 1)
            selection[bi] = sel
            cur = (mask[bi].byte() != 0) if mode == _MASK_NONZERO_BYTE else (mask[bi] == 1)
            p = max_num / torch.tensor(fg[bi], device=dev).float()      # same expression as :539
            tn = int((cur & (sel < p)).sum().item())                    # rare path: second sync
        for r in range(rounds):
            idxs[bi, r * hn:(r + 1) * hn] = torch.zeros([hn, vn, 2], dtype=torch.int32,
                                                        device=dev).random_(0, max(tn, 1))
    return idxs, selection, fg


def _draw_batched(b, h, w, vn, hn_total, max_num, device):
    idxs = torch.empty([b, hn_total, vn, 2], dtype=torch.int32, device=device).random_(0, 2 ** 31 - 1)
    selection = None
    if max_num < h * w:
        selection = torch.empty([b, h, w], dtype=torch.float32, device=device).uniform_(0, 1)
    return idxs, selection


def _check_injected(idxs, selection, b, h, w, vn, hn_total, device):
    idxs = torch.as_tensor(idxs, device=device)
    if idxs.dtype != torch.int32:
        idxs = idxs.to(torch.int32)
    if tuple(idxs.shape) != (b, hn_total, vn, 2):
        raise ValueError(f"idxs must be [b={b},{hn_total},{vn},2], got {tuple(idxs.shape)}")
    idxs = idxs.contiguous()
    if selection is not None:
        selection = torch.as_tensor(selection, device=device, dtype=torch.float32).contiguous()
        if tuple(selection.shape) != (b, h, w):
            raise ValueError(f"selection must be [b,h,w], got {tuple(selection.shape)}")
    return idxs, selection


def ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=30000, *, idxs=None, selection=None, rng="reference",
                           return_debug=False):
    """Reference signature (ransac_voting_gpu.py:514-515) plus keyword-only extras.

    :param mask:      [b,h,w] integer/bool CUDA tensor; nonzero (after `.byte()`) = foreground
    :param vertex:    [b,h,w,vn,2] float32 CUDA tensor, any strides (the NCHW permuted view
                      the reference's callers pass is read in place)
    :param round_hyp_num: hypotheses per keypoint
    :param inlier_thresh: cosine threshold of the inlier test
    :param confidence, max_iter: accepted for compatibility; the reference's extra RANSAC
                      rounds re-score the same samples (idxs drawn once at :547), so they
                      never change its result and are not executed here
    :return: [b,vn,2] float32 keypoints (x,y); with return_debug also a dict of
             counts [b,hn,vn] int32, hyp [b,hn,vn,2], tn [b] int32 (device tensors)
    """
    del confidence, max_iter
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_NONZERO_BYTE)
    v, strides = _prep_vertex(vertex)
    with torch.cuda.device(dev):
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hn, dev)
        elif rng == "reference":
            idxs, selection, _ = _draw_reference(m, _MASK_NONZERO_BYTE, b, h, w, vn, hn, 1, min_num, max_num)
        elif rng == "batched":
            idxs, selection = _draw_batched(b, h, w, vn, hn, max_num, dev)
        elif rng == "device":
            return ransac_voting_pipeline(mask, vertex, hn, inlier_thresh, with_covariance=False, min_num=min_num,
                                          max_num=max_num, rng="device", return_debug=return_debug)
        else:
            raise ValueError(f"unknown rng mode {rng!r}")
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        counts = hyp = tn = None
        if return_debug:
            counts = torch.empty([b, hn, vn], dtype=torch.int32, device=dev)
            hyp = torch.empty([b, hn, vn, 2], dtype=torch.float32, device=dev)
            tn = torch.empty([b], dtype=torch.int32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, hn, dev)
        _native.check(_native.lib().pvnet_ransac_voting_v3(
            _ptr(m), esz, _ptr(v), strides, _ptr(idxs), _ptr(selection), b, h, w, vn, hn,
            float(inlier_thresh), int(min_num), int(min(max_num, 2 ** 31 - 1)),
            _ptr(out), _ptr(counts), _ptr(hyp), _ptr(tn), _ptr(ws), ws_bytes, _stream(dev)),
            "pvnet_ransac_voting_v3")
    if return_debug:
        return out, dict(counts=counts, hyp=hyp, tn=tn, idxs=idxs, selection=selection)
    return out


def ransac_voting_pipeline(mask, vertex, round_hyp_num, inlier_thresh=0.99, with_covariance=True, cov_round_hyp_num=256,
                           cov_min_hyp_num=4096, cov_inlier_thresh=0.99, min_num=5, max_num=30000, *,
                           mask_mode="nonzero", idxs=None, cov_idxs=None, selection=None, rng="device",
                           return_debug=False):
    """``ransac_voting_layer_v3`` followed by ``estimate_voting_distribution_with_mean`` on its result
    (tools/train_linemod.py:119-130) as one launch sequence over `pvnet_ransac_voting_pipeline`.

    :param mask_mode: "nonzero" (v3's reading, :527) or "equals_one" (with_mean's, :339) for BOTH layers;
                      identical for the binary argmax mask of a 2-class network
    :param rng:       "device" (in-kernel Philox, no torch RNG launches, graph-capturable) or "batched"
                      (torch draws once per batch); injected idxs / cov_idxs / selection override
    :return: keypoints [b,vn,2] (and cov [b,vn,2,2] when with_covariance); with return_debug also a dict
    """
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    rounds = int(math.ceil(cov_min_hyp_num / cov_round_hyp_num)) if with_covariance else 0
    hnt = int(cov_round_hyp_num) * rounds
    dev = mask.device
    mode = {"nonzero": _MASK_NONZERO_BYTE, "equals_one": _MASK_EQUALS_ONE}[mask_mode]
    m, esz = _prep_mask(mask, mode)
    v, strides = _prep_vertex(vertex)
    with torch.cuda.device(dev):
        state = None
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hn, dev)
        if with_covariance and cov_idxs is not None:
            cov_idxs, _ = _check_injected(cov_idxs, None, b, h, w, vn, hnt, dev)
        if rng == "batched":
            if idxs is None:
                idxs, sel2 = _draw_batched(b, h, w, vn, hn, max_num, dev)
                selection = sel2 if selection is None else selection
            if with_covariance and cov_idxs is None:
                cov_idxs = torch.empty([b, hnt, vn, 2], dtype=torch.int32, device=dev).random_(0, 2 ** 31 - 1)
        elif rng == "device":
            state = _rng_state(dev)
        elif idxs is None or (with_covariance and cov_idxs is None):
            raise ValueError(f"rng mode {rng!r} needs injected idxs (and cov_idxs)")
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        cov = torch.empty([b, vn, 2, 2], dtype=torch.float32, device=dev) if with_covariance else None
        dbg = {}
        if return_debug:
            dbg = dict(counts=torch.empty([b, hn, vn], dtype=torch.int32, device=dev),
                       hyp=torch.empty([b, hn, vn, 2], dtype=torch.float32, device=dev),
                       tn=torch.empty([b], dtype=torch.int32, device=dev))
            if with_covariance:
                dbg.update(cov_counts=torch.empty([b, hnt, vn], dtype=torch.int32, device=dev),
                           cov_hyp=torch.empty([b, hnt, vn, 2], dtype=torch.float32, device=dev))
        ws, ws_bytes = _workspace(b, h, w, vn, hn + hnt, dev)
        _native.check(_native.lib().pvnet_ransac_voting_pipeline(
            _ptr(m), esz, mode, _ptr(v), strides, _ptr(idxs), _ptr(cov_idxs), _ptr(selection), _ptr(state),
            b, h, w, vn, hn, float(inlier_thresh), int(cov_round_hyp_num), max(rounds, 1), int(cov_min_hyp_num),
            float(cov_inlier_thresh), int(min_num), int(min(max_num, 2 ** 31 - 1)), _ptr(out), _ptr(cov),
            _ptr(dbg.get("counts")), _ptr(dbg.get("hyp")), _ptr(dbg.get("cov_counts")), _ptr(dbg.get("cov_hyp")),
            _ptr(dbg.get("tn")), _ptr(ws), ws_bytes, _stream(dev)), "pvnet_ransac_voting_pipeline")
    res = (out, cov) if with_covariance else out
    if return_debug:
        dbg.update(idxs=idxs, cov_idxs=cov_idxs, selection=selection)
        return (out, cov, dbg) if with_covariance else (out, dbg)
    return res


def ransac_voting_layer_v5(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=100, *, idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:763-764; note its max_num default of 100).
    Returns (keypoints [b,vn,2], confidence [b,vn]): confidence = share of the voting pixels
    that are inliers of the REFITTED keypoint at threshold 0.999 (:850-852).  Used by
    tools/train_linemod.py:104 (`EvalWrapper(use_uncertainty=True)`)."""
    del confidence, max_iter
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_NONZERO_BYTE)
    v, strides = _prep_vertex(vertex)
    with torch.cuda.device(dev):
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hn, dev)
        elif rng == "reference":
            idxs, selection, _ = _draw_reference(m, _MASK_NONZERO_BYTE, b, h, w, vn, hn, 1, min_num, max_num)
        elif rng == "batched":
            idxs, selection = _draw_batched(b, h, w, vn, hn, max_num, dev)
        else:
            raise ValueError(f"unknown rng mode {rng!r}")
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        conf = torch.empty([b, vn], dtype=torch.float32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, hn, dev)
        _native.check(_native.lib().pvnet_ransac_voting_v5(
            _ptr(m), esz, _ptr(v), strides, _ptr(idxs), _ptr(selection), b, h, w, vn, hn,
            float(inlier_thresh), 0.999, int(min_num), int(min(max_num, 2 ** 31 - 1)),
            _ptr(out), _ptr(conf), None, None, None, _ptr(ws), ws_bytes, _stream(dev)), "pvnet_ransac_voting_v5")
    return out, conf


def estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, topk=128,
                                           inlier_thresh=0.99, min_num=5, max_num=30000, output_hyp=False, *,
                                           idxs=None, selection=None, rng="reference", return_debug=False):
    """Reference signature (ransac_voting_gpu.py:333-334).  Returns (mean, cov [b,vn,2,2]).

    mask foreground is `mask == 1` here (:339), not `nonzero` as in v3.  `topk` and
    `output_hyp` are unused by the reference in this variant and are ignored.
    idxs, when injected, is [b, rounds*round_hyp_num, vn, 2] with rounds =
    ceil(min_hyp_num/round_hyp_num).
    """
    del topk, output_hyp
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    rounds = int(math.ceil(min_hyp_num / round_hyp_num))
    hnt = hn * rounds
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_EQUALS_ONE)
    v, strides = _prep_vertex(vertex)
    mean_c = mean.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(mean_c.shape) != (b, vn, 2):
        raise ValueError(f"mean must be [b,vn,2], got {tuple(mean_c.shape)}")
    with torch.cuda.device(dev):
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hnt, dev)
        elif rng == "reference":
            idxs, selection, fg = _draw_reference(m, _MASK_EQUALS_ONE, b, h, w, vn, hn, rounds, min_num, max_num)
            skipped = [f < min_num for f in fg]
            if any(skipped) and not all(skipped) and int(min_hyp_num) != hnt:
                # the reference's torch.cat at :389 fails on this mix (SURVEY App. C.4)
                raise RuntimeError("Sizes of tensors must match except in dimension 0 "
                                   f"(skipped images carry {min_hyp_num} rows, others {hnt})")
        elif rng == "batched":
            idxs, selection = _draw_batched(b, h, w, vn, hnt, max_num, dev)
        else:
            raise ValueError(f"unknown rng mode {rng!r}")
        cov = torch.empty([b, vn, 2, 2], dtype=torch.float32, device=dev)
        counts = hyp = tn = None
        if return_debug:
            counts = torch.empty([b, hnt, vn], dtype=torch.int32, device=dev)
            hyp = torch.empty([b, hnt, vn, 2], dtype=torch.float32, device=dev)
            tn = torch.empty([b], dtype=torch.int32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, hnt, dev)
        _native.check(_native.lib().pvnet_vote_cov_with_mean(
            _ptr(m), esz, _ptr(v), strides, _ptr(idxs), _ptr(selection), _ptr(mean_c), b, h, w, vn, hn, rounds,
            int(min_hyp_num), float(inlier_thresh), int(min_num), int(min(max_num, 2 ** 31 - 1)),
            _ptr(cov), _ptr(counts), _ptr(hyp), _ptr(tn), _ptr(ws), ws_bytes, _stream(dev)),
            "pvnet_vote_cov_with_mean")
    if return_debug:
        return mean, cov, dict(counts=counts, hyp=hyp, tn=tn, idxs=idxs, selection=selection)
    return mean, cov


def generate_hypothesis(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                        min_num=5, max_num=30000, *, idxs=None, selection=None, rng="reference"):
    """Reference ransac_voting_gpu.py:983-1034: the hypotheses [b,hn,vn,2] and their
    inlier counts [b,hn,vn] (int64, as torch.sum of a uint8 tensor gives).  Used by
    tools/demo.py:120-134 (`visualize_hypothesis`).  The reference's skip branch hits a
    NameError (:1003); here an image below min_num contributes zeros."""
    _, dbg = ransac_voting_layer_v3(mask, vertex, round_hyp_num, inlier_thresh, confidence, max_iter, min_num,
                                    max_num, idxs=idxs, selection=selection, rng=rng, return_debug=True)
    return dbg["hyp"], dbg["counts"].long()


# ------------------------------------------------------------------ the other variants of the module
def ransac_motion_voting(mask, vertex):
    """Reference ransac_voting_gpu.py:960-981 (tools/train_linemod.py:117, `MotionEvalWrapper`):
    [b,vn,2] mean over the foreground pixels of vertex + (x, y); zeros for an empty mask."""
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_NONZERO_BYTE)
    v, strides = _prep_vertex(vertex)
    with torch.cuda.device(dev):
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, 1, dev)
        _native.check(_native.lib().pvnet_ransac_motion_voting(_ptr(m), esz, _ptr(v), strides, b, h, w, vn, _ptr(out),
                                                               _ptr(ws), ws_bytes, _stream(dev)),
                      "pvnet_ransac_motion_voting")
    return out


def ransac_voting_layer_v4(mask, vertex, round_hyp_num, inlier_thresh=0.99, confidence=0.999, max_iter=20,
                           min_num=5, max_num=30000, *, idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:669-670).  Returns (keypoints [b,vn,2],
    var [b,vn]): var = mean squared residual n.p - n.c of the refit over the winner's inliers
    (:750-752); skipped images: zeros and var = 1."""
    del confidence, max_iter
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_NONZERO_BYTE)
    v, strides = _prep_vertex(vertex)
    with torch.cuda.device(dev):
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hn, dev)
        elif rng == "reference":
            idxs, selection, _ = _draw_reference(m, _MASK_NONZERO_BYTE, b, h, w, vn, hn, 1, min_num, max_num)
        elif rng == "batched":
            idxs, selection = _draw_batched(b, h, w, vn, hn, max_num, dev)
        else:
            raise ValueError(f"unknown rng mode {rng!r}")
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        var = torch.empty([b, vn], dtype=torch.float32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, hn, dev)
        _native.check(_native.lib().pvnet_ransac_voting_v4(
            _ptr(m), esz, _ptr(v), strides, _ptr(idxs), _ptr(selection), b, h, w, vn, hn,
            float(inlier_thresh), int(min_num), int(min(max_num, 2 ** 31 - 1)),
            _ptr(out), _ptr(var), None, None, None, _ptr(ws), ws_bytes, _stream(dev)), "pvnet_ransac_voting_v4")
    return out, var


def _class_mask(mask, value):
    """`mask == value` as a uint8 tensor (the class-selecting variants: :24, :223, :269)."""
    return (mask == value).to(torch.uint8)


def _draw_reference_classes(mask, class_num, b, h, w, vn, hn, min_num, max_num):
    """The reference's class-selecting layers loop `for bi: for k:` (ransac_voting_gpu.py:23-26, :113-117)
    and draw inside: replay the torch RNG calls in that order.  Returns per-class lists of
    (idxs [b,hn,vn,2], selection [b,h,w] or None)."""
    dev = mask.device
    ncls = int(class_num) - 1
    fgs = [foreground_counts(_class_mask(mask, k + 1)).cpu().tolist() for k in range(ncls)]   # one sync per class
    idxs = [torch.zeros([b, hn, vn, 2], dtype=torch.int32, device=dev) for _ in range(ncls)]
    sels = [None] * ncls
    for bi in range(b):
        for k in range(ncls):
            fg = fgs[k][bi]
            if fg < min_num:
                continue
            tn = fg
            if fg > max_num:
                if sels[k] is None:
                    sels[k] = torch.empty([b, h, w], dtype=torch.float32, device=dev)
                sel = torch.zeros([h, w], dtype=torch.float32, device=dev).uniform_(0, 1)
                sels[k][bi] = sel
                p = max_num / torch.tensor(fg, device=dev).float()
                tn = int(((mask[bi] == k + 1) & (sel < p)).sum().item())
            idxs[k][bi] = torch.zeros([hn, vn, 2], dtype=torch.int32, device=dev).random_(0, max(tn, 1))
    return idxs, sels


def _per_class_v3(mask, vertex, class_num, hn, inlier_thresh, min_num, max_num, idxs, selection, rng):
    """v3 on every class mask; yields (class index, keypoints, debug dict)."""
    b, h, w, vn, _ = vertex.shape
    ncls = int(class_num) - 1
    if idxs is None and rng == "reference" and ncls > 0:
        idxs, selection = _draw_reference_classes(mask, class_num, b, h, w, vn, hn, min_num, max_num)
    for k in range(ncls):
        kp, dbg = ransac_voting_layer_v3(_class_mask(mask, k + 1), vertex, hn, inlier_thresh, min_num=min_num,
                                         max_num=max_num, idxs=None if idxs is None else idxs[k],
                                         selection=None if selection is None else selection[k], rng=rng,
                                         return_debug=True)
        yield k, kp, dbg


def ransac_voting_layer(mask, vertex, class_num, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                        min_num=5, max_num=30000, *, idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:10-11), the first voting layer: for every class
    1..class_num-1 the pixels with mask == class vote and the WINNING HYPOTHESIS (no refit) is
    returned: [b, class_num-1, vn, 2].  idxs / selection, when injected, carry a leading class
    axis: [class_num-1, b, hn, vn, 2] / [class_num-1, b, h, w].  With rng="reference" the torch RNG
    calls are replayed in the reference's (image, class) order."""
    del confidence, max_iter
    b, h, w, vn, _ = vertex.shape
    outs = []
    for _, _, dbg in _per_class_v3(mask, vertex, class_num, int(round_hyp_num), inlier_thresh, min_num, max_num, idxs,
                                   selection, rng):
        counts, hyp = dbg["counts"], dbg["hyp"]                   # [b,hn,vn], [b,hn,vn,2]
        win = torch.argmax(counts, 1)                              # first maximum (:68)
        win_cnt = torch.gather(counts, 1, win[:, None, :])[:, 0]   # [b,vn]
        win_pts = torch.gather(hyp, 1, win[:, None, :, None].expand(b, 1, vn, 2))[:, 0]
        outs.append(torch.where((win_cnt > 0)[..., None], win_pts, torch.zeros_like(win_pts)))   # :74-75
    if not outs:
        return torch.zeros([b, 0, vn, 2], dtype=torch.float32, device=vertex.device)
    return torch.stack(outs, 1)


def ransac_voting_layer_v2(mask, vertex, class_num, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                           min_num=5, max_num=30000, refine_iter_num=1, *, idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:99-100): per class, vote, then `refine_iter_num`
    rounds of (inliers of the current point -> least-squares intersection of their lines): [b, class_num-1,
    vn, 2].  The reference solves each refit with `torch.pinverse(A) @ b` (:198); for a full-rank A that is
    the normal-equation solution v3's refit computes (in fp64 here).  A keypoint without inliers gives
    zeros (:190-192); a rank-deficient inlier set (all lines parallel) gives NaN here, the minimum-norm
    point there."""
    del confidence, max_iter
    b, h, w, vn, _ = vertex.shape
    outs = []
    for k, kp, dbg in _per_class_v3(mask, vertex, class_num, int(round_hyp_num), inlier_thresh, min_num, max_num, idxs,
                                    selection, rng):
        if int(refine_iter_num) < 1:                # no refinement at all: the winning hypothesis (:149-158)
            counts, hyp = dbg["counts"], dbg["hyp"]
            win = torch.argmax(counts, 1)
            kp = torch.gather(hyp, 1, win[:, None, :, None].expand(b, 1, vn, 2))[:, 0]
            kp = torch.where((torch.gather(counts, 1, win[:, None, :])[:, 0] > 0)[..., None], kp, torch.zeros_like(kp))
        for _ in range(int(refine_iter_num) - 1):   # v3 already did the first refit
            kp = refit_at_points(_class_mask(mask, k + 1), vertex, torch.nan_to_num(kp, nan=0.0), inlier_thresh,
                                 min_num=min_num, max_num=max_num, selection=dbg["selection"])
        outs.append(torch.nan_to_num(kp, nan=0.0) if int(refine_iter_num) >= 1 else kp)
    if not outs:
        return torch.zeros([b, 0, vn, 2], dtype=torch.float32, device=vertex.device)
    return torch.stack(outs, 1)


def refit_at_points(mask, vertex, points, inlier_thresh, min_num=5, max_num=30000, *, selection=None):
    """One refinement round of ransac_voting_gpu.py:178-204 for a whole batch: the pixels (mask nonzero)
    that are inliers of points [b,vn,2] re-estimate them by least squares.  Returns [b,vn,2]."""
    _require_cuda(mask, "mask")
    _require_cuda(vertex, "vertex")
    b, h, w, vn, _ = vertex.shape
    dev = mask.device
    m, esz = _prep_mask(mask, _MASK_NONZERO_BYTE)
    v, strides = _prep_vertex(vertex)
    pts = points.to(device=dev, dtype=torch.float32).contiguous()
    if tuple(pts.shape) != (b, vn, 2):
        raise ValueError(f"points must be [b,vn,2], got {tuple(pts.shape)}")
    with torch.cuda.device(dev):
        if selection is not None:
            selection = torch.as_tensor(selection, device=dev, dtype=torch.float32).contiguous()
        out = torch.empty([b, vn, 2], dtype=torch.float32, device=dev)
        ws, ws_bytes = _workspace(b, h, w, vn, 1, dev)
        _native.check(_native.lib().pvnet_refit_at_points(
            _ptr(m), esz, _ptr(v), strides, _ptr(selection), _ptr(pts), b, h, w, vn, float(inlier_thresh), int(min_num),
            int(min(max_num, 2 ** 31 - 1)), _ptr(out), _ptr(ws), ws_bytes, _stream(dev)), "pvnet_refit_at_points")
    return out


def ransac_voting_vanish_point_layer(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20,
                                     min_num=5, max_num=30000, refine_iter_num=1, *, class_num=2, idxs=None):
    """Reference ransac_voting_gpu.py:408-501 (its body reads an undefined `class_num`, :415, so it cannot
    run as written; it is a keyword here, default 2 = one foreground class).  Per class: homogeneous
    hypotheses from pixel pairs (`generate_hypothesis_vanishing_point`), |cos| vote, the winner normalised,
    then `refine_iter_num` rounds of (inliers -> smallest right singular vector of [-n | n.c], sign fixed by
    the first inlier, :485-492).  Returns [b, class_num-1, vn, 3].  The two kernels are the native
    stand-ins (bit-exact to the reference's); compaction, argmax and SVD are the reference's torch ops --
    this layer is off the hot path (only commented-out code calls it, :1083).
    idxs, when injected: [b, class_num-1, hn, vn, 2]."""
    from . import ransac_voting as ext
    del confidence, max_iter
    _require_cuda(mask, "mask")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    dev = mask.device
    out = torch.zeros([b, int(class_num) - 1, vn, 3], dtype=torch.float32, device=dev)
    for bi in range(b):
        for k in range(int(class_num) - 1):
            cur_mask = mask[bi] == k + 1
            fg = int(cur_mask.sum())
            if fg < min_num:
                continue
            if fg > max_num:
                sel = torch.zeros(cur_mask.shape, dtype=torch.float32, device=dev).uniform_(0, 1)
                cur_mask = cur_mask & (sel < (max_num / torch.tensor(fg, device=dev).float()))
            coords = torch.nonzero(cur_mask).float()[:, [1, 0]].contiguous()
            direct = vertex[bi][cur_mask].reshape(-1, vn, 2).contiguous().float()
            tn = coords.shape[0]
            if idxs is not None:
                cur_idxs = torch.as_tensor(idxs[bi][k], device=dev).to(torch.int32).contiguous()
            else:
                cur_idxs = torch.zeros([hn, vn, 2], dtype=torch.int32, device=dev).random_(0, tn)
            hyp = ext.generate_hypothesis_vanishing_point(direct, coords, cur_idxs)                 # [hn,vn,3]
            counts = ext.voting_for_hypothesis_vanishing_point(direct, coords, hyp, None, inlier_thresh,
                                                               return_counts=True)                  # [hn,vn]
            hyp = hyp / torch.norm(hyp, 2, 2, keepdim=True)                                         # :446
            win = torch.argmax(counts, 0)
            win_pts = hyp[win, torch.arange(vn, device=dev)]
            pts = torch.where((counts.max(0).values > 0)[:, None], win_pts, torch.zeros_like(win_pts))
            normal = torch.stack([direct[:, :, 1], -direct[:, :, 0]], 2)
            for _ in range(int(refine_iter_num)):
                inl = torch.zeros([1, vn, tn], dtype=torch.uint8, device=dev)
                ext.voting_for_hypothesis_vanishing_point(direct, coords, pts[None].contiguous(), inl, inlier_thresh)
                new = []
                for vi in range(vn):
                    sel_v = inl[0, vi].bool()
                    if int(sel_v.sum()) == 0:
                        new.append(pts[vi:vi + 1])
                        continue
                    cc, nn = coords[sel_v], normal[:, vi][sel_v]
                    H = torch.cat([-nn, (nn * cc).sum(1, keepdim=True)], 1)                          # :485
                    _, _, Vh = torch.linalg.svd(H, full_matrices=False)
                    p = Vh[2:3]
                    if float((p[0, 0] - p[0, 2] * cc[0, 0]) * (-nn[0, 1])) < 0:                      # :489-490
                        p = -p
                    new.append(p)
                pts = torch.cat(new, 0)
            out[bi, k] = pts
    return out


def ransac_voting_hypothesis(mask, vertex, round_hyp_num, inlier_thresh=0.999, min_num=5, max_num=30000, *,
                             idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:218): hypotheses [b,hn,vn,2] and int64 inlier
    counts [b,hn,vn] of the pixels with mask == 1; a skipped image has zero hypotheses and
    counts of one (:228-233)."""
    _, dbg = ransac_voting_layer_v3(_class_mask(mask, 1), vertex, round_hyp_num, inlier_thresh, min_num=min_num,
                                    max_num=max_num, idxs=idxs, selection=selection, rng=rng, return_debug=True)
    counts = dbg["counts"].long()
    skipped = (dbg["tn"] == 0)[:, None, None]
    return dbg["hyp"], torch.where(skipped, torch.ones_like(counts), counts)


def estimate_voting_distribution(mask, vertex, round_hyp_num=256, min_hyp_num=4096, topk=128, inlier_thresh=0.99,
                                 min_num=5, max_num=30000, *, idxs=None, selection=None, rng="reference"):
    """Reference signature (ransac_voting_gpu.py:263-264): (mean [b,vn,2], cov [b,vn,2,2]) of
    the top-k hypotheses per keypoint weighted by their inlier ratio.  The hypotheses and
    counts come from the vote kernels; the top-k / moment arithmetic on the [b,vn,hn] result is
    the reference's own torch expression (:315-325) evaluated on the device."""
    _require_cuda(mask, "mask")
    b, h, w, vn, _ = vertex.shape
    hn = int(round_hyp_num)
    rounds = int(math.ceil(min_hyp_num / hn))
    dev = mask.device
    m = _class_mask(mask, 1)
    with torch.cuda.device(dev):
        if idxs is not None:
            idxs, selection = _check_injected(idxs, selection, b, h, w, vn, hn * rounds, dev)
        elif rng == "reference":
            idxs, selection, _ = _draw_reference(m, _MASK_NONZERO_BYTE, b, h, w, vn, hn, rounds, min_num, max_num)
        elif rng == "batched":
            idxs, selection = _draw_batched(b, h, w, vn, hn * rounds, max_num, dev)
        else:
            raise ValueError(f"unknown rng mode {rng!r}")
        _, dbg = ransac_voting_layer_v3(m, vertex, hn * rounds, inlier_thresh, min_num=min_num, max_num=max_num,
                                        idxs=idxs, selection=selection, return_debug=True)
        tn = dbg["tn"].float()[:, None, None]
        ratio = torch.where(tn > 0, dbg["counts"].float() / tn.clamp(min=1), torch.ones_like(tn))   # :276, :302
        hyp = dbg["hyp"].permute(0, 2, 1, 3)                       # [b,vn,hn,2]   :313
        ratio = ratio.permute(0, 2, 1)                             # [b,vn,hn]     :314
        values, indexes = torch.topk(ratio, min(int(topk), ratio.shape[2]), dim=2, sorted=False)
        ratio = torch.zeros_like(ratio).scatter_(2, indexes, values)
        wsum = torch.sum(ratio, 2)
        mean = torch.sum(ratio[..., None] * hyp, 2) / wsum[..., None]
        diff = hyp - mean[:, :, None]
        cov = torch.matmul(diff.transpose(2, 3), diff * ratio[..., None]) / wsum[..., None, None]
    return mean, cov
