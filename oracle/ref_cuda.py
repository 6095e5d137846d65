"""The reference's own CUDA voting layer, run on the GPU -- TEST INFRASTRUCTURE ONLY.

`oracle/_ref/libpvnet_refcuda.so` is the reference project's lib/ransac_voting_gpu_layer/src/
ransac_voting_kernel.cu compiled verbatim (oracle/Makefile, target `ref`) plus our C shim
(oracle/ref_shim.cu).  This module binds it with ctypes and re-states, with the torch
ops the reference uses and in the reference's order, the Python orchestration of

    ransac_voting_layer_v3                   ransac_voting_gpu.py:514-598
    estimate_voting_distribution_with_mean   ransac_voting_gpu.py:333-406

with the two edits torch 2.x forces (SURVEY.md §8c): `masked_select` needs a bool mask
(the reference passes uint8, :544) and `torch.gesv` (:511) no longer exists, so the 2x2
inverse is `torch.linalg.solve(A, I)` (LU with partial pivoting, as gesv was).
Everything it produces is "the reference run here": tests use it to pin the oracle and
to measure the product's distance from the reference CUDA layer.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libpvnet_refcuda.so")
_lib = None


def available() -> bool:
    return os.path.exists(LIB_PATH) and torch.cuda.is_available()


def lib():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(LIB_PATH)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.pvref_generate_hypothesis.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci]
        L.pvref_generate_hypothesis.restype = ci
        L.pvref_voting_for_hypothesis.argtypes = [vp, vp, vp, vp, ci, ci, ci, ctypes.c_float, ci]
        L.pvref_voting_for_hypothesis.restype = ci
        if hasattr(L, "pvref_generate_hypothesis_vp"):
            L.pvref_generate_hypothesis_vp.argtypes = [vp, vp, vp, vp, ci, ci, ci, ci]
            L.pvref_generate_hypothesis_vp.restype = ci
            L.pvref_voting_for_hypothesis_vp.argtypes = [vp, vp, vp, vp, ci, ci, ci, ctypes.c_float, ci]
            L.pvref_voting_for_hypothesis_vp.restype = ci
        _lib = L
    return _lib


def _dev(t):
    return t.device.index if t.device.index is not None else torch.cuda.current_device()


def generate_hypothesis(direct, coords, idxs):
    """ransac_voting.cpp:20-31 -> ransac_voting_kernel.cu:51-86"""
    assert direct.is_cuda and direct.is_contiguous() and coords.is_contiguous() and idxs.is_contiguous()
    tn, vn, _ = direct.shape
    hn = idxs.shape[0]
    torch.cuda.synchronize()
    out = torch.empty([hn, vn, 2], dtype=torch.float32, device=direct.device)
    rc = lib().pvref_generate_hypothesis(direct.data_ptr(), coords.data_ptr(), idxs.data_ptr(), out.data_ptr(),
                                         tn, vn, hn, _dev(direct))
    if rc != 0:
        raise RuntimeError(f"pvref_generate_hypothesis -> {rc}")
    return out


def voting_for_hypothesis(direct, coords, hypo, inliers, thresh):
    """ransac_voting.cpp:41-55 -> ransac_voting_kernel.cu:129-167"""
    assert direct.is_cuda and hypo.is_contiguous() and inliers.is_contiguous() and inliers.dtype == torch.uint8
    tn, vn, _ = direct.shape
    hn = hypo.shape[0]
    torch.cuda.synchronize()
    rc = lib().pvref_voting_for_hypothesis(direct.data_ptr(), coords.data_ptr(), hypo.data_ptr(),
                                           inliers.data_ptr(), tn, vn, hn, float(thresh), _dev(direct))
    if rc != 0:
        raise RuntimeError(f"pvref_voting_for_hypothesis -> {rc}")


def generate_hypothesis_vanishing_point(direct, coords, idxs):
    """ransac_voting.cpp:61-72 -> ransac_voting_kernel.cu:232-260"""
    tn, vn, _ = direct.shape
    hn = idxs.shape[0]
    torch.cuda.synchronize()
    out = torch.empty([hn, vn, 3], dtype=torch.float32, device=direct.device)
    rc = lib().pvref_generate_hypothesis_vp(direct.data_ptr(), coords.data_ptr(), idxs.data_ptr(), out.data_ptr(),
                                            tn, vn, hn, _dev(direct))
    if rc != 0:
        raise RuntimeError(f"pvref_generate_hypothesis_vp -> {rc}")
    return out


def voting_for_hypothesis_vanishing_point(direct, coords, hypo, inliers, thresh):
    """ransac_voting.cpp:82-96 -> ransac_voting_kernel.cu:307-351"""
    tn, vn, _ = direct.shape
    hn = hypo.shape[0]
    torch.cuda.synchronize()
    rc = lib().pvref_voting_for_hypothesis_vp(direct.data_ptr(), coords.data_ptr(), hypo.data_ptr(), inliers.data_ptr(),
                                              tn, vn, hn, float(thresh), _dev(direct))
    if rc != 0:
        raise RuntimeError(f"pvref_voting_for_hypothesis_vp -> {rc}")


def _inverse_2x2(mats):
    eye = torch.eye(2, dtype=mats.dtype, device=mats.device).expand_as(mats)
    return torch.linalg.solve(mats, eye)


def _select_pixels(cur_mask_u8, vertex_img, vn):
    coords = torch.nonzero(cur_mask_u8).float()[:, [1, 0]].contiguous()
    sel = cur_mask_u8.bool()[:, :, None, None]
    direct = vertex_img.masked_select(sel).view([coords.shape[0], vn, 2]).contiguous()
    return coords, direct


def layer_v3(mask, vertex, round_hyp_num, inlier_thresh=0.999, confidence=0.99, max_iter=20, min_num=5,
             max_num=30000, record=None, refit_dtype=torch.float32):
    """The reference's v3, torch op for torch op (RNG calls included).  `record`, if a list,
    receives per-image dicts (idxs, counts, tn, selection) for the parity tests.
    refit_dtype=torch.float64 runs the SAME least-squares refit ops (:578-595) in double:
    the difference to the float32 run is the reference's own rounding noise (cuBLAS /
    torch.sum fp32 summation order), which no other implementation can reproduce."""
    b, h, w, vn, _ = vertex.shape
    dev = mask.device
    results = []
    for bi in range(b):
        rec = {}
        total_hyp = 0
        cur_mask = mask[bi].byte()
        n_fg = torch.sum(cur_mask)
        if n_fg < min_num:
            results.append(torch.zeros([1, vn, 2], dtype=torch.float32, device=dev))
            if record is not None:
                record.append(None)
            continue
        if n_fg > max_num:
            field = torch.zeros(cur_mask.shape, dtype=torch.float32, device=dev).uniform_(0, 1)
            keep = field < (max_num / n_fg.float())
            cur_mask *= keep
            rec["selection"] = field
        coords, direct = _select_pixels(cur_mask, vertex[bi], vn)
        tn = coords.shape[0]
        idxs = torch.zeros([round_hyp_num, vn, 2], dtype=torch.int32, device=dev).random_(0, direct.shape[0])
        best_ratio = torch.zeros([vn], dtype=torch.float32, device=dev)
        best_pts = torch.zeros([vn, 2], dtype=torch.float32, device=dev)
        rounds = 0
        while True:
            hyp = generate_hypothesis(direct, coords, idxs)
            inl = torch.zeros([round_hyp_num, vn, tn], dtype=torch.uint8, device=dev)
            voting_for_hypothesis(direct, coords, hyp, inl, inlier_thresh)
            counts = torch.sum(inl, 2)
            top_counts, top_idx = torch.max(counts, 0)
            top_pts = hyp[top_idx, torch.arange(vn, device=dev)]
            top_ratio = top_counts.float() / tn
            better = best_ratio < top_ratio
            best_pts[better, :] = top_pts[better, :]
            best_ratio[better] = top_ratio[better]
            total_hyp += round_hyp_num
            rounds += 1
            if rounds == 1:
                rec.update(idxs=idxs, counts=counts.clone(), hyp=hyp.clone(), tn=tn)
            lowest = torch.min(best_ratio)
            if (1 - (1 - lowest ** 2) ** total_hyp) > confidence or rounds > max_iter:
                break
        normal = torch.zeros_like(direct)
        normal[:, :, 0] = direct[:, :, 1]
        normal[:, :, 1] = -direct[:, :, 0]
        final_inl = torch.zeros([1, vn, tn], dtype=torch.uint8, device=dev)
        voting_for_hypothesis(direct, coords, best_pts[None].contiguous(), final_inl, inlier_thresh)
        wgt = final_inl.to(refit_dtype)[0]                      # [vn,tn]
        normal = normal.to(refit_dtype).permute(1, 0, 2) * wgt[:, :, None]      # [vn,tn,2]
        rhs = torch.sum(normal * coords.to(refit_dtype)[None], 2)               # [vn,tn]
        ata = torch.matmul(normal.permute(0, 2, 1), normal)     # [vn,2,2]
        atb = torch.sum(normal * rhs[:, :, None], 1)            # [vn,2]
        pts = torch.matmul(_inverse_2x2(ata), atb[:, :, None])  # [vn,2,1]
        results.append(pts[None, :, :, 0].float())
        rec["rounds"] = rounds
        if record is not None:
            record.append(rec)
    return torch.cat(results)


def layer_cov_with_mean(mask, vertex, mean, round_hyp_num=256, min_hyp_num=4096, inlier_thresh=0.99, min_num=5,
                        max_num=30000, record=None):
    """The reference's estimate_voting_distribution_with_mean, torch op for torch op."""
    b, h, w, vn, _ = vertex.shape
    dev = mask.device
    hyp_all, ratio_all = [], []
    for bi in range(b):
        cur_mask = mask[bi] == 1
        n_fg = torch.sum(cur_mask)
        if n_fg < min_num:
            hyp_all.append(torch.zeros([1, min_hyp_num, vn, 2], dtype=torch.float32, device=dev))
            ratio_all.append(torch.ones([1, min_hyp_num, vn], dtype=torch.int64, device=dev).float())
            if record is not None:
                record.append(None)
            continue
        rec = {}
        if n_fg > max_num:
            field = torch.zeros(cur_mask.shape, dtype=torch.float32, device=dev).uniform_(0, 1)
            cur_mask = cur_mask * (field < (max_num / n_fg.float()))
            n_fg = torch.sum(cur_mask)
            rec["selection"] = field
        coords, direct = _select_pixels(cur_mask.byte(), vertex[bi], vn)
        tn = coords.shape[0]
        hyps, ratios, all_idxs, all_counts = [], [], [], []
        for _ in range(int(np.ceil(min_hyp_num / round_hyp_num))):
            idxs = torch.zeros([round_hyp_num, vn, 2], dtype=torch.int32, device=dev).random_(0, direct.shape[0])
            hyp = generate_hypothesis(direct, coords, idxs)
            inl = torch.zeros([round_hyp_num, vn, tn], dtype=torch.uint8, device=dev)
            voting_for_hypothesis(direct, coords, hyp, inl, inlier_thresh)
            cnt = torch.sum(inl, 2)
            hyps.append(hyp)
            ratios.append(cnt.float() / n_fg.float())
            all_idxs.append(idxs)
            all_counts.append(cnt)
        hyp_all.append(torch.cat(hyps, 0)[None])
        ratio_all.append(torch.cat(ratios, 0)[None])
        rec.update(idxs=torch.cat(all_idxs, 0), counts=torch.cat(all_counts, 0), tn=tn)
        if record is not None:
            record.append(rec)
    hyp_all = torch.cat(hyp_all, 0).permute(0, 2, 1, 3)      # b,vn,hn,2
    ratio_all = torch.cat(ratio_all, 0).permute(0, 2, 1)     # b,vn,hn
    cut = torch.max(ratio_all, 2)[0] - 0.1
    ratio_all[ratio_all < cut[:, :, None]] = 0.0
    diff = hyp_all - mean[:, :, None]
    wdiff = diff * ratio_all[:, :, :, None]
    cov = torch.matmul(diff.transpose(2, 3), wdiff)
    cov /= torch.sum(ratio_all, 2)[:, :, None, None] + 1e-3
    return mean, cov
