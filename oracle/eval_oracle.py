"""CPU oracle for the pose metrics -- TEST INFRASTRUCTURE ONLY.

An fp64 numpy restatement of what `pvnet_pose_metrics` (pvnet_b200/csrc/eval.cu) computes, written from the
metric definitions of the reference's lib/utils/evaluation_utils.py:75-141 (ADD, ADD-S, 2-D projection error,
5 cm 5 degree), in the operation order the kernel fixes:

    p_r  = ((R[r,0] X + R[r,1] Y) + R[r,2] Z) + t[r]                  (every product and sum rounded once)
    h_r  = (K[r,0] p_0 + K[r,1] p_1) + K[r,2] p_2,   uv = (h_0 / h_2, h_1 / h_2)
    tr   = sum_r ((Rp[r,0] Rg[r,0] + Rp[r,1] Rg[r,1]) + Rp[r,2] Rg[r,2])   (summed over r = 0, 1, 2)

numpy's elementwise float64 operations round once each and never fuse, so the fp32 roundings the nearest-point
search runs on are bit-equal to the kernel's, and so are the ADD-S indices.  The search itself is the C oracle
`pvo_find_nearest_point_idx` (oracle/eval_oracle.c).  Only the means are summed in another order (np.mean), which
is why distances agree to ~1e-12 relative rather than bit for bit.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libpvnet_eval_oracle.so")
_F32P = ctypes.POINTER(ctypes.c_float)
_I32P = ctypes.POINTER(ctypes.c_int32)
_lib_handle = None


def build(force: bool = False) -> str:
    """Compile eval_oracle.c (oracle/eval.mk) if the .so is missing or stale."""
    src = os.path.join(_HERE, "eval_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-f", os.path.join(_HERE, "eval.mk"), "oracle"])
    return _LIB_PATH


def _lib():
    global _lib_handle
    if _lib_handle is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        L.pvo_find_nearest_point_idx.argtypes = [_F32P, _F32P, _I32P] + [ctypes.c_int] * 4
        L.pvo_find_nearest_point_idx.restype = None
        _lib_handle = L
    return _lib_handle


def find_nearest_point_idx(ref_pts, que_pts):
    """ref [pn1,dim] or [b,pn1,dim], que [pn2,dim] or [b,pn2,dim] (float32) -> int32 [pn2] or [b,pn2]."""
    ref = np.ascontiguousarray(ref_pts, np.float32)
    que = np.ascontiguousarray(que_pts, np.float32)
    single = ref.ndim == 2
    if single:
        ref, que = ref[None], que[None]
    b, pn1, dim = ref.shape
    pn2 = que.shape[1]
    assert que.shape == (b, pn2, dim) and dim in (2, 3)
    out = np.zeros((b, pn2), np.int32)
    _lib().pvo_find_nearest_point_idx(ref.ctypes.data_as(_F32P), que.ctypes.data_as(_F32P),
                                      out.ctypes.data_as(_I32P), b, pn1, pn2, dim)
    return out[0] if single else out


def _rows(A, x, y, z):
    """(A[r,0] x + A[r,1] y) + A[r,2] z for r = 0, 1, 2."""
    return [(A[r, 0] * x + A[r, 1] * y) + A[r, 2] * z for r in range(3)]


def transform(pose, model):
    """pose [3,4] f64, model [n,3] -> [n,3] f64, the kernel's order."""
    X = np.asarray(model, np.float64)
    pose = np.asarray(pose, np.float64)
    r = _rows(pose[:, :3], X[:, 0], X[:, 1], X[:, 2])
    return np.stack([r[i] + pose[i, 3] for i in range(3)], 1)


def project(K, p):
    """K [3,3] f64, p [n,3] -> uv [n,2], the kernel's order."""
    h = _rows(np.asarray(K, np.float64), p[:, 0], p[:, 1], p[:, 2])
    return np.stack([h[0] / h[2], h[1] / h[2]], 1)


def _norm(d):
    s = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]
    if d.shape[1] == 3:
        s = s + d[:, 2] * d[:, 2]
    return np.sqrt(s)


def pose_metrics_one(pose_pred, pose_gt, model, K, symmetric=False, sym_proj=False):
    """One image -> (array [4] = add, proj, trans_cm, angle_deg; dict of the ADD-S / 2-D search indices)."""
    pose_pred = np.asarray(pose_pred, np.float64)
    pose_gt = np.asarray(pose_gt, np.float64)
    P, G = transform(pose_pred, model), transform(pose_gt, model)
    Pu, Gu = project(K, P), project(K, G)
    idx = {}
    if symmetric:
        idx["add"] = find_nearest_point_idx(P.astype(np.float32), G.astype(np.float32))
        add = np.mean(_norm(P[idx["add"]] - G))
    else:
        add = np.mean(_norm(P - G))
    if sym_proj:
        idx["proj"] = find_nearest_point_idx(Pu.astype(np.float32), Gu.astype(np.float32))
        proj = np.mean(_norm(Pu[idx["proj"]] - Gu))
    else:
        proj = np.mean(_norm(Pu - Gu))
    dt = (pose_pred[:, 3] - pose_gt[:, 3])[None]
    trans = _norm(dt)[0] * 100.0
    Rp, Rg = pose_pred[:, :3], pose_gt[:, :3]
    tr = 0.0
    for r in range(3):
        tr = tr + ((Rp[r, 0] * Rg[r, 0] + Rp[r, 1] * Rg[r, 1]) + Rp[r, 2] * Rg[r, 2])
    tr = tr if tr <= 3 else 3.0
    with np.errstate(invalid="ignore"):
        ang = np.rad2deg(np.arccos((tr - 1.0) / 2.0))
    return np.array([add, proj, trans, ang]), idx


def pose_metrics(pose_pred, pose_gt, model, K, symmetric=False, sym_proj=False):
    """Batched: poses [b,3,4], K [3,3] or [b,3,3] -> [b,4]."""
    pose_pred = np.asarray(pose_pred, np.float64)
    K = np.asarray(K, np.float64)
    out = []
    for i in range(pose_pred.shape[0]):
        Ki = K[i] if K.ndim == 3 else K
        out.append(pose_metrics_one(pose_pred[i], pose_gt[i], model, Ki, symmetric, sym_proj)[0])
    return np.stack(out)


def passes(metrics, diameter):
    """The reference's three decisions from [b,4] metrics: (add < diameter*0.1, proj < 5, trans < 5 and ang < 5)."""
    m = np.asarray(metrics)
    return m[:, 0] < diameter * 0.1, m[:, 1] < 5, (m[:, 2] < 5) & (m[:, 3] < 5)


# ------------------------------------------------------------------ the reference's own kernel (oracle/_ref)
REF_NN_PATH = os.path.join(_HERE, "_ref", "libpvnet_refnn.so")
_ref_nn = None


def ref_nn_available() -> bool:
    return os.path.exists(REF_NN_PATH)


def ref_find_nearest_point_idx(ref_pts, que_pts):
    """The reference's findNearestPointIdxLauncher (nearest_neighborhood.cu:123-163, compiled verbatim into
    oracle/_ref/libpvnet_refnn.so by oracle/eval.mk): host arrays [b,pn1,dim], [b,pn2,dim] -> int32 [b,pn2].
    Needs a GPU; the launcher allocates, copies and synchronises itself."""
    global _ref_nn
    if _ref_nn is None:
        L = ctypes.CDLL(REF_NN_PATH)
        L.findNearestPointIdxLauncher.argtypes = [_F32P, _F32P, _I32P] + [ctypes.c_int] * 5
        L.findNearestPointIdxLauncher.restype = None
        _ref_nn = L
    ref = np.ascontiguousarray(ref_pts, np.float32)
    que = np.ascontiguousarray(que_pts, np.float32)
    b, pn1, dim = ref.shape
    pn2 = que.shape[1]
    out = np.zeros((b, pn2), np.int32)
    _ref_nn.findNearestPointIdxLauncher(ref.ctypes.data_as(_F32P), que.ctypes.data_as(_F32P),
                                        out.ctypes.data_as(_I32P), b, pn1, pn2, dim, 0)
    return out
