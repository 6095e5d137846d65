"""CPU oracle for farthest point sampling and binary mesh rasterisation -- TEST INFRASTRUCTURE ONLY.

`extend_oracle.c` restates the reference's lib/utils/extend_utils/src/farthest_point_sampling.cpp and
mesh_rasterization.cpp one rounded operation at a time (DESIGN.md §11); this module builds it on first use
(oracle/extend.mk) and binds it.  The `ref_*` functions call the reference's own code, compiled verbatim into
oracle/_ref/libpvnet_refextend.so by `make -f oracle/extend.mk ref` (build() does so when PVNET_REFERENCE names a
checkout); tests/golden/make_golden_ref_extend.py records their outputs.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libpvnet_extend_oracle.so")
REF_LIB_PATH = os.path.join(_HERE, "_ref", "libpvnet_refextend.so")
_F32P = ctypes.POINTER(ctypes.c_float)
_I32P = ctypes.POINTER(ctypes.c_int32)
_U8P = ctypes.POINTER(ctypes.c_uint8)
_lib_handle = None
_ref_handle = None


def build(force: bool = False) -> str:
    """Compile extend_oracle.c (oracle/extend.mk) if the .so is missing or stale."""
    src = os.path.join(_HERE, "extend_oracle.c")
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-f", os.path.join(_HERE, "extend.mk"), "oracle"])
    return _LIB_PATH


def _lib():
    global _lib_handle
    if _lib_handle is None:
        build()
        L = ctypes.CDLL(_LIB_PATH)
        L.pvo_farthest_point_sampling.argtypes = [_F32P, _I32P] + [ctypes.c_int] * 3 + [_I32P]
        L.pvo_farthest_point_sampling.restype = None
        L.pvo_mesh_binary_rasterization.argtypes = [_F32P] + [ctypes.c_int] * 4 + [_U8P]
        L.pvo_mesh_binary_rasterization.restype = None
        _lib_handle = L
    return _lib_handle


def farthest_point_sampling(pts, sn, start=None):
    """pts [pn,3] or [b,pn,3]; start: None (init_center) or int / int array [b] -> int32 indices [sn] or [b,sn]."""
    p = np.ascontiguousarray(pts, np.float32)
    single = p.ndim == 2
    if single:
        p = p[None]
    b, pn, _ = p.shape
    out = np.zeros((b, sn), np.int32)
    st = None if start is None else np.ascontiguousarray(np.broadcast_to(np.asarray(start, np.int32), (b,)))
    _lib().pvo_farthest_point_sampling(p.ctypes.data_as(_F32P), None if st is None else st.ctypes.data_as(_I32P),
                                       b, pn, sn, out.ctypes.data_as(_I32P))
    return out[0] if single else out


def mesh_binary_rasterization(triangles, h, w):
    """triangles [tn,3,2] or [b,tn,3,2] -> uint8 mask [h,w] or [b,h,w]."""
    t = np.ascontiguousarray(triangles, np.float32)
    single = t.ndim == 3
    if single:
        t = t[None]
    b, tn = t.shape[:2]
    out = np.empty((b, h, w), np.uint8)
    _lib().pvo_mesh_binary_rasterization(t.ctypes.data_as(_F32P), b, tn, h, w, out.ctypes.data_as(_U8P))
    return out[0] if single else out


# ------------------------------------------------------------------ the reference's own code (oracle/_ref)
def ref_available() -> bool:
    return os.path.exists(REF_LIB_PATH)


def _ref():
    global _ref_handle
    if _ref_handle is None:
        L = ctypes.CDLL(REF_LIB_PATH)
        for name in ("farthest_point_sampling", "farthest_point_sampling_init_center"):
            getattr(L, name).argtypes = [_F32P, _I32P, ctypes.c_int, ctypes.c_int]
            getattr(L, name).restype = None
        L.mesh_binary_rasterization.argtypes = [_F32P, _U8P, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.mesh_binary_rasterization.restype = None
        L.pvnet_ref_set_start.argtypes = [ctypes.c_int]
        L.pvnet_ref_set_start.restype = None
        _ref_handle = L
    return _ref_handle


def ref_farthest_point_sampling(pts, sn, start=None):
    """The reference's farthest_point_sampling[_init_center] on one cloud [pn,3]; start (>= 0) is what its rand()
    returns, None selects the init_center mode.  -> int32 [sn]."""
    p = np.ascontiguousarray(pts, np.float32)
    idxs = np.zeros(sn, np.int32)
    L = _ref()
    if start is None:
        L.farthest_point_sampling_init_center(p.ctypes.data_as(_F32P), idxs.ctypes.data_as(_I32P), p.shape[0], sn)
    else:
        L.pvnet_ref_set_start(int(start))
        L.farthest_point_sampling(p.ctypes.data_as(_F32P), idxs.ctypes.data_as(_I32P), p.shape[0], sn)
    return idxs


def ref_mesh_binary_rasterization(triangles, h, w):
    """The reference's mesh_binary_rasterization on [tn,3,2] -> uint8 [h,w] (zero-initialised, as extend_utils.py
    does)."""
    t = np.ascontiguousarray(triangles, np.float32)
    mask = np.zeros((h, w), np.uint8)
    _ref().mesh_binary_rasterization(t.ctypes.data_as(_F32P), mask.ctypes.data_as(_U8P), t.shape[0], h, w)
    return mask
