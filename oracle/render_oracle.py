"""numpy restatement of `pvnet_render_mesh` (csrc/render.cu, DESIGN.md §24): depth and flat-shaded RGB of a mesh at a
batch of poses, with the reference OpenGL backend's conventions (lib/utils/opengl_render_backend.py `render`).

The contract, which the kernel follows bit for bit:

* Output pixel (r, c) samples the OpenCV image point p = (c + 0.5, r + 0.5, 1), where u = fx X/Z + s Y/Z + cx and
  v = fy Y/Z + cy.  That is what the reference's y-down `_compute_calib_proj`, the yz flip of its view matrix, GL's
  viewport transform and the `[::-1]` row flip on readback give together.
* Vertices, R, t, K, the clip planes and the ambient weight are fp32 (what the reference hands to GL); everything
  after is fp64, one rounding per operation, in the order written below (numpy never fuses a multiply and an add).
* V_i = ((R[r,0] x + R[r,1] y) + R[r,2] z) + t[r];  h_i = ((fx X + s Y) + cx Z, fy Y + cy Z, Z).
* Edge i (opposite vertex i, between the next two vertices j, k): c_i = h_j x h_k when index_j < index_k, else
  -(h_k x h_j), so faces that share an edge get exactly opposite edge values.  x is
  (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0).
* A face covers nothing when an index is outside [0, nv), two indices are equal, an h_i is not finite, or
  D = c_0 . h_0 is 0 or not finite.  a . b = (a0 b0 + a1 b1) + a2 b2.
* E_i = (c_i0 px + c_i1 py) + c_i2, S = (E_0 + E_1) + E_2, lambda_i = E_i / S, Z = (l0 Z0 + l1 Z1) + l2 Z2.  Covered:
  S != 0, every E_i is 0 or has the sign of S, and near <= Z <= far.
* The winner is the covering face with the smallest (fp32(Z), face index); depth is its fp32(Z), 0 where none.
* Flat RGB: m = (V1 - V0) x (V2 - V0), negated when m . V0 > 0 (turned toward the camera); n = m / sqrt(m . m).
  u_i = -(V_i / sqrt(V_i . V_i)); L = sum lambda_i u_i (in the order of Z), L = L / sqrt(L . L).
  light_w = min(ambient + max(L . n, 0), 1); colour_ch = light_w * ((l0 c0 + l1 c1) + l2 c2) with c from `colors`
  (0.5 when None); stored as fp32, then rint(fp32 * 255) (half to even) clamped to [0, 255], NaN to 0.  Uncovered
  pixels get bg through the same fp32 rounding.

Every face is evaluated at every pixel: no bounding box.  CPU only; nothing here reads the reference.
"""
from __future__ import annotations

import numpy as np


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def to_u8(x):
    """np.round(fp32(x) * 255) as uint8, clamped to [0, 255], NaN to 0."""
    r = np.rint(np.asarray(x).astype(np.float32) * np.float32(255))
    return np.where(r >= 255, 255, np.where(r > 0, r, 0)).astype(np.uint8)


def camera_vertices(verts, pose, K):
    """fp32 inputs -> camera-space V [nv,3] and homogeneous image points h [nv,3], fp64."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    P = np.asarray(pose, np.float32).astype(np.float64).reshape(3, 4)
    k = np.asarray(K, np.float32).astype(np.float64).reshape(3, 3)
    V = np.stack([((P[r, 0] * v[:, 0] + P[r, 1] * v[:, 1]) + P[r, 2] * v[:, 2]) + P[r, 3] for r in range(3)], -1)
    h = np.stack([(k[0, 0] * V[:, 0] + k[0, 1] * V[:, 1]) + k[0, 2] * V[:, 2],
                  k[1, 1] * V[:, 1] + k[1, 2] * V[:, 2], V[:, 2]], -1)
    return V, h


def face_setup(faces, nv, h):
    """-> edge vectors c [nf,3,3] (c[:, i] opposite vertex i), valid [nf], clamped indices [nf,3]."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    inr = ((f >= 0) & (f < nv)).all(1)
    fi = np.where(inr[:, None], f, 0)
    distinct = (fi[:, 0] != fi[:, 1]) & (fi[:, 1] != fi[:, 2]) & (fi[:, 0] != fi[:, 2])
    hf = h[fi] if nv else np.zeros((len(f), 3, 3))
    c = np.empty((len(f), 3, 3))
    for i in range(3):
        j, k = (i + 1) % 3, (i + 2) % 3
        fwd = fi[:, j] < fi[:, k]
        c[:, i] = np.where(fwd[:, None], _cross(hf[:, j], hf[:, k]), -_cross(hf[:, k], hf[:, j]))
    with np.errstate(invalid="ignore", over="ignore"):
        D = _dot(c[:, 0], hf[:, 0])
        ok = inr & distinct & np.isfinite(hf).all((1, 2)) & np.isfinite(D) & (D != 0)
    return c, ok, fi


def fragments(c, z, px, py, nearp, farp):
    """c [...,3,3], z [...,3] against pixel centres px, py (broadcastable) -> covered, lambda [3 x ...], Z."""
    E = [(c[..., i, 0] * px + c[..., i, 1] * py) + c[..., i, 2] for i in range(3)]
    S = (E[0] + E[1]) + E[2]
    cov = ((S > 0) & (E[0] >= 0) & (E[1] >= 0) & (E[2] >= 0)) | ((S < 0) & (E[0] <= 0) & (E[1] <= 0) & (E[2] <= 0))
    lam = [e / S for e in E]
    Z = (lam[0] * z[..., 0] + lam[1] * z[..., 1]) + lam[2] * z[..., 2]
    cov &= (Z >= nearp) & (Z <= farp)
    return cov, lam, Z


def shade(V, lam, col, ambient):
    """V [P,3,3] camera-space vertices of each pixel's face, lam 3 x [P], col [P,3,3] vertex colours -> fp64 [P,3]."""
    m = _cross(V[:, 1] - V[:, 0], V[:, 2] - V[:, 0])
    m = np.where((_dot(m, V[:, 0]) > 0)[:, None], -m, m)
    n = m / np.sqrt(_dot(m, m))[:, None]
    u = -(V / np.sqrt(_dot(V, V))[..., None])
    L = (lam[0][:, None] * u[:, 0] + lam[1][:, None] * u[:, 1]) + lam[2][:, None] * u[:, 2]
    L = L / np.sqrt(_dot(L, L))[:, None]
    dt = _dot(L, n)
    lw = ambient + np.where(dt > 0, dt, 0.0)
    lw = np.where(lw > 1, 1.0, lw)
    return lw[:, None] * ((lam[0][:, None] * col[:, 0] + lam[1][:, None] * col[:, 1]) + lam[2][:, None] * col[:, 2])


def render(verts, faces, K, poses, h, w, near, far, colors=None, ambient=0.5, bg=(0.0, 0.0, 0.0), chunk=16):
    """verts [nv,3], faces [nf,3], K [3,3] or [b,3,3], poses [b,3,4] -> depth f32 [b,h,w], rgb u8 [b,h,w,3],
    winning face int64 [b,h,w] (-1 where nothing covers the pixel)."""
    poses = np.asarray(poses, np.float32).reshape(-1, 3, 4)
    b = poses.shape[0]
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    nearp, farp = float(np.float32(near)), float(np.float32(far))
    assert 0 < nearp < farp
    amb = float(np.float32(ambient))
    nv = int(np.asarray(verts).shape[0])
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nf = faces.shape[0]
    col = np.full((nv, 3), 0.5) if colors is None else np.asarray(colors, np.float32).astype(np.float64)
    px = (np.arange(w) + 0.5)[None, None, :]
    py = (np.arange(h) + 0.5)[None, :, None]
    depth = np.zeros((b, h, w), np.float32)
    rgb = np.broadcast_to(to_u8(np.asarray(bg, np.float32)[:3]), (b, h, w, 3)).copy()
    win = np.full((b, h, w), -1, np.int64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for img in range(b):
            V, hh = camera_vertices(verts, poses[img], Ks[img])
            c, ok, fi = face_setup(faces, nv, hh)
            z = V[fi, 2] if nv else np.zeros((nf, 3))
            best = np.full((h, w), np.inf, np.float32)
            bidx = np.full((h, w), -1, np.int64)
            for f0 in range(0, nf, chunk):
                sl = slice(f0, min(nf, f0 + chunk))
                cov, _, Z = fragments(c[sl, None, None], z[sl, None, None], px, py, nearp, farp)
                cov &= ok[sl, None, None]
                Zm = np.where(cov, Z.astype(np.float32), np.float32(np.inf))
                a = np.argmin(Zm, axis=0)                                  # first minimum: the lower face index
                zmin = np.take_along_axis(Zm, a[None], 0)[0]
                upd = zmin < best                                          # an earlier chunk keeps a tie
                best = np.where(upd, zmin, best)
                bidx = np.where(upd, a + f0, bidx)
            hit = bidx >= 0
            win[img] = bidx
            depth[img][hit] = best[hit]
            if hit.any():
                r, cc = np.nonzero(hit)
                f = bidx[hit]
                cov, lam, _ = fragments(c[f], z[f], cc + 0.5, r + 0.5, nearp, farp)
                assert cov.all()
                rgb[img][hit] = to_u8(shade(V[fi[f]], lam, col[fi[f]], amb))
    return depth, rgb, win
