"""numpy restatement of the stem fold, the training max-pool and the head convraw.3 of Resnet18_8s's training step
(csrc/train_layers.cu, csrc/backbone_aux.cu).

* Stem: the 7x7 stride-2 pad-3 weight gradient is the 4x4 stride-1 one on the 2x2 space-to-depth image S (taps at
  offsets -2..1), folded back: dW[co][c][kh][kw] = dW_s2d[co][ty][tx][(py*2+px)*3+c], kh = 2ty+py-1, kw = 2tx+px-1.
* Max-pool 3x3/2 pad 1: torch's argmax rule (row-major scan from -inf, `v > max or isnan(v)` wins, no winner -> the
  first in-image element) with a window code dy*3+dx; the backward adds, per input pixel, the dY of the windows
  whose code points at it, outputs ascending over ATen's window bounds, from 0.0f, in fp32.
* Head: out = fmaf chain over c ascending from bias[o]; dy = fmaf chain over o ascending from 0; dW, db = fp64 sums
  over HEAD_CHUNK-pixel partials (pixels ascending, from 0.0), merged in bn_train_oracle.merge's lane-then-tree order,
  rounded once to fp32.
"""
from __future__ import annotations

import numpy as np

from oracle.bn_train_oracle import F32, fma32, merge

HEAD_CHUNK = 4096


# ----------------------------------------------------------------------------- stem
def stem_fold_map():
    """[(ty, tx, ch, c, kh, kw)] for the 147 entries of the [4][4][16] space-to-depth weight that carry a weight."""
    out = []
    for ty in range(4):
        for tx in range(4):
            for ch in range(12):
                par, c = divmod(ch, 3)
                py, px = divmod(par, 2)
                kh, kw = 2 * ty + py - 1, 2 * tx + px - 1
                if 0 <= kh <= 6 and 0 <= kw <= 6:
                    out.append((ty, tx, ch, c, kh, kw))
    return out


def space_to_depth(x):
    """[b,3,H,W] -> S [b,H/2,W/2,16]: channel (py*2+px)*3+c holds x[c][2i+py][2j+px]; channels 12..15 are zero."""
    b, _, H, W = x.shape
    s = np.zeros((b, H // 2, W // 2, 16), dtype=x.dtype)
    for py in range(2):
        for px in range(2):
            for c in range(3):
                s[..., (py * 2 + px) * 3 + c] = x[:, c, py::2, px::2]
    return s


def stem_wgrad_s2d(s, dy):
    """dW_s2d [co][ty][tx][ch] = sum_p dY[p][co] * S[p + (ty-2, tx-2)][ch] (zero outside), fp64.  s [b,h,w,16],
    dy [b,h,w,Co]."""
    b, h, w, _ = s.shape
    sp = np.zeros((b, h + 3, w + 3, 16))
    sp[:, 2:2 + h, 2:2 + w] = s
    out = np.zeros((dy.shape[3], 4, 4, 16))
    for ty in range(4):
        for tx in range(4):
            win = sp[:, ty:ty + h, tx:tx + w].reshape(-1, 16)
            out[:, ty, tx] = dy.reshape(-1, dy.shape[3]).astype(np.float64).T @ win
    return out


def stem_fold(dw_s2d):
    """[Co][4][4][16] -> [Co][3][7][7]."""
    out = np.zeros((dw_s2d.shape[0], 3, 7, 7), dtype=dw_s2d.dtype)
    for ty, tx, ch, c, kh, kw in stem_fold_map():
        out[:, c, kh, kw] = dw_s2d[:, ty, tx, ch]
    return out


# ----------------------------------------------------------------------------- max-pool 3x3 / 2, pad 1
def maxpool_forward(x):
    """x NHWC [b,H,W,C] float32 -> (out [b,H/2,W/2,C] float32, code uint8 [b,H/2,W/2,C])."""
    x = np.asarray(x, F32)
    b, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    m = np.full((b, Ho, Wo, C), -np.inf, dtype=F32)
    k = np.full((b, Ho, Wo, C), -1, dtype=np.int64)
    first = np.full((Ho, Wo), -1, dtype=np.int64)
    oy, ox = np.mgrid[0:Ho, 0:Wo]
    for dy in range(3):
        for dx in range(3):
            iy, ix = 2 * oy - 1 + dy, 2 * ox - 1 + dx
            ok = (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
            v = np.full((b, Ho, Wo, C), -np.inf, dtype=F32)
            v[:, ok] = x[:, iy[ok], ix[ok]]
            first = np.where(ok & (first < 0), dy * 3 + dx, first)
            with np.errstate(invalid="ignore"):
                win = ok[None, :, :, None] & ((v > m) | np.isnan(v))
            m = np.where(win, v, m)
            k = np.where(win, dy * 3 + dx, k)
    k = np.where(k < 0, first[None, :, :, None], k)
    return m, k.astype(np.uint8)


def maxpool_backward(dout, code, H, W):
    """dout, code [b,H/2,W/2,C] -> din [b,H,W,C] float32 in ATen's gather order."""
    dout = np.asarray(dout, F32)
    b, Ho, Wo, C = dout.shape
    din = np.zeros((b, H, W, C), dtype=F32)
    for iy in range(H):
        oy0, oy1 = (0 if iy + 1 < 3 else (iy + 1 - 3) // 2 + 1), min((iy + 1) // 2 + 1, Ho)
        for ix in range(W):
            ox0, ox1 = (0 if ix + 1 < 3 else (ix + 1 - 3) // 2 + 1), min((ix + 1) // 2 + 1, Wo)
            acc = np.zeros((b, C), dtype=F32)
            for oy in range(oy0, oy1):
                for ox in range(ox0, ox1):
                    want = (iy - (2 * oy - 1)) * 3 + (ix - (2 * ox - 1))
                    hit = code[:, oy, ox] == want
                    acc = np.where(hit, (acc + dout[:, oy, ox]).astype(F32), acc)
            din[:, iy, ix] = acc
    return din


# ----------------------------------------------------------------------------- head (1x1 + bias)
def head_forward(y, w, bias):
    """y [N, Cin], w [Cout, Cin], bias [Cout] float32 -> out [N, Cout]: acc = bias[o], then fma(w[o][c], y[c], acc)."""
    y, w = np.asarray(y, F32), np.asarray(w, F32)
    acc = np.broadcast_to(np.asarray(bias, F32), (y.shape[0], w.shape[0])).copy()
    for c in range(y.shape[1]):
        acc = fma32(w[None, :, c], y[:, c:c + 1], acc)
    return acc


def head_dy(g, w):
    """g [N, Cout], w [Cout, Cin] -> dy [N, Cin]: acc = 0, then fma(w[o][c], g[o], acc) for o ascending."""
    g, w = np.asarray(g, F32), np.asarray(w, F32)
    acc = np.zeros((g.shape[0], w.shape[1]), dtype=F32)
    for o in range(w.shape[0]):
        acc = fma32(w[None, o, :], g[:, o:o + 1], acc)
    return acc


def head_param_sums(g, y):
    """(dW [Cout, Cin], db [Cout]) float32 from g [N, Cout] and y [N, Cin], in the kernels' fixed fp64 order."""
    g64, y64 = np.asarray(g, F32).astype(np.float64), np.asarray(y, F32).astype(np.float64)
    N, Cout = g64.shape
    Cin = y64.shape[1]
    ye = np.concatenate([y64, np.ones((N, 1))], 1)          # the last column gives db
    P = -(-N // HEAD_CHUNK)
    acc = np.zeros((P, Cout, Cin + 1))
    base = np.arange(P, dtype=np.int64) * HEAD_CHUNK
    for i in range(HEAD_CHUNK):
        rows = base + i
        ok = rows < N
        if not ok.any():
            break
        acc[ok] = acc[ok] + g64[rows[ok], :, None] * ye[rows[ok], None, :]
    tot = merge(acc.reshape(P, -1)).reshape(Cout, Cin + 1)
    return tot[:, :Cin].astype(F32), tot[:, Cin].astype(F32)
