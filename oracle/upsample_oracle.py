"""CPU oracle for the bilinear x2 upsampling backward -- TEST INFRASTRUCTURE ONLY.

numpy float32 restatement of what `pvnet_upsample2x_backward_nhwc` (pvnet_b200/csrc/backbone_aux.cu,
k_upsample2x_backward; DESIGN.md §15) computes: dX = U^T dY of F.interpolate(scale_factor=2, mode='bilinear',
align_corners=True) (nn.UpsamplingBilinear2d, lib/networks/model_repository.py:35,43,51), as a gather in which each
input pixel sums exactly the terms ATen's CUDA backward (upsample_bilinear2d_backward_nhwc_out_frame) adds with
atomics, in a fixed order:

    scale = f32(in - 1) / f32(out - 1)            (0 when out == 1; out = 2 * in)
    src = scale * f32(o), i0 = int(src), i0p = 1 if i0 < in - 1 else 0
    l1 = src - f32(i0), l0 = 1 - l1               output o feeds input i0 with l0 and i0 + i0p with l1
    term = f32(f32(hl * wl) * g)                  the four terms in ATen's order (l0 l0, l0 l1, l1 l0, l1 l1)

Order: ascending output pixel (row-major), then ATen's term order within one output pixel.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def scale(in_size):
    """launch_upsample2x's (and ATen's area_pixel_compute_scale's) align_corners scale for out = 2 * in."""
    out = 2 * in_size
    return F32(in_size - 1) / F32(out - 1) if out > 1 else F32(0)


def source_index(in_size, o):
    """ATen's index expressions for output index (array) o: (i0, i0 + i0p, l0, l1), fp32 weights."""
    o = np.asarray(o)
    src = (scale(in_size) * o.astype(F32)).astype(F32)
    i0 = src.astype(np.int64)                                    # (int) truncates; src >= 0
    i1 = i0 + (i0 < in_size - 1)
    l1 = (src - i0.astype(F32)).astype(F32)
    l0 = (F32(1) - l1).astype(F32)
    return i0, i1, l0, l1


def window_brute(in_size):
    """{input index: [(output index, slot, weight), ...]} over all 2 * in_size outputs, ascending (o, slot): the
    terms ATen's backward adds along one axis (slot 0 carries l0, slot 1 carries l1)."""
    o = np.arange(2 * in_size)
    i0, i1, l0, l1 = source_index(in_size, o)
    win = {i: [] for i in range(in_size)}
    for k in range(2 * in_size):
        win[int(i0[k])].append((k, 0, l0[k]))
        win[int(i1[k])].append((k, 1, l1[k]))
    return win


WINDOW = 6          # candidate outputs per input index: 2i-2 ... 2i+3


def window_table(in_size):
    """The kernel's rule for every input index i at once: the candidates o = 2i-2+r (r < WINDOW) inside
    [0, 2 * in_size) whose ATen expressions land on i.  Returns o, hit0, hit1, l0, l1, each [in_size, WINDOW]:
    hit0 -- o feeds i through slot 0 (weight l0), hit1 -- through slot 1 (weight l1)."""
    o = 2 * np.arange(in_size)[:, None] - 2 + np.arange(WINDOW)[None, :]
    valid = (o >= 0) & (o < 2 * in_size)
    i0, i1, l0, l1 = source_index(in_size, np.clip(o, 0, 2 * in_size - 1))
    i = np.arange(in_size)[:, None]
    return o, valid & (i0 == i), valid & (i1 == i), l0, l1


def window_rule(in_size, i, table=None):
    """[(o, slot, weight), ...] feeding input index i by the kernel's rule, ascending (o, slot)."""
    o, hit0, hit1, l0, l1 = window_table(in_size) if table is None else table
    out = []
    for r in range(WINDOW):
        if hit0[i, r]:
            out.append((int(o[i, r]), 0, l0[i, r]))
        if hit1[i, r]:
            out.append((int(o[i, r]), 1, l1[i, r]))
    return out


def _grouped(win):
    """[(o, [weights in slot order]), ...]"""
    groups = []
    for o, _slot, wt in win:
        if groups and groups[-1][0] == o:
            groups[-1][1].append(wt)
        else:
            groups.append((o, [wt]))
    return groups


def upsample2x_backward(dy):
    """dy [b, 2h, 2w, C] float32 -> dX [b, h, w, C] float32, k_upsample2x_backward's gather in its order: output rows
    ascending, then output columns ascending, then ATen's term order within the output pixel; every product and
    every sum rounded to fp32 (the accumulator starts at 0, as ATen's zero-filled gradient does)."""
    dy = np.asarray(dy, F32)
    b, H, W, C = dy.shape
    h, w = H // 2, W // 2
    th, tw = window_table(h), window_table(w)
    rows = [_grouped(window_rule(h, i, th)) for i in range(h)]
    cols = [_grouped(window_rule(w, j, tw)) for j in range(w)]
    dx = np.zeros((b, h, w, C), F32)
    for i in range(h):
        for j in range(w):
            acc = np.zeros((b, C), F32)
            for oy, hws in rows[i]:
                for ox, wws in cols[j]:
                    g = dy[:, oy, ox]
                    for hl in hws:
                        for wl in wws:
                            acc = (acc + (F32(hl * wl) * g).astype(F32)).astype(F32)
            dx[:, i, j] = acc
    return dx


def upsample2x_backward_scatter(dy):
    """The same sum as a plain scatter over ATen's terms: output pixels row-major, the four terms in ATen's order, each
    added to its input pixel in fp32 -- what ATen's backward computes when its atomics land in this order."""
    dy = np.asarray(dy, F32)
    b, H, W, C = dy.shape
    h, w = H // 2, W // 2
    yi0, yi1, yl0, yl1 = source_index(h, np.arange(H))
    xi0, xi1, xl0, xl1 = source_index(w, np.arange(W))
    dx = np.zeros((b, h, w, C), F32)
    for oy in range(H):
        for ox in range(W):
            g = dy[:, oy, ox]
            for iy, hl in ((yi0[oy], yl0[oy]), (yi1[oy], yl1[oy])):
                for ix, wl in ((xi0[ox], xl0[ox]), (xi1[ox], xl1[ox])):
                    dx[:, iy, ix] = (dx[:, iy, ix] + (F32(hl * wl) * g).astype(F32)).astype(F32)
    return dx


def interp_matrix(in_size):
    """[2 * in_size, in_size] float64 matrix of the fp32 weights: U = Uh (x) Uw is the forward."""
    o = np.arange(2 * in_size)
    i0, i1, l0, l1 = source_index(in_size, o)
    m = np.zeros((2 * in_size, in_size))
    np.add.at(m, (o, i0), l0.astype(np.float64))
    np.add.at(m, (o, i1), l1.astype(np.float64))
    return m
