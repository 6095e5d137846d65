"""CPU: the index / weight logic of k_upsample2x's interior fast path (backbone_aux.cu), restated in numpy float32
with the kernel's rounding sequence (fmul of the first product, fma of the second): its two-term sums round exactly
like the general three-term window and like the direct per-pixel ATen formula of
F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) (lib/networks/model_repository.py:75) evaluated
the same way -- bit for bit."""
import numpy as np
import pytest

f32 = np.float32


def _fma(a, b, c):
    return f32(np.float64(a) * np.float64(b) + np.float64(c))


def _lerp2(w0, a, w1, b):           # fma(w1, b, rn(w0 * a)): lerp3 with a zero third weight
    return _fma(w1, b, f32(w0 * a))


def _lerp3(w0, a, w1, b, w2, c):
    return _fma(w2, c, _fma(w1, b, f32(w0 * a)))


def _direct(L, y, x, sy, sx):
    h2, w2 = L.shape
    fy = f32(sy * f32(y)); ylo = int(fy); yhi = min(ylo + 1, h2 - 1); h1 = f32(fy - f32(ylo)); h0 = f32(f32(1) - h1)
    fx = f32(sx * f32(x)); xlo = int(fx); xhi = min(xlo + 1, w2 - 1); w1 = f32(fx - f32(xlo)); w0 = f32(f32(1) - w1)
    return _lerp2(h0, _lerp2(w0, L[ylo, xlo], w1, L[ylo, xhi]), h1, _lerp2(w0, L[yhi, xlo], w1, L[yhi, xhi]))


@pytest.mark.parametrize("h,w", [(8, 8), (30, 40), (36, 52)])
def test_upsample_kernel_interior_path_equals_window_path(h, w):
    """k_upsample2x: blocks whose pattern is (rows (j-1, j) for output 2j, (j, j+1) for 2j+1; same for columns) take two-term
    sums; they must round exactly like the general three-term lerp3 with its zero weight."""
    L = np.random.default_rng(h * 100 + w).standard_normal((h, w)).astype(f32)
    sy, sx = f32(h - 1) / f32(2 * h - 1), f32(w - 1) / f32(2 * w - 1)
    n_interior = 0
    for j in range(h):
        for k in range(w):
            wy = np.zeros((2, 3), f32); wx = np.zeros((2, 3), f32); pat = [[False, False], [False, False]]
            for o in range(2):
                fy = f32(sy * f32(2 * j + o)); fx = f32(sx * f32(2 * k + o)); y0 = int(fy); x0 = int(fx)
                h1 = f32(fy - f32(y0)); h0 = f32(f32(1) - h1); w1 = f32(fx - f32(x0)); w0 = f32(f32(1) - w1)
                uy, ux = y0 >= j, x0 >= k
                pat[o] = [uy, ux]
                wy[o] = [0, h0, h1] if uy else [h0, h1, 0]
                wx[o] = [0, w0, w1] if ux else [w0, w1, 0]
            rows = [min(max(j - 1 + r, 0), h - 1) for r in range(3)]
            cols = [min(max(k - 1 + c, 0), w - 1) for c in range(3)]
            t = [[_lerp3(wx[o][0], L[rows[r], cols[0]], wx[o][1], L[rows[r], cols[1]], wx[o][2], L[rows[r], cols[2]])
                  for o in range(2)] for r in range(3)]
            gen = [[_lerp3(wy[oy][0], t[0][ox], wy[oy][1], t[1][ox], wy[oy][2], t[2][ox]) for ox in range(2)] for oy in range(2)]
            for oy in range(2):
                for ox in range(2):
                    assert gen[oy][ox] == _direct(L, 2 * j + oy, 2 * k + ox, sy, sx)
            if (not pat[0][0]) and pat[1][0] and (not pat[0][1]) and pat[1][1]:
                n_interior += 1
                tf = [[_lerp2(wx[0][0], L[rows[r], cols[0]], wx[0][1], L[rows[r], cols[1]]),
                       _lerp2(wx[1][1], L[rows[r], cols[1]], wx[1][2], L[rows[r], cols[2]])] for r in range(3)]
                fast = [[_lerp2(wy[0][0], tf[0][ox], wy[0][1], tf[1][ox]) for ox in range(2)],
                        [_lerp2(wy[1][1], tf[1][ox], wy[1][2], tf[2][ox]) for ox in range(2)]]
                assert fast == gen
    assert n_interior >= (h - 2) * (w - 2)
