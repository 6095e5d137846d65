"""numpy restatement of csrc/batchnorm.cu (train-mode BatchNorm2d fused with its activation and residual add), and
the exact fp64 references it is held to.

Tensors are NHWC flattened to [N, C] (N = b*H*W pixels).  The kernels' summation order:
  * partial j sums the pixels [j*CHUNK, (j+1)*CHUNK) in ascending order, from 0.0, in fp64;
  * per channel, lane t (of LANES) sums partials t, t+LANES, ... ascending, from 0.0; then lane[i] += lane[i+s] for
    s = LANES/2, ..., 1, and lane 0 is the total.
Every fp64 operation is a separately rounded IEEE operation (the kernels use _rn intrinsics), so numpy's float64
arithmetic gives the kernels' bits.  fp32 steps are float32 arithmetic, and fma32 is a correctly rounded fp32 fma.
"""
from __future__ import annotations

import numpy as np

CHUNK = 256
LANES = 256
ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2
F32 = np.float32


# ----------------------------------------------------------------------------- fixed-order sums
def chunk_sums(term, N: int, C: int) -> np.ndarray:
    """[P, C] fp64 partials, P = ceil(N / CHUNK): term(rows) gives the fp64 terms of pixel rows `rows` ([k] int64
    indices) as [k, C]; partial j adds pixel j*CHUNK + i for i = 0, 1, ... in order."""
    P = -(-N // CHUNK)
    acc = np.zeros((P, C))
    base = np.arange(P, dtype=np.int64) * CHUNK
    for i in range(CHUNK):
        rows = base + i
        ok = rows < N
        if not ok.any():
            break
        acc[ok] = acc[ok] + term(rows[ok])
    return acc


def merge(partials: np.ndarray) -> np.ndarray:
    """[P, C] partials -> [C] in the kernels' lane-then-tree order."""
    P, C = partials.shape
    lane = np.zeros((LANES, C))
    for k in range(0, P, LANES):
        blk = partials[k:k + LANES]
        lane[:blk.shape[0]] = lane[:blk.shape[0]] + blk
    s = LANES // 2
    while s:
        lane[:s] = lane[:s] + lane[s:2 * s]
        s //= 2
    return lane[0].copy()


# ----------------------------------------------------------------------------- forward
def batch_stats(x: np.ndarray, eps: float):
    """x [N, C] float32 -> (mean, biased var, invstd) fp64 [C], as k_bn_stats_partial + k_bn_finalize compute them:
    shifted sums of d = x - x[0] and d*d, mean = x[0] + S1/N, var = max(S2/N - (S1/N)^2, 0)."""
    N, C = x.shape
    K = x[0].astype(np.float64)

    def d(rows):
        return x[rows].astype(np.float64) - K
    S1 = merge(chunk_sums(d, N, C))
    S2 = merge(chunk_sums(lambda rows: d(rows) * d(rows), N, C))
    rN = 1.0 / N
    m = S1 * rN
    mean = K + m
    var = np.maximum(S2 * rN - m * m, 0.0)
    return mean, var, invstd_of(var, eps)


def invstd_of(var, eps):
    return 1.0 / np.sqrt(np.asarray(var, np.float64) + eps)


def scale_shift(mean, invstd, gamma=None, beta=None):
    """fp32 scale = gamma*invstd and shift = beta - mean*scale, each rounded once from fp64."""
    g = np.ones_like(mean) if gamma is None else np.asarray(gamma, np.float64)
    b = np.zeros_like(mean) if beta is None else np.asarray(beta, np.float64)
    scale = (g * invstd).astype(F32)
    shift = (b - mean * scale.astype(np.float64)).astype(F32)
    return scale, shift


def unbiased32(var, N: int):
    """The variance running_var is updated with: fp32(var * N * (1/(N-1)))."""
    return (np.asarray(var, np.float64) * float(N) * (1.0 / (N - 1.0))).astype(F32)


def running_update(r, stat32, factor: float):
    """nn.BatchNorm2d's rule in fp32: r * fp32(1 - f) + stat * fp32(f)."""
    return (np.asarray(r, F32) * F32(1.0 - factor) + np.asarray(stat32, F32) * F32(factor)).astype(F32)


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c): a*b is exact in fp64, the fp64 sum's error comes from TwoSum, and a tie of
    the fp64 sum between two fp32 values is broken by that error's sign."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        toward = np.where(s > r64, np.inf, -np.inf).astype(F32)
        nb = np.nextafter(r, toward)
        mid = (r64 + nb.astype(np.float64)) * 0.5
        tie = (s != r64) & (s == mid) & (err != 0)
        # at a tie the exact value lies on err's side of the midpoint
        pick_nb = tie & (np.sign(err) == np.sign(nb.astype(np.float64) - r64))
        alt = np.where(pick_nb, nb, r)
        # s exactly representable in fp32 with err != 0 cannot change the rounding (|err| < half an fp32 ulp)
    return np.where(tie, alt, r).astype(F32)


def act_fwd(v, act):
    v = np.asarray(v, F32)
    if act == ACT_RELU:
        return np.where(v <= 0, F32(0), v).astype(F32)
    if act == ACT_LEAKY:
        return np.where(v > 0, v, v * F32(0.1)).astype(F32)
    return v


def pre_activation(x, scale, shift, z=None, scale_z=None, shift_z=None):
    """The forward's pre-activation value: fma(x, scale, shift) in fp32, then + z (form 1) or + fma(z, ...) (form 2)."""
    v = fma32(x, scale, shift)
    if z is not None and scale_z is None:
        v = (v + np.asarray(z, F32)).astype(F32)
    elif z is not None:
        v = (v + fma32(z, scale_z, shift_z)).astype(F32)
    return v


def masked_grad(dy, pre, act):
    """g = dy * act'(pre): torch's threshold_backward (0 where the result <= 0) and leaky_relu_backward (dy * 0.1f
    where the result <= 0); the result has the sign of `pre`."""
    dy = np.asarray(dy, F32)
    pre = np.asarray(pre, F32)
    if act == ACT_RELU:
        return np.where(pre <= 0, F32(0), dy).astype(F32)
    if act == ACT_LEAKY:
        return np.where(pre > 0, dy, dy * F32(0.1)).astype(F32)
    return dy


# ----------------------------------------------------------------------------- backward
def backward_sums(g, x, mean):
    """(sum g, sum g*(x - mean)) fp64 [C] in the kernels' order; g, x [N, C] float32, mean fp64 [C]."""
    N, C = x.shape
    Sg = merge(chunk_sums(lambda r: g[r].astype(np.float64), N, C))
    Sgx = merge(chunk_sums(lambda r: g[r].astype(np.float64) * (x[r].astype(np.float64) - mean), N, C))
    return Sg, Sgx


def backward_coef(Sg, Sgx, N: int, mean, invstd, gamma=None, batch_stats=True):
    """fp32 (A, B, Cc) with dx = A*g + B*x + Cc, and fp32 (dgamma, dbeta), rounded once from fp64."""
    g = np.ones_like(invstd) if gamma is None else np.asarray(gamma, np.float64)
    A = g * invstd
    if batch_stats:
        rN = 1.0 / N
        B = -((A * (invstd * invstd)) * (Sgx * rN))
        Cc = -(A * (Sg * rN)) - B * mean
    else:
        B = np.zeros_like(A)
        Cc = np.zeros_like(A)
    return (A.astype(F32), B.astype(F32), Cc.astype(F32)), ((Sgx * invstd).astype(F32), Sg.astype(F32))


def backward_apply(g, x, coef):
    A, B, Cc = coef
    return fma32(A, g, fma32(B, x, Cc))


# ----------------------------------------------------------------------------- exact fp64 references
def exact_stats(x):
    """Two-pass fp64 mean and biased variance of x [N, C]."""
    x64 = np.asarray(x, np.float64)
    mean = x64.mean(0)
    return mean, ((x64 - mean) ** 2).mean(0)


def exact_backward(g, x, eps, gamma=None, batch_stats=True, mean=None, var=None):
    """The analytic BatchNorm backward in fp64 for the upstream gradient g (after the activation's mask): (dx, dgamma,
    dbeta).  With batch_stats=False, mean/var are the running statistics and dx = gamma*invstd*g."""
    g64, x64 = np.asarray(g, np.float64), np.asarray(x, np.float64)
    if batch_stats:
        mean, var = exact_stats(x)
    invstd = 1.0 / np.sqrt(np.asarray(var, np.float64) + eps)
    gm = np.ones_like(invstd) if gamma is None else np.asarray(gamma, np.float64)
    xhat = (x64 - mean) * invstd
    if batch_stats:
        dx = gm * invstd * (g64 - g64.mean(0) - xhat * (g64 * xhat).mean(0))
    else:
        dx = gm * invstd * g64
    return dx, (g64 * xhat).sum(0), g64.sum(0)
