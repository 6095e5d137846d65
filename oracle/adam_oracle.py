"""CPU oracle for the Adam step -- TEST INFRASTRUCTURE ONLY.

numpy float32 restatement of the sequence DESIGN.md §19 states for `pvnet_adam_step`: torch.optim.Adam(foreach=False)
(`_single_tensor_adam`, torch/optim/adam.py, with amsgrad, maximize, capturable and differentiable off) as ATen's CUDA
element-wise kernels compute it.  Scalars are Python floats (doubles), prepared as torch's Python prepares them and
converted to fp32 once, where ATen converts them; tensors are fp32, every operation rounded to nearest:

    g'    = fma(p, f32(wd), g)                           grad.add(param, alpha=wd); only when wd != 0
    d     = g' - m                                       exp_avg.lerp_(grad, 1 - beta1), w1 = f32(1 - beta1):
    m'    = fma(w1, d, m)                 if |w1| < 0.5    self + w*(end - self)
            fma(-d, 1f - w1, g')          otherwise        end - (end - self)*(1 - w)
    v'    = fma(f32(1 - beta2), g'*g', v*f32(beta2))     exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    denom = sqrt(v') * f32(1.0 / bc2_sqrt) + f32(eps)    (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
    p'    = fma(f32(-step_size), m' / denom, p)          param.addcdiv_(exp_avg, denom, value=-step_size)

with bias_correction1 = 1 - beta1**step, bias_correction2 = 1 - beta2**step, step_size = lr / bias_correction1 and
bc2_sqrt = bias_correction2**0.5 in double.  One function per line, written from that statement and not from the kernel.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
F64 = np.float64


def fma(a, b, c):
    """fl32(a*b + c) with one rounding, for fp32 a, b, c (arrays or scalars).

    The product of two fp32 values is exact in fp64 (48 significant bits, exponent well inside fp64's range).  Adding
    the addend in fp64 and then rounding to fp32 would round twice, and that is NOT always the FMA's result: the fp64
    sum can land exactly on an fp32 tie that the discarded low bits would have broken (a = b*c + 1 with b*c =
    2^-24 + 2^-60).  So the fp64 sum is rounded to odd instead of to nearest -- TwoSum recovers the sum's exact error,
    and where the sum is inexact and its last mantissa bit is even, the neighbour on the error's side is taken.  A
    53-bit round-to-odd value rounds to 24 bits (or fewer, for subnormal results) as the exact value does (Boldo and
    Melquiond, "Emulation of FMA and correctly rounded sums: proved algorithms using rounding to odd", 2008)."""
    with np.errstate(all="ignore"):
        P = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)
        P, C = np.broadcast_arrays(P, np.asarray(c, F32).astype(F64))
        s = P + C
        t = s - P
        err = (P - (s - t)) + (C - t)                     # TwoSum: P + C == s + err exactly
        fix = np.isfinite(s) & (err != 0) & ((s.view(np.int64) & 1) == 0)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def scalars(lr, beta1, beta2, eps, weight_decay, step):
    """The step's scalars: doubles as torch's Python computes them, then the fp32 values the kernels take."""
    step = float(step)                                   # torch's step is a float32 tensor read back as a float
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    step_size = lr / bias_correction1
    bias_correction2_sqrt = bias_correction2 ** 0.5
    w1 = F32(1 - beta1)
    return {
        "wd": F32(weight_decay), "has_wd": weight_decay != 0,
        "w1": w1, "one_m_w1": F32(1) - w1, "lerp_small": bool(abs(w1) < F32(0.5)),
        "b2": F32(beta2), "w2": F32(1 - beta2),
        # Tensor / Python scalar multiplies by the scalar's reciprocal, taken in double and rounded to fp32 once
        "inv_bc2": F32(1.0 / bias_correction2_sqrt),
        "eps": F32(eps), "neg_step": F32(-step_size),
    }


def decayed_grad(p, g, s):
    return fma(p, s["wd"], g) if s["has_wd"] else g


def exp_avg(m, g, s):
    with np.errstate(all="ignore"):
        d = g - m
    return fma(s["w1"], d, m) if s["lerp_small"] else fma(-d, s["one_m_w1"], g)


def exp_avg_sq(v, g, s):
    with np.errstate(all="ignore"):
        return fma(s["w2"], g * g, v * s["b2"])


def denominator(v, s):
    with np.errstate(all="ignore"):
        return np.sqrt(v) * s["inv_bc2"] + s["eps"]


def param(p, m, denom, s):
    with np.errstate(all="ignore"):
        return fma(s["neg_step"], m / denom, p)


def adam_step(p, g, m, v, *, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, step=1):
    """One step for fp32 arrays p, g, m, v (not modified); `step` is the count this step reaches (1 on the first).
    Returns the new (p, m, v)."""
    p, g, m, v = (np.asarray(x, F32) for x in (p, g, m, v))
    s = scalars(lr, betas[0], betas[1], eps, weight_decay, step)
    g = decayed_grad(p, g, s)
    m = exp_avg(m, g, s)
    v = exp_avg_sq(v, g, s)
    return param(p, m, denominator(v, s), s), m, v
