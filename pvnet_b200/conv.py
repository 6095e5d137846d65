"""Host helpers for the tensor-core convolution primitive (pvnet_conv2d_nhwc).

Weight packing (done once at load time, not on the hot path): PyTorch's
[Cout,Cin,kh,kw] conv weight with an eval-mode BatchNorm folded in
(w' = w * gamma/sqrt(var+eps), b' = beta - mean*gamma/sqrt(var+eps)) becomes the
K-major [Cout][kh*kw][Cin] matrix the kernel's weight tensor map reads, rounded to TF32.
"""
from __future__ import annotations

import ctypes

import torch

from . import _native

ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2
MODE_AUTO, MODE_PER_TAP, MODE_COLUMN = 0, 1, 2


def set_mode(mode: int):
    """Test hook (pvnet_conv_set_mode): which kernel runs layers both kernels support."""
    _native.check(_native.lib().pvnet_conv_set_mode(int(mode)), "pvnet_conv_set_mode")


def set_multicast(mode: int):
    """Test hook (pvnet_conv_set_multicast): 0 single CTAs (default), 1 two-CTA clusters with weight multicast."""
    _native.check(_native.lib().pvnet_conv_set_multicast(int(mode)), "pvnet_conv_set_multicast")


def set_persistent(on: bool):
    """Test hook (pvnet_conv_set_persistent): persistent variant of the per-tap kernel."""
    _native.check(_native.lib().pvnet_conv_set_persistent(int(bool(on))), "pvnet_conv_set_persistent")


def round_tf32(t: torch.Tensor) -> torch.Tensor:
    """Round fp32 to the nearest TF32 value (10 explicit mantissa bits), kept in fp32."""
    i = t.contiguous().view(torch.int32)
    i = (i + 0x1000) & ~0x1FFF          # round half away from zero on the magnitude bits
    return i.view(torch.float32)


def fold_bn(weight, bn_weight=None, bn_bias=None, bn_mean=None, bn_var=None, eps=1e-5, conv_bias=None):
    w = weight.detach().to(torch.float64)
    cout = w.shape[0]
    b = torch.zeros(cout, dtype=torch.float64, device=w.device) if conv_bias is None else conv_bias.detach().double()
    if bn_weight is not None:
        scale = bn_weight.detach().double() / torch.sqrt(bn_var.detach().double() + eps)
        w = w * scale[:, None, None, None]
        b = (b - bn_mean.detach().double()) * scale + bn_bias.detach().double()
    return w.float(), b.float()


def cin_padded(cin: int) -> int:
    """Channels per tap in the packed weights: 16 stays 16, everything else rounds up to 32."""
    return 16 if cin == 16 else (cin + 31) // 32 * 32


def pack_weight(w: torch.Tensor, cin_pad: int | None = None, cout_pad: int | None = None, tf32: bool = True):
    """[Cout,Cin,kh,kw] -> [Cout_pad][kh*kw][cin_pad] contiguous (zero padded; cin_pad defaults to
    cin_padded(Cin), what the kernels expect)."""
    cout, cin, kh, kw = w.shape
    cin_pad = cin_padded(cin) if cin_pad is None else cin_pad
    cout_pad = cout if cout_pad is None else cout_pad
    p = torch.zeros(cout_pad, kh * kw, cin_pad, dtype=torch.float32, device=w.device)
    p[:cout, :, :cin] = w.permute(0, 2, 3, 1).reshape(cout, kh * kw, cin)
    return round_tf32(p) if tf32 else p.contiguous()


def pack_stem_s2d(w: torch.Tensor) -> torch.Tensor:
    """conv1 [64,3,7,7] (stride 2, pad 3) -> [64][4][4][16], the equivalent 4x4 stride-1 conv on
    the 2x2 space-to-depth image: out(o) = sum_k w[k] in(2o+k-3); with in(2j+p) = S[j][p] the tap
    t = j-o+2 in {0..3} and parity p carry k = 2t+p-1 (zero weight when k is outside 0..6)."""
    cout = w.shape[0]
    out = torch.zeros(cout, 4, 4, 16, dtype=torch.float32, device=w.device)
    for ty in range(4):
        for py in range(2):
            kh = 2 * ty + py - 1
            if not 0 <= kh <= 6:
                continue
            for tx in range(4):
                for px in range(2):
                    kw = 2 * tx + px - 1
                    if not 0 <= kw <= 6:
                        continue
                    ch = (py * 2 + px) * 3
                    out[:, ty, tx, ch:ch + 3] = w[:, :, kh, kw]
    return round_tf32(out)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def conv2d_nhwc(inp, in_co, cin, w_packed, bias, out, out_co, cout, ksize, stride=1, dilation=1, act=ACT_NONE,
                res=None, res_co=0, round_out=False):
    """inp [b,H,W,in_cs] / out [b,Ho,Wo,out_cs] / res [b,Ho,Wo,res_cs]: contiguous NHWC fp32
    CUDA tensors; the conv reads channels [in_co,in_co+cin) and writes [out_co,out_co+cout)."""
    b, H, W, in_cs = inp.shape
    with torch.cuda.device(inp.device):
        _native.check(_native.lib().pvnet_conv2d_nhwc(
            _p(inp), in_cs, in_co, cin, _p(w_packed), _p(bias), _p(res), 0 if res is None else res.shape[3], res_co,
            _p(out), out.shape[3], out_co, cout, b, H, W, ksize, stride, dilation, act, int(round_out),
            ctypes.c_void_p(torch.cuda.current_stream(inp.device).cuda_stream)), "pvnet_conv2d_nhwc")
    return out
