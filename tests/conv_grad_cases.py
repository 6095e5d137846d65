"""The 24 native convolutions of Resnet18_8s.forward_train (slots 1..24) and fp64 restatements of their gradients.

Each row: (name, Cin, Cout, ksize, stride, dilation, (H, W) of the output at a 480x640 input).  convraw.0's weight has
35 input channels and reads a 40-channel buffer (fm, image, 5 zeros); only fm's 32 channels get a data gradient."""
from __future__ import annotations

import torch
import torch.nn.functional as F

ROWS = [
    ("layer1.0.conv1", 64, 64, 3, 1, 1, (120, 160)), ("layer1.0.conv2", 64, 64, 3, 1, 1, (120, 160)),
    ("layer1.1.conv1", 64, 64, 3, 1, 1, (120, 160)), ("layer1.1.conv2", 64, 64, 3, 1, 1, (120, 160)),
    ("layer2.0.conv1", 64, 128, 3, 2, 1, (60, 80)), ("layer2.0.downsample.0", 64, 128, 1, 2, 1, (60, 80)),
    ("layer2.0.conv2", 128, 128, 3, 1, 1, (60, 80)),
    ("layer2.1.conv1", 128, 128, 3, 1, 1, (60, 80)), ("layer2.1.conv2", 128, 128, 3, 1, 1, (60, 80)),
    ("layer3.0.conv1", 128, 256, 3, 1, 2, (60, 80)), ("layer3.0.downsample.0", 128, 256, 1, 1, 2, (60, 80)),
    ("layer3.0.conv2", 256, 256, 3, 1, 2, (60, 80)),
    ("layer3.1.conv1", 256, 256, 3, 1, 2, (60, 80)), ("layer3.1.conv2", 256, 256, 3, 1, 2, (60, 80)),
    ("layer4.0.conv1", 256, 512, 3, 1, 4, (60, 80)), ("layer4.0.downsample.0", 256, 512, 1, 1, 4, (60, 80)),
    ("layer4.0.conv2", 512, 512, 3, 1, 4, (60, 80)),
    ("layer4.1.conv1", 512, 512, 3, 1, 4, (60, 80)), ("layer4.1.conv2", 512, 512, 3, 1, 4, (60, 80)),
    ("fc.0", 512, 256, 3, 1, 1, (60, 80)), ("conv8s.0", 384, 128, 3, 1, 1, (60, 80)),
    ("conv4s.0", 192, 64, 3, 1, 1, (120, 160)), ("conv2s.0", 128, 32, 3, 1, 1, (240, 320)),
    ("convraw.0", 35, 32, 3, 1, 1, (480, 640)),
]
CONVRAW_BUFFER, CONVRAW_DGRAD = 40, 32


def pad_of(ksize, dilation):
    return dilation * (ksize - 1) // 2


def buffer_channels(name, cin):
    return CONVRAW_BUFFER if name == "convraw.0" else cin


def dgrad_channels(name, cin):
    return CONVRAW_DGRAD if name == "convraw.0" else cin


def zero_insert(dy):
    """[b,C,h,w] -> [b,C,2h,2w] with dy at the even pixels and zeros elsewhere."""
    b, c, h, w = dy.shape
    up = dy.new_zeros(b, c, 2 * h, 2 * w)
    up[:, :, ::2, ::2] = dy
    return up


def unpack_dgrad(packed, n, cout, ksize):
    """pack_dgrad_weight's [n][k*k][cin_pad] back to a torch conv weight [n, Cout, k, k] (taps as stored)."""
    return packed[:n, :, :cout].reshape(n, ksize, ksize, cout).permute(0, 3, 1, 2)


def dgrad_stride1_form(dy, packed, n, cout, ksize, stride, dilation):
    """The data gradient as the kernels compute it: a stride-1 forward conv of (zero-inserted) dy with the pack."""
    src = zero_insert(dy) if stride == 2 else dy
    return F.conv2d(src, unpack_dgrad(packed, n, cout, ksize).to(dy.dtype), padding=pad_of(ksize, dilation),
                    dilation=dilation)


def wgrad_sum(x, dy, ksize, dilation):
    """dW[co][ci][kh][kw] = sum_{n,y,x} dy[n,co,y,x] * x[n,ci,y+(kh-c)d,x+(kw-c)d] (zero outside), stride 1."""
    p = pad_of(ksize, dilation)
    xp = F.pad(x, (p, p, p, p))
    H, W = dy.shape[2:]
    out = x.new_zeros(dy.shape[1], x.shape[1], ksize, ksize)
    for kh in range(ksize):
        for kw in range(ksize):
            xs = xp[:, :, kh * dilation:kh * dilation + H, kw * dilation:kw * dilation + W]
            out[:, :, kh, kw] = torch.einsum("nohw,nihw->oi", dy, xs)
    return out


def wgrad_stride1_form(x, dy, ksize, stride, dilation):
    """The weight gradient as the kernels compute it: the stride-1 sum over (zero-inserted) dy."""
    return wgrad_sum(x, zero_insert(dy) if stride == 2 else dy, ksize, dilation)


def tf32_trunc(t):
    """What a TF32 MMA reads from an fp32 value: the low 13 mantissa bits dropped."""
    return (t.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
