"""The 24 native convolutions of Resnet18_8s.forward_train (slots 1..24), then every other distinct convolution shape
(ksize, Cin, Cout, stride, dilation) of Resnet34_8s ("r34.") and Resnet50_8s ("r50.") under the name of its first
module, and fp64 restatements of their gradients.

Each row: (name, Cin, Cout, ksize, stride, dilation, (H, W) of the output at a 480x640 input).  convraw.0's weight has
s2dim + 3 input channels and reads a buffer of s2dim + 8 (fm, image, 5 zeros): 40 for Resnet18_8s, 72 for the deep
networks; only fm's s2dim channels get a data gradient.  A 1x1 downsample's dilation is its block's (it has one tap,
so the value does not change the convolution)."""
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
    # Resnet34_8s: fc.0 over layer4's 512 channels, the decoder over 320 channels and convraw.0 over 72; its conv8s.0
    # (512 -> 256) and conv2s.0 (192 -> 64) have the shapes of Resnet18_8s's fc.0 and conv4s.0
    ("r34.fc.0", 512, 384, 3, 1, 1, (60, 80)), ("r34.conv4s.0", 320, 128, 3, 1, 1, (120, 160)),
    ("r34.convraw.0", 67, 64, 3, 1, 1, (480, 640)),
    # Resnet50_8s: the Bottlenecks' 1x1 convs, conv2 (s2) of layer2.0, fc.0 at K = 18 432, the wider decoder inputs
    ("r50.layer1.0.conv1", 64, 64, 1, 1, 1, (120, 160)), ("r50.layer1.0.conv3", 64, 256, 1, 1, 1, (120, 160)),
    ("r50.layer1.1.conv1", 256, 64, 1, 1, 1, (120, 160)), ("r50.layer2.0.conv1", 256, 128, 1, 1, 1, (120, 160)),
    ("r50.layer2.0.conv2", 128, 128, 3, 2, 1, (60, 80)), ("r50.layer2.0.conv3", 128, 512, 1, 1, 1, (60, 80)),
    ("r50.layer2.0.downsample.0", 256, 512, 1, 2, 1, (60, 80)), ("r50.layer2.1.conv1", 512, 128, 1, 1, 1, (60, 80)),
    ("r50.layer3.0.conv1", 512, 256, 1, 1, 1, (60, 80)), ("r50.layer3.0.conv3", 256, 1024, 1, 1, 1, (60, 80)),
    ("r50.layer3.0.downsample.0", 512, 1024, 1, 1, 1, (60, 80)), ("r50.layer3.1.conv1", 1024, 256, 1, 1, 1, (60, 80)),
    ("r50.layer4.0.conv1", 1024, 512, 1, 1, 1, (60, 80)), ("r50.layer4.0.conv3", 512, 2048, 1, 1, 1, (60, 80)),
    ("r50.layer4.0.downsample.0", 1024, 2048, 1, 1, 1, (60, 80)), ("r50.layer4.1.conv1", 2048, 512, 1, 1, 1, (60, 80)),
    ("r50.fc.0", 2048, 384, 3, 1, 1, (60, 80)), ("r50.conv8s.0", 896, 256, 3, 1, 1, (60, 80)),
    ("r50.conv4s.0", 512, 128, 3, 1, 1, (120, 160)),
]
PAD_CHANNELS = 5          # convraw.0's buffer: cat[fm, image (3), 5 zero channels]


def pad_of(ksize, dilation):
    return dilation * (ksize - 1) // 2


def is_convraw(name):
    return name.endswith("convraw.0")


def buffer_channels(name, cin):
    return cin + PAD_CHANNELS if is_convraw(name) else cin


def dgrad_channels(name, cin):
    return cin - 3 if is_convraw(name) else cin


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
