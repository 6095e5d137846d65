"""GPU: the per-tap convolution at the 1/8-resolution shapes of the benchmark (batch 16, 60x80), where
conv_plan picks 256-channel N tiles, against an fp64 reference; and the wide tile against the 128-channel
one bit for bit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pvnet_b200 import conv as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _inputs(b, H, W, cin, cout, k, with_res, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(b, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / np.sqrt(cin * k * k)
    bias = torch.randn(cout, generator=g)
    res = torch.randn(b, cout, H, W, generator=g) if with_res else None
    return x.to(DEV), w.to(DEV), bias.to(DEV), None if res is None else res.to(DEV)


def _conv(x_nhwc, w, bias, cout, k, dil, act, res_nhwc):
    b, H, W, cin = x_nhwc.shape
    out = torch.full((b, H, W, cout), -3.0, device=DEV)
    pc.conv2d_nhwc(x_nhwc, 0, cin, pc.pack_weight(w), bias, out, 0, cout, k, 1, dil, act, res_nhwc, 0)
    return out


@pytest.mark.parametrize("cfg", [
    # b,  H,  W, cin, cout, k, d, act, res
    (16, 60, 80, 256, 512, 3, 4, 1, False),     # layer4.0.conv1
    (16, 60, 80, 512, 512, 3, 4, 1, True),      # layer4.x.conv2: residual + ReLU
    (16, 60, 80, 512, 256, 3, 1, 1, False),     # fc.0
])
def test_conv_bench_shapes_vs_fp64(cfg):
    b, H, W, cin, cout, k, dil, act, with_res = cfg
    x, w, bias, res = _inputs(b, H, W, cin, cout, k, with_res, seed=21)
    pc.set_mode(pc.MODE_PER_TAP)
    try:
        got = _conv(x.permute(0, 2, 3, 1).contiguous(), w, bias, cout, k, dil, act,
                    None if res is None else res.permute(0, 2, 3, 1).contiguous())
        torch.cuda.synchronize()
    finally:
        pc.set_mode(pc.MODE_AUTO)
    # fp64 on the device from what the MMA sees: tf32-rounded weights, tf32-truncated activations
    ref = F.conv2d(_trunc_tf32(x).double(), pc.round_tf32(w).double(), bias.double(), padding=dil * (k - 1) // 2,
                   dilation=dil)
    if with_res:
        ref = ref + res.double()
    ref = F.relu(ref)
    err = (got.permute(0, 3, 1, 2).double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-5 * max(scale, 1.0) + 1e-5, f"max err {err:.3e} (scale {scale:.2f})"


def test_conv_wide_tile_equals_128_channel_slices():
    """Cout 512 at the benchmark's layer4 shape runs on 256-channel N tiles; each 128-channel slice of its
    weights alone runs on 128-channel tiles. Every output element sums the same K sequence either way,
    so the results are identical, not merely close."""
    b, H, W, cin, cout, k, dil = 16, 60, 80, 512, 512, 3, 4
    x, w, bias, res = _inputs(b, H, W, cin, cout, k, True, seed=22)
    xin = x.permute(0, 2, 3, 1).contiguous()
    resn = res.permute(0, 2, 3, 1).contiguous()
    pc.set_mode(pc.MODE_PER_TAP)
    try:
        wide = _conv(xin, w, bias, cout, k, dil, pc.ACT_RELU, resn)
        parts = [_conv(xin, w[i:i + 128].contiguous(), bias[i:i + 128].contiguous(), 128, k, dil, pc.ACT_RELU,
                       resn[..., i:i + 128].contiguous())
                 for i in range(0, cout, 128)]
        torch.cuda.synchronize()
    finally:
        pc.set_mode(pc.MODE_AUTO)
    assert torch.equal(wide, torch.cat(parts, dim=3))
