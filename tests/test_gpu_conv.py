"""GPU: the wgmma convolution primitive against torch (fp64 reference computed from
TF32-truncated operands: isolates indexing / layout / descriptor errors from TF32 rounding)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pvnet_b200 import conv as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _run_case(b, H, W, cin, cout, k, stride, dil, act, with_res, in_extra=0, out_extra=0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(b, cin, H, W, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / np.sqrt(cin * k * k)
    bias = torch.randn(cout, generator=g)
    Ho, Wo = H // stride, W // stride
    res = torch.randn(b, cout, Ho, Wo, generator=g) if with_res else None
    # reference: fp64 conv of tf32-rounded weights and tf32-TRUNCATED activations (what the MMA sees)
    wq = pc.round_tf32(w)
    xq = _trunc_tf32(x)
    ref = F.conv2d(xq.double(), wq.double(), bias.double(), stride=stride, padding=dil * (k - 1) // 2, dilation=dil)
    if with_res:
        ref = ref + res.double()
    if act == 1:
        ref = F.relu(ref)
    elif act == 2:
        ref = F.leaky_relu(ref, 0.1)
    # device buffers, NHWC, with channel padding on both sides to exercise offsets
    in_cs, in_co = cin + in_extra, in_extra // 2 // 4 * 4
    out_cs, out_co = cout + out_extra, out_extra // 2 // 4 * 4
    xin = torch.full((b, H, W, in_cs), 7.0, device=DEV)
    xin[..., in_co:in_co + cin] = x.permute(0, 2, 3, 1).to(DEV)
    out = torch.full((b, Ho, Wo, out_cs), -3.0, device=DEV)
    resd = res.permute(0, 2, 3, 1).contiguous().to(DEV) if with_res else None
    wp = pc.pack_weight(w.to(DEV))
    pc.conv2d_nhwc(xin, in_co, cin, wp, bias.to(DEV), out, out_co, cout, k, stride, dil, act, resd, 0)
    torch.cuda.synchronize()
    got = out[..., out_co:out_co + cout].permute(0, 3, 1, 2).double().cpu()
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-5 * max(scale, 1.0) + 1e-5, f"max err {err:.3e} (scale {scale:.2f})"
    # untouched padding channels
    if out_extra:
        mask = torch.ones(out_cs, dtype=torch.bool)
        mask[out_co:out_co + cout] = False
        assert (out[..., mask.to(DEV)] == -3.0).all()


@pytest.mark.parametrize("cfg", [
    # b, H,  W,  cin, cout, k, s, d, act, res
    (1, 16, 32, 32, 32, 1, 1, 1, 0, False),     # smallest: single K-block, exact tiles
    (1, 16, 32, 32, 32, 3, 1, 1, 0, False),     # 9 taps, zero padding via TMA OOB fill
    (2, 24, 40, 64, 64, 3, 1, 1, 1, True),      # partial tiles, residual + ReLU (BasicBlock)
    (1, 24, 40, 128, 256, 3, 1, 2, 1, False),   # dilation 2 (layer3)
    (1, 24, 40, 64, 512, 3, 1, 4, 1, True),     # dilation 4, two N tiles (layer4)
    (2, 24, 40, 128, 256, 1, 1, 1, 0, False),   # 1x1 downsample, no stride
    (2, 48, 80, 64, 128, 3, 2, 1, 1, False),    # stride-2 3x3 through parity planes (layer2.0.conv1)
    (2, 48, 80, 64, 128, 1, 2, 1, 0, False),    # stride-2 1x1 downsample
    (1, 40, 48, 40, 32, 3, 1, 1, 2, False),     # Cin=40 -> 8-channel K-blocks (convraw.0), LeakyReLU
    (1, 60, 80, 384, 128, 3, 1, 1, 2, False),   # conv8s shape
])
@pytest.mark.parametrize("persistent", [True, False], ids=["persistent", "tile-per-cta"])
def test_conv_vs_torch(cfg, persistent):
    pc.set_mode(pc.MODE_PER_TAP)
    pc.set_persistent(persistent)
    try:
        _run_case(*cfg)
    finally:
        pc.set_persistent(True)
        pc.set_mode(pc.MODE_AUTO)


def test_conv_persistent_many_items_per_cta():
    """More (M tile, N tile) items than resident CTAs: every CTA loops, the TMA ring runs on across items."""
    pc.set_mode(pc.MODE_PER_TAP)
    try:
        _run_case(4, 120, 160, 64, 128, 3, 1, 1, 1, True, seed=11)     # 600 items, 1 CTA/SM
        _run_case(2, 60, 80, 128, 512, 1, 1, 1, 0, False, seed=12)     # four N tiles per M tile
    finally:
        pc.set_mode(pc.MODE_AUTO)


@pytest.mark.parametrize("cfg", [
    # the persistent weights-resident column kernel (3x3, stride 1, Cout <= 64)
    (1, 16, 32, 32, 32, 3, 1, 1, 0, False),     # one tile, one chunk
    (2, 24, 40, 64, 64, 3, 1, 1, 1, True),      # layer1 BasicBlock conv2: residual + ReLU, partial tiles, N=64
    (1, 40, 48, 40, 32, 3, 1, 1, 2, False),     # convraw.0: Cin=40 -> 8-channel chunks, LeakyReLU
    (1, 48, 80, 128, 32, 3, 1, 1, 2, False),    # conv2s.0 shape (weights 147 KB resident)
    (3, 64, 96, 64, 64, 3, 1, 1, 1, False),     # many tiles per CTA: exercises the persistent loop
    (1, 32, 40, 192, 64, 3, 1, 1, 2, False),    # conv4s.0 shape: 442 KB of weights -> tiles stream with the A boxes
    (2, 20, 44, 64, 64, 3, 1, 1, 1, True),      # width and height not multiples of the 16 x 8 tile, residual
])
def test_conv_column_kernel_vs_torch(cfg):
    pc.set_mode(pc.MODE_COLUMN)
    try:
        _run_case(*cfg)
    finally:
        pc.set_mode(pc.MODE_AUTO)


def test_conv_column_kernel_rejects_dilation():
    """The halo-box kernel is dilation-1 only; forcing it on a dilated layer is an error, not a fallback."""
    pc.set_mode(pc.MODE_COLUMN)
    try:
        with pytest.raises((RuntimeError, ValueError)):
            _run_case(1, 24, 40, 32, 32, 3, 1, 2, 0, False)
    finally:
        pc.set_mode(pc.MODE_AUTO)


def test_conv_column_kernel_large_persistent():
    """More tiles than resident CTAs (one per SM): every CTA loops several times."""
    pc.set_mode(pc.MODE_COLUMN)
    try:
        _run_case(2, 240, 320, 40, 32, 3, 1, 1, 2, False, seed=3)
    finally:
        pc.set_mode(pc.MODE_AUTO)


def test_conv_channel_offsets():
    _run_case(1, 24, 40, 64, 64, 3, 1, 1, 2, False, in_extra=32, out_extra=64)


def test_conv_round_out_is_tf32():
    x = torch.randn(1, 16, 32, 32, device=DEV)
    w = torch.randn(32, 32, 1, 1, device=DEV)
    out = torch.empty(1, 16, 32, 32, device=DEV)
    pc.conv2d_nhwc(x, 0, 32, pc.pack_weight(w), torch.zeros(32, device=DEV), out, 0, 32, 1, round_out=True)
    assert ((out.view(torch.int32) & 0x1FFF) == 0).all()


def _run_4x4_case(cout, seed):
    """ksize 4 = taps at offsets {-2,-1,0,1} (the space-to-depth form of the 7x7/2 stem), Cin=16 -> 64-byte
    swizzled rows, weights [cout][4][4][16] resident."""
    g = torch.Generator().manual_seed(seed)
    b, H, W = 2, 40, 56
    x = torch.randn(b, 16, H, W, generator=g)
    w = torch.randn(cout, 16, 4, 4, generator=g) / 16.0
    bias = torch.randn(cout, generator=g)
    ref = F.relu(F.conv2d(F.pad(_trunc_tf32(x), (2, 1, 2, 1)).double(), pc.round_tf32(w).double(), bias.double()))
    xin = x.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.full((b, H, W, cout + 32), -3.0, device=DEV)        # 32 channels beyond cout must stay untouched
    pc.conv2d_nhwc(xin, 0, 16, pc.pack_weight(w.to(DEV)), bias.to(DEV), out, 0, cout, 4, 1, 1, pc.ACT_RELU)
    torch.cuda.synchronize()
    err = (out[..., :cout].permute(0, 3, 1, 2).double().cpu() - ref).abs().max().item()
    assert err <= 2e-5 * max(ref.abs().max().item(), 1.0) + 1e-5, err
    assert (out[..., cout:] == -3.0).all()


def test_conv_column_kernel_4x4_s2d_stem_shape():
    """The stem's shape: 64 output channels."""
    _run_4x4_case(64, 4)


def test_conv_column_kernel_4x4_cout32():
    """A 4x4 layer with 32 output channels runs on its own instantiation (N = 32)."""
    _run_4x4_case(32, 5)


@pytest.mark.parametrize("mc", [1, 0], ids=["multicast", "single-cta"])
@pytest.mark.parametrize("cfg", [
    (1, 24, 40, 128, 256, 3, 1, 2, 1, False),   # 9 M tiles: odd -> the last cluster's 2nd CTA duplicates a tile
    (2, 24, 40, 64, 512, 3, 1, 4, 1, True),     # four N tiles, residual
    (2, 60, 80, 256, 256, 1, 1, 1, 0, False),   # 1x1, 80 M tiles
])
def test_conv_cluster_multicast(cfg, mc):
    """Wide layers: 2-CTA clusters sharing each weight tile through TMA multicast vs the plain launch."""
    pc.set_mode(pc.MODE_PER_TAP)
    pc.set_multicast(mc)
    try:
        _run_case(*cfg)
        pc.set_persistent(False)      # one (M tile pair, N tile) per cluster
        _run_case(*cfg)
    finally:
        pc.set_persistent(True)
        pc.set_multicast(0)
        pc.set_mode(pc.MODE_AUTO)
