"""GPU: the column kernel's tap addressing, exactly.  Each tap's A operand is a shared-memory descriptor that
starts at the tap's pixel inside the TMA halo box, off the swizzle pattern's boundary.  With a single 1.0 in
the weights at (tap, input channel, output channel) and TF32-valued inputs, the output channel must equal the
input channel shifted by the tap offset, bit for bit: a wrong start row, group stride or swizzle phase moves
or scrambles values instead of rounding them."""
import pytest
import torch

from pvnet_b200 import conv as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("ksize,cin,cout,ci,co", [
    (3, 40, 32, 35, 29),     # 8-channel chunks (convraw.0 form): last chunk, second half of its K step
    (3, 64, 64, 45, 50),     # 32-channel chunks, N = 64: second chunk, third K step
    (3, 32, 32, 7, 3),       # 32-channel chunks, N = 32
    (4, 16, 64, 13, 60),     # 16-channel chunks, 4x4 taps (space-to-depth stem form)
], ids=["kc8", "kc32-n64", "kc32-n32", "kc16-4x4"])
def test_column_kernel_one_hot_taps(ksize, cin, cout, ci, co):
    b, H, W = 2, 36, 21                              # partial tiles in both directions
    g = torch.Generator().manual_seed(ksize * 1000 + cin)
    x = pc.round_tf32(torch.randn(b, H, W, cin, generator=g)).to(DEV)
    pad = ksize // 2                                 # taps at offsets -pad .. ksize-1-pad
    xp = torch.zeros(b, H + ksize - 1, W + ksize - 1, cin, device=DEV)
    xp[:, pad:pad + H, pad:pad + W] = x
    bias = torch.zeros(cout, device=DEV)
    pc.set_mode(pc.MODE_COLUMN)
    try:
        for kh in range(ksize):
            for kw in range(ksize):
                w = torch.zeros(cout, cin, ksize, ksize, device=DEV)
                w[co, ci, kh, kw] = 1.0
                out = torch.full((b, H, W, cout), -3.0, device=DEV)
                pc.conv2d_nhwc(x, 0, cin, pc.pack_weight(w), bias, out, 0, cout, ksize)
                torch.cuda.synchronize()
                want = xp[:, kh:kh + H, kw:kw + W, ci]
                assert torch.equal(out[..., co], want), f"tap ({kh}, {kw}): output is not the shifted input channel"
                others = torch.ones(cout, dtype=torch.bool, device=DEV)
                others[co] = False
                assert (out[..., others] == 0).all(), f"tap ({kh}, {kw}): other output channels not zero"
    finally:
        pc.set_mode(pc.MODE_AUTO)
