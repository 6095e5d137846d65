"""GPU: the per-tap convolution's epilogue stages each 32-channel slab of a finished tile in shared memory and
stores it with TMA (residual slabs arrive the same way).  Only the route of the bytes changed, so every stored value
must equal the digests recorded with the direct register -> global epilogue
(tests/golden/make_golden_conv_tap_store.py), next to an fp64 restatement; nothing outside the destination's channel
slice may be written, TMA's clipping included; and two runs must give the same bytes.

Every shape has 160 M tiles (8x16 pixels each), so on the 132 SMs of an H100 conv_plan picks N = 32, 64, 128, 256,
256 for Cout = 32, 64, 128, 256, 512: one, two, four and eight slabs per item, and two items per CTA for some CTAs.
60x80 has a partial last tile row, 13x21 partial tiles in both directions, 8x16 none."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pvnet_b200 import conv as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conv_tap_store.json")

COUTS = (32, 64, 128, 256, 512)
SHAPES = ((4, 60, 80), (40, 13, 21), (160, 8, 16))      # b, H, W
CIN, KSIZE, DIL = 64, 3, 1
PAD_C = 32              # the destination and the residual are channel slices [PAD_C, PAD_C + Cout) of wider buffers
SENTINEL = -7.25
# activation (0 none, 1 ReLU, 2 LeakyReLU(0.1)) x round_out x residual
VARIANTS = [(act, rnd, res) for act in (pc.ACT_NONE, pc.ACT_RELU, pc.ACT_LEAKY) for rnd in (False, True)
            for res in (False, True)]


def case_key(cout, shape, act, rnd, res):
    return f"cout{cout}_b{shape[0]}_{shape[1]}x{shape[2]}_act{act}_round{int(rnd)}_res{int(res)}"


def make_inputs(cout, shape):
    """Seeded operands on the device: x [b,H,W,CIN] with TF32-exact values, weights [cout,CIN,3,3], bias [cout], and
    the residual as a channel slice of a [b,H,W,cout + 2*PAD_C] buffer."""
    b, H, W = shape
    g = torch.Generator(device="cpu").manual_seed(cout * 7919 + b * 131 + H * 17 + W)
    x = pc.round_tf32(torch.randn(b, H, W, CIN, generator=g).to(DEV))
    w = (torch.randn(cout, CIN, KSIZE, KSIZE, generator=g) / np.sqrt(CIN * KSIZE * KSIZE)).to(DEV)
    bias = torch.randn(cout, generator=g).to(DEV)
    res_buf = torch.randn(b, H, W, cout + 2 * PAD_C, generator=g).to(DEV)
    return x, w, bias, res_buf


def run_case(x, w_packed, bias, res_buf, cout, act, rnd, with_res):
    """One per-tap launch into channels [PAD_C, PAD_C + cout) of a sentinel-filled buffer that is one pixel row longer
    than the tensor the kernel is told about.  Returns the whole flat buffer [b*H*W + W, cout + 2*PAD_C]."""
    b, H, W, _ = x.shape
    cs = cout + 2 * PAD_C
    flat = torch.full((b * H * W + W, cs), SENTINEL, device=DEV)
    out = flat[:b * H * W].view(b, H, W, cs)
    pc.set_mode(pc.MODE_PER_TAP)
    try:
        pc.conv2d_nhwc(x, 0, CIN, w_packed, bias, out, PAD_C, cout, KSIZE, 1, DIL, act, res_buf if with_res else None,
                       PAD_C, round_out=rnd)
        torch.cuda.synchronize()
    finally:
        pc.set_mode(pc.MODE_AUTO)
    return flat


def digest(flat, cout):
    """sha256 of the destination slice's bytes"""
    return hashlib.sha256(flat[:, PAD_C:PAD_C + cout].contiguous().cpu().numpy().tobytes()).hexdigest()


def reference_fp64(x, w, bias):
    """The convolution in fp64 from what the MMA sees (TF32-rounded weights; x is TF32-exact already), + bias:
    [b,H,W,cout]"""
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), pc.round_tf32(w).double(), bias.double(),
                   padding=DIL * (KSIZE - 1) // 2, dilation=DIL)
    return ref.permute(0, 2, 3, 1)


def finish_fp64(pre, res_buf, cout, act, with_res):
    v = pre + res_buf[..., PAD_C:PAD_C + cout].double() if with_res else pre
    if act == pc.ACT_RELU:
        v = F.relu(v)
    elif act == pc.ACT_LEAKY:
        v = torch.maximum(v, 0.1 * v)
    return v


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN_PATH) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "b%d_%dx%d" % s)
@pytest.mark.parametrize("cout", COUTS)
def test_tap_store(golden, cout, shape):
    b, H, W = shape
    x, w, bias, res_buf = make_inputs(cout, shape)
    wp = pc.pack_weight(w)
    pre = reference_fp64(x, w, bias)
    npix = b * H * W
    for act, rnd, with_res in VARIANTS:
        what = case_key(cout, shape, act, rnd, with_res)
        flat = run_case(x, wp, bias, res_buf, cout, act, rnd, with_res)
        # nothing but the slice was written: the channels on both sides, and the pixel row behind the tensor
        assert bool((flat[:, :PAD_C] == SENTINEL).all()) and bool((flat[:, PAD_C + cout:] == SENTINEL).all()), \
            f"{what}: channels outside the destination slice were written"
        assert bool((flat[npix:] == SENTINEL).all()), f"{what}: pixels behind the tensor were written"
        got = flat[:npix, PAD_C:PAD_C + cout].view(b, H, W, cout)
        ref = finish_fp64(pre, res_buf, cout, act, with_res)
        scale = max(ref.abs().max().item(), 1.0)
        tol = 2e-5 * scale + 1e-5 + (scale * 2.0 ** -11 if rnd else 0.0)       # round_out: half a TF32 ulp more
        err = (got.double() - ref).abs().max().item()
        assert err <= tol, f"{what}: max err {err:.3e} against fp64 (scale {scale:.2f})"
        if rnd:
            assert bool(((got.view(torch.int32) & 0x1FFF) == 0).all()), f"{what}: stored values are not TF32"
        d = digest(flat, cout)
        assert d == digest(run_case(x, wp, bias, res_buf, cout, act, rnd, with_res), cout), \
            f"{what}: two runs gave different bytes"
        assert d == golden[what], f"{what}: bytes differ from the digest recorded with the direct epilogue"
