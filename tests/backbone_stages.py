"""The native Resnet18_8s forward as the tests see it: the workspace layout and, for each of the
`pvnet_backbone_run_stage` stages, the regions it reads and writes.

Restated from pvnet_b200/csrc/backbone.cu (`carve_buffers`, `build_plans`, `run_stage`) so that a test can open
every intermediate tensor of a caller-owned workspace without any help from the library.  The CPU test
(test_backbone_stages_cpu.py) pins the layout and the stage names to the built library; the GPU test
(test_gpu_backbone_stages.py) runs the stages one at a time against this table.
"""
from typing import NamedTuple, Optional, Tuple

DEFAULT_DIMS = (256, 128, 64, 32, 32)          # fcdim, s8dim, s4dim, s2dim, raw_dim of Resnet18_8s
ALIGN = 256                                    # every buffer starts on a 256-byte boundary

# carve_buffers: allocation order
BUFFERS = ("S2D", "C1", "R0", "C2", "U2", "P", "A1", "B1", "C4", "U4", "A2", "D2", "B2", "C8", "U8",
           "A3", "D3", "B3", "E3", "A4", "D4", "B4", "E4")


def buffer_floats(dims, b, h, w):
    """Floats of each workspace buffer."""
    fc, s8, s4, s2, raw = dims
    p1 = b * h * w
    p2, p4, p8 = p1 // 4, p1 // 16, p1 // 64
    return {"S2D": p2 * 16, "C1": p1 * (s2 + 8), "R0": p1 * raw, "C2": p2 * (s4 + 64), "U2": p2 * s2,
            "P": p4 * 64, "A1": p4 * 64, "B1": p4 * 64, "C4": p4 * (s8 + 64), "U4": p4 * s4,
            "A2": p8 * 128, "D2": p8 * 128, "B2": p8 * 128, "C8": p8 * (fc + 128), "U8": p8 * s8,
            "A3": p8 * 256, "D3": p8 * 256, "B3": p8 * 256, "E3": p8 * 256,
            "A4": p8 * 512, "D4": p8 * 512, "B4": p8 * 512, "E4": p8 * 512}


def layout(dims, b, h, w):
    """(byte offset of each buffer, bytes the buffers span rounded up to ALIGN)."""
    sizes = buffer_floats(dims, b, h, w)
    off, at = 0, {}
    for name in BUFFERS:
        off = (off + ALIGN - 1) // ALIGN * ALIGN
        at[name] = off
        off += sizes[name] * 4
    return at, (off + ALIGN - 1) // ALIGN * ALIGN


class Region(NamedTuple):
    """Channels [co, co + cc) of an NHWC tensor [n, H, W, cs] that starts `off` floats into buffer `buf`.
    `buf` "x" is the NCHW input image, "out" / "mask" the caller's outputs (whole tensors)."""
    buf: str
    off: int
    grid: Tuple[int, int, int]
    cs: int
    co: int
    cc: int


class Stage(NamedTuple):
    name: str                   # pvnet_backbone_stage_name
    kind: str                   # pack, stem, pool, conv, up, head
    reads: Tuple[Region, ...]   # for a conv: its input, concatenated in this order
    writes: Tuple[Region, ...]  # empty: the stage launches nothing in this configuration
    conv: Optional[str] = None  # module names of the conv and its BatchNorm
    bn: Optional[str] = None
    act: Optional[str] = None   # relu, leaky or None
    res: Optional[Region] = None
    round_out: bool = True      # output rounded to TF32 (it feeds a tensor-core conv)


def stages(dims, seg_dim, ver_dim, b, h, w):
    """The stage table for one configuration: the tensor-core stem over the space-to-depth image, convraw.0 reading
    two dense buffers, the head fused into convraw.0 when seg_dim + ver_dim <= 32."""
    fc, s8, s4, s2, raw = dims
    p1 = b * h * w
    g1, g2, g4, g8 = (b, h, w), (b, h // 2, w // 2), (b, h // 4, w // 4), (b, h // 8, w // 8)
    c2s, c4s, c8s = s4 + 64, s8 + 64, fc + 128
    ctot = seg_dim + ver_dim
    fused = raw == 32 and ctot <= 32

    def full(buf, grid, c):
        return Region(buf, 0, grid, c, 0, c)

    x = Region("x", 0, g1, 3, 0, 3)
    s2d = full("S2D", g2, 16)
    # two dense buffers: the upsampled features, then the 8-channel image slice
    up1, img = Region("C1", 0, g1, s2, 0, s2), Region("C1", p1 * s2, g1, 8, 0, 8)
    x2s, up2 = Region("C2", 0, g2, c2s, s4, 64), Region("C2", 0, g2, c2s, 0, s4)
    x4s, up4 = Region("C4", 0, g4, c4s, s8, 64), Region("C4", 0, g4, c4s, 0, s8)
    x8s, xfc = Region("C8", 0, g8, c8s, fc, 128), Region("C8", 0, g8, c8s, 0, fc)
    P, A1, B1 = full("P", g4, 64), full("A1", g4, 64), full("B1", g4, 64)
    A2, D2, B2 = full("A2", g8, 128), full("D2", g8, 128), full("B2", g8, 128)
    A3, D3, B3, E3 = (full(n, g8, 256) for n in ("A3", "D3", "B3", "E3"))
    A4, D4, B4, E4 = (full(n, g8, 512) for n in ("A4", "D4", "B4", "E4"))
    U8, U4, U2, R0 = full("U8", g8, s8), full("U4", g4, s4), full("U2", g2, s2), full("R0", g1, raw)
    out, mask = full("out", g1, ctot), Region("mask", 0, g1, 1, 0, 1)

    T = "resnet18_8s."

    def block(name, layer, conv, inp, outp, res=None, bn=None):
        mod = f"{T}{layer}.{conv}"
        bn = bn or f"{T}{layer}.{conv.replace('conv', 'bn')}"
        act = None if conv.startswith("downsample") else "relu"
        return Stage(name, "conv", (inp,), (outp,), mod, bn, act, res)

    def dec(name, conv, inputs, outp, round_out=True):
        return Stage(name, "conv", inputs, outp, f"{conv}.0", f"{conv}.1", "leaky", None, round_out)

    return [
        Stage("image: space-to-depth + NHWC slice packing", "pack", (x,), (s2d, img)),
        Stage("stem conv1+bn1+relu", "stem", (s2d,), (x2s,), T + "conv1", T + "bn1", "relu"),
        Stage("maxpool 3x3/2", "pool", (x2s,), (P,)),
        block("layer1.0.conv1", "layer1.0", "conv1", P, A1),
        block("layer1.0.conv2", "layer1.0", "conv2", A1, B1, res=P),
        block("layer1.1.conv1", "layer1.1", "conv1", B1, A1),
        block("layer1.1.conv2", "layer1.1", "conv2", A1, x4s, res=B1),
        block("layer2.0.conv1 (s2)", "layer2.0", "conv1", x4s, A2),
        block("layer2.0.downsample (1x1 s2)", "layer2.0", "downsample.0", x4s, D2, bn=T + "layer2.0.downsample.1"),
        block("layer2.0.conv2", "layer2.0", "conv2", A2, B2, res=D2),
        block("layer2.1.conv1", "layer2.1", "conv1", B2, A2),
        block("layer2.1.conv2", "layer2.1", "conv2", A2, x8s, res=B2),
        block("layer3.0.conv1 (d2)", "layer3.0", "conv1", x8s, A3),
        block("layer3.0.downsample (1x1)", "layer3.0", "downsample.0", x8s, D3, bn=T + "layer3.0.downsample.1"),
        block("layer3.0.conv2 (d2)", "layer3.0", "conv2", A3, B3, res=D3),
        block("layer3.1.conv1 (d2)", "layer3.1", "conv1", B3, A3),
        block("layer3.1.conv2 (d2)", "layer3.1", "conv2", A3, E3, res=B3),
        block("layer4.0.conv1 (d4)", "layer4.0", "conv1", E3, A4),
        block("layer4.0.downsample (1x1)", "layer4.0", "downsample.0", E3, D4, bn=T + "layer4.0.downsample.1"),
        block("layer4.0.conv2 (d4)", "layer4.0", "conv2", A4, B4, res=D4),
        block("layer4.1.conv1 (d4)", "layer4.1", "conv1", B4, A4),
        block("layer4.1.conv2 (d4)", "layer4.1", "conv2", A4, E4, res=B4),
        Stage("fc.0", "conv", (E4,), (xfc,), T + "fc.0", T + "fc.1", "relu"),
        # the decoder's torch.cat order (Resnet18_8s._forward_torch): upsampled features first, skip second
        dec("conv8s.0", "conv8s", (xfc, x8s), (U8,)),
        Stage("upsample 1/8->1/4", "up", (U8,), (up4,)),
        dec("conv4s.0", "conv4s", (up4, x4s), (U4,)),
        Stage("upsample 1/4->1/2", "up", (U4,), (up2,)),
        dec("conv2s.0", "conv2s", (up2, x2s), (U2,)),
        Stage("upsample 1/2->1", "up", (U2,), (up1,)),
        dec("convraw.0", "convraw", (up1, img), (out, mask) if fused else (R0,), round_out=False),
        Stage("convraw.3 1x1 + argmax head (fp32)", "head", (R0,), () if fused else (out, mask), "convraw.3"),
    ]
