"""The native Resnet*_8s forward as the tests see it: the workspace layout and, for each of the
`pvnet_backbone_run_stage` stages, the regions it reads and writes, for any trunk `pvnet_backbone_create_trunk` plans.

Restated from pvnet_b200/csrc/backbone.cu (`generate`, `carve_buffers`, `build_plans`, `run_stage`) so that a test can
open every intermediate tensor of a caller-owned workspace without any help from the library.  The CPU test
(test_backbone_stages_cpu.py) pins the layout and the stage names to the built library; the GPU test
(test_gpu_backbone_stages.py) runs the stages one at a time against this table.
"""
from typing import NamedTuple, Optional, Tuple

DEFAULT_DIMS = (256, 128, 64, 32, 32)          # fcdim, s8dim, s4dim, s2dim, raw_dim of Resnet18_8s
DEEP_DIMS = (384, 256, 128, 64, 64)            # ... of Resnet34_8s and Resnet50_8s
ALIGN = 256                                    # every buffer starts on a 256-byte boundary


class Trunk(NamedTuple):
    """What `pvnet_backbone_create_trunk` plans from: block kind, blocks per stage, decoder widths; and where the
    trunk's modules live in the network (Resnet34_8s keeps its trunk under `resnet50_8s.`)."""
    bottleneck: bool
    blocks: Tuple[int, int, int, int]
    dims: Tuple[int, int, int, int, int]      # fcdim, s8dim, s4dim, s2dim, raw_dim
    prefix: str

    @property
    def expansion(self):
        return 4 if self.bottleneck else 1


RESNET18 = Trunk(False, (2, 2, 2, 2), DEFAULT_DIMS, "resnet18_8s.")
RESNET34 = Trunk(False, (3, 4, 6, 3), DEEP_DIMS, "resnet50_8s.")
RESNET50 = Trunk(True, (3, 4, 6, 3), DEEP_DIMS, "resnet50_8s.")


def _stage_buffers(trunk, s):
    """Names of stage s's own buffers (s = 1..4) in carving order: A (conv1's output), M (a Bottleneck's conv2
    output), D (the downsample's), B and E (block outputs; E only where a block output has to avoid B)."""
    n = trunk.blocks[s - 1]
    has_ds = s > 1 or trunk.bottleneck         # stride 2, or a width change in layer1
    return ([f"A{s}"] + ([f"M{s}"] if trunk.bottleneck else []) + ([f"D{s}"] if has_ds else []) + [f"B{s}"]
            + ([f"E{s}"] if s >= 3 or n > 2 else []))


def buffers(trunk):
    """Buffer names in carve_buffers' allocation order."""
    out = ["S2D", "C1", "R0", "C2", "U2", "P"]
    for s in range(1, 5):
        out += _stage_buffers(trunk, s) + {1: ["C4", "U4"], 2: ["C8", "U8"]}.get(s, [])
    return out


def _levels_and_channels(trunk):
    """{buffer: (level, channels)}: NHWC fp32 at resolution 1/2^level."""
    fc, s8, s4, s2, raw = trunk.dims
    e = trunk.expansion
    spec = {"S2D": (1, 16), "C1": (0, s2 + 8), "R0": (0, raw), "C2": (1, s4 + 64), "U2": (1, s2), "P": (2, 64),
            "C4": (2, s8 + 64 * e), "U4": (2, s4), "C8": (3, fc + 128 * e), "U8": (3, s8)}
    for s in range(1, 5):
        planes, level = 64 << (s - 1), 2 if s == 1 else 3
        # a Bottleneck's conv1 (1x1) reads at the stage's input resolution; its conv2 carries the stride
        a_level = 2 if trunk.bottleneck and s == 2 else level
        for name in _stage_buffers(trunk, s):
            spec[name] = (a_level, planes) if name[0] == "A" else (level, planes if name[0] == "M" else planes * e)
    return spec


def buffer_floats(trunk, b, h, w):
    """Floats of each workspace buffer."""
    p1 = b * h * w
    return {name: (p1 >> (2 * lv)) * ch for name, (lv, ch) in _levels_and_channels(trunk).items()}


def layout(trunk, b, h, w):
    """(byte offset of each buffer, bytes the buffers span rounded up to ALIGN)."""
    sizes = buffer_floats(trunk, b, h, w)
    off, at = 0, {}
    for name in buffers(trunk):
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
    name: str                   # pvnet_backbone_handle_stage_name
    kind: str                   # pack, stem, pool, conv, up, head
    reads: Tuple[Region, ...]   # for a conv: its input, concatenated in this order
    writes: Tuple[Region, ...]  # empty: the stage launches nothing in this configuration
    conv: Optional[str] = None  # module names of the conv and its BatchNorm
    bn: Optional[str] = None
    act: Optional[str] = None   # relu, leaky or None
    res: Optional[Region] = None
    round_out: bool = True      # output rounded to TF32 (it feeds a tensor-core conv)


def stages(trunk, seg_dim, ver_dim, b, h, w):
    """The stage table for one configuration: the tensor-core stem over the space-to-depth image, the trunk's blocks
    (resnet.py's stage rule: layer3 / layer4 dilate instead of striding), convraw.0 reading two dense buffers, the head
    fused into convraw.0 when raw_dim is 32 and seg_dim + ver_dim <= 32."""
    fc, s8, s4, s2, raw = trunk.dims
    e, T = trunk.expansion, trunk.prefix
    p1 = b * h * w
    grids = {0: (b, h, w), 1: (b, h // 2, w // 2), 2: (b, h // 4, w // 4), 3: (b, h // 8, w // 8)}
    g1, g2, g4, g8 = grids[0], grids[1], grids[2], grids[3]
    c2s, c4s, c8s = s4 + 64, s8 + 64 * e, fc + 128 * e
    ctot = seg_dim + ver_dim
    fused = raw == 32 and ctot <= 32
    spec = _levels_and_channels(trunk)

    def full(buf):
        level, c = spec[buf]
        return Region(buf, 0, grids[level], c, 0, c)

    x = Region("x", 0, g1, 3, 0, 3)
    s2d = full("S2D")
    # two dense buffers: the upsampled features, then the 8-channel image slice
    up1, img = Region("C1", 0, g1, s2, 0, s2), Region("C1", p1 * s2, g1, 8, 0, 8)
    x2s, up2 = Region("C2", 0, g2, c2s, s4, 64), Region("C2", 0, g2, c2s, 0, s4)
    x4s, up4 = Region("C4", 0, g4, c4s, s8, 64 * e), Region("C4", 0, g4, c4s, 0, s8)
    x8s, xfc = Region("C8", 0, g8, c8s, fc, 128 * e), Region("C8", 0, g8, c8s, 0, fc)
    out, mask = Region("out", 0, g1, ctot, 0, ctot), Region("mask", 0, g1, 1, 0, 1)

    def conv(name, mod, inp, outp, res=None, act="relu"):
        bn = mod[:-1] + "1" if mod.endswith("downsample.0") else mod.replace(".conv", ".bn")
        return Stage(name, "conv", (inp,), (outp,), T + mod, T + bn, act, res)

    def dec(name, conv, inputs, outp, round_out=True):
        return Stage(name, "conv", inputs, outp, f"{conv}.0", f"{conv}.1", "leaky", None, round_out)

    table = [
        Stage("image: space-to-depth + NHWC slice packing", "pack", (x,), (s2d, img)),
        Stage("stem conv1+bn1+relu", "stem", (s2d,), (x2s,), T + "conv1", T + "bn1", "relu"),
        Stage("maxpool 3x3/2", "pool", (x2s,), (full("P"),)),
    ]
    xr = full("P")
    for s in range(1, 5):
        n = trunk.blocks[s - 1]
        stride = 2 if s == 2 else 1              # output stride 8 reached in layer2: layer3 and layer4 dilate
        dil = {3: 2, 4: 4}.get(s, 1)
        dtag = f" (d{dil})" if dil > 1 else ""
        names = _stage_buffers(trunk, s)
        A, B = full(names[0]), full(f"B{s}")
        M = full(f"M{s}") if trunk.bottleneck else None
        D = full(f"D{s}") if f"D{s}" in names else None
        E = full(f"E{s}") if f"E{s}" in names else None
        last = {1: x4s, 2: x8s}.get(s, E)
        for i in range(n):
            pre = f"layer{s}.{i}."
            st = stride if i == 0 else 1
            left = n - 1 - i
            y = last if left == 0 else (B if left % 2 else E)    # the last block writes the stage's output
            tag3 = " (s2)" if st == 2 else dtag
            res = xr
            ds = []
            if i == 0 and D is not None:        # the downsample runs just before the conv whose epilogue adds it
                ds = [conv(pre + ("downsample (1x1 s2)" if st == 2 else "downsample (1x1)"), pre + "downsample.0",
                           xr, D, act=None)]
                res = D
            if trunk.bottleneck:
                # A is sized for layer2.0's conv1, at the input resolution; later blocks use its first 1/4
                a = A._replace(grid=xr.grid)
                table += [conv(pre + "conv1 (1x1)", pre + "conv1", xr, a),
                          conv(pre + "conv2" + tag3, pre + "conv2", a, M)]
                table += ds + [conv(pre + "conv3 (1x1)", pre + "conv3", M, y, res)]
            else:
                table += [conv(pre + "conv1" + tag3, pre + "conv1", xr, A)]
                table += ds + [conv(pre + "conv2" + dtag, pre + "conv2", A, y, res)]
            xr = y
    R0 = full("R0")
    table += [
        Stage("fc.0", "conv", (xr,), (xfc,), T + "fc.0", T + "fc.1", "relu"),
        # the decoder's torch.cat order (_Resnet8s._forward_torch): upsampled features first, skip second
        dec("conv8s.0", "conv8s", (xfc, x8s), (full("U8"),)),
        Stage("upsample 1/8->1/4", "up", (full("U8"),), (up4,)),
        dec("conv4s.0", "conv4s", (up4, x4s), (full("U4"),)),
        Stage("upsample 1/4->1/2", "up", (full("U4"),), (up2,)),
        dec("conv2s.0", "conv2s", (up2, x2s), (full("U2"),)),
        Stage("upsample 1/2->1", "up", (full("U2"),), (up1,)),
        dec("convraw.0", "convraw", (up1, img), (out, mask) if fused else (R0,), round_out=False),
        Stage("convraw.3 1x1 + argmax head (fp32)", "head", (R0,), () if fused else (out, mask), "convraw.3"),
    ]
    return table
