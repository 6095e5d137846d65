"""GPU: the native Resnet18_8s, Resnet34_8s and Resnet50_8s forwards one launch at a time, each stage against an fp64
restatement of its own layer.

The end-to-end tests (test_gpu_backbone.py, test_gpu_deep_backbones.py) bound the whole network by the error
cuDNN-TF32 makes over 26, 36 or 53 layers; a fault that moves one layer by 0.1 % hides in that.  Here every stage of
`pvnet_backbone_run_stage` runs on a workspace the test owns (layout and stage table: tests/backbone_stages.py), and
for each one:

(a) exactly its output region changes: the rest of the workspace and the guard bands around `out` and the mask keep
    their bytes;
(b) its region is fully written: the NaN sentinel the region is filled with before the launch is gone, including
    partial tiles, the zero channels of the image slice and of the space-to-depth image;
(c) what a tensor-core conv reads, and what every stage but convraw.0 writes, is TF32-valued (low 13 bits zero);
(d) its values match an fp64 reference computed from the snapshot of its own inputs, so errors do not accumulate
    and a failure names the stage.

The reference is independent of the host layer: BatchNorm is folded here from the module's statistics, the stem is
the module's 7x7/2 convolution (not the 4x4 space-to-depth form the library packs), and the weights, activations and
concatenation order come from the module.  r(.) is rounding to TF32 (nearest, ties away from zero).

Bounds, per element:
  conv / stem        |got - ref| <= 2^-11 |ref| + acc, acc = 1e-5 R (tests/helpers.py conv_acc_bound)
                     (output rounding to TF32; fp32 accumulation of K exact TF32 products).  R is the same conv on
                     absolute values plus |bias| and |residual|, so the term grows with K: Resnet50_8s's fc.0 sums
                     K = 18 432 products, where the largest (|err| - 2^-11 |ref|) / R measured on an H100 was 1.7e-6
                     (2.8e-6 for the same shape in test_gpu_conv.py).  Where K <= 4608 (all of Resnet18_8s) acc is
                     also held to 2e-5 max(max|ref|, 1) + 1e-5.  The 2^-11 term is dropped where the output is not
                     rounded (convraw.0 -> R0)
  upsample x2        2^-11 |ref| + 2^-20 max|src|      (output rounding; fp32 interpolation weights and sums)
  fused head         sum_k |W_ck| (2^-10 |a_k| + acc_k) + 1e-6   (a = convraw.0's activation, which may land on
                     either TF32 neighbour before the head MMA)
  k_head (fp32)      2^-18 sum_k |W_ck R0_k| + 2^-23 |b_c|   (32 or 64 fp32 FMAs: 64 2^-24 is the worst case of 64)
  pack, max-pool     bit-exact;  mask: torch.argmax of the stage's own logits (first maximum wins), exact.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pvnet_b200 import _native
from pvnet_b200.model_repository import Resnet18_8s, Resnet34_8s, Resnet50_8s
from tests import backbone_stages as bs
from tests.helpers import conv_acc_bound, seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD, GUARD_BYTE = 1 << 16, 0xA5        # bytes of margin around `out` and the mask, and their fill
# Before a stage runs its output region is filled with 0xFF bytes: as fp32 a NaN no stage computes, as a mask
# element -1 / 255, no class index.

NARROW = (128, 64, 32, 64, 32)           # convraw.0 in = 64 + 8 channels: the non-wide fused-head variant
WIDE_S2 = (256, 128, 64, 256, 32)        # convraw.0 in = 256 + 8: 33 eight-channel chunks x 9 taps x 32 outputs of
                                         # weights (297 KB) exceed shared memory, so the fused head streams them
                                         # with each A stage (resident = 0 in conv_col_plan_at; checked with a
                                         # printf there while writing this test)
NETS = {Resnet18_8s: bs.RESNET18, Resnet34_8s: bs.RESNET34, Resnet50_8s: bs.RESNET50}
CASES = [
    # id, network, ver_dim, seg_dim, decoder widths, (b, h, w)
    ("k9-2x64x96", Resnet18_8s, 18, 2, bs.DEFAULT_DIMS, (2, 64, 96)),
    ("k9-1x72x104", Resnet18_8s, 18, 2, bs.DEFAULT_DIMS, (1, 72, 104)),  # 1/8 grid 9 x 13: odd stride-2 parity planes
    ("k9-3x16x16", Resnet18_8s, 18, 2, bs.DEFAULT_DIMS, (3, 16, 16)),
    ("k9-1x256x264", Resnet18_8s, 18, 2, bs.DEFAULT_DIMS, (1, 256, 264)),
    ("k9-16x480x640", Resnet18_8s, 18, 2, bs.DEFAULT_DIMS, (16, 480, 640)),  # bench.py --config 2
    ("k17-4x480x640", Resnet18_8s, 34, 2, bs.DEFAULT_DIMS, (4, 480, 640)),   # bench.py --config 5: unfused k_head
    ("k17-2x48x64", Resnet18_8s, 34, 2, bs.DEFAULT_DIMS, (2, 48, 64)),
    ("k17-2x64x96", Resnet18_8s, 34, 2, bs.DEFAULT_DIMS, (2, 64, 96)),
    ("k17-1x72x104", Resnet18_8s, 34, 2, bs.DEFAULT_DIMS, (1, 72, 104)),
    # head width 21: odd, channel 21 in the padding
    ("narrow-seg3-1x72x104", Resnet18_8s, 18, 3, NARROW, (1, 72, 104)),
    ("s2dim256-1x72x104", Resnet18_8s, 18, 2, WIDE_S2, (1, 72, 104)),
    # the deep networks (raw_dim 64: k_head at Cin 64): 1x1 Bottleneck convs up to Cin 2048, fc.0 over 2048 channels
    # (K = 18 432), decoder inputs of 320 / 512 / 896 channels, convraw.0 reading 64 + 8 channels
    ("r34-k9-2x64x96", Resnet34_8s, 18, 2, bs.DEEP_DIMS, (2, 64, 96)),
    ("r34-k9-1x72x104", Resnet34_8s, 18, 2, bs.DEEP_DIMS, (1, 72, 104)),
    ("r34-k9-1x480x640", Resnet34_8s, 18, 2, bs.DEEP_DIMS, (1, 480, 640)),
    ("r50-k9-2x64x96", Resnet50_8s, 18, 2, bs.DEEP_DIMS, (2, 64, 96)),
    ("r50-k9-1x72x104", Resnet50_8s, 18, 2, bs.DEEP_DIMS, (1, 72, 104)),     # Bottleneck conv2 (s2) onto 9 x 13
    ("r50-k9-1x480x640", Resnet50_8s, 18, 2, bs.DEEP_DIMS, (1, 480, 640)),
]
OUTPUT_FORMS = [(False, torch.int64), (True, torch.uint8), (False, torch.uint8), (True, torch.int64)]


def _r(t):
    """fp32 -> nearest TF32 value, ties away from zero (cvt.rna.tf32.f32), kept in fp32."""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def _trunc(t):
    """What the tensor cores read of an fp32 operand: the low 13 mantissa bits dropped."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _fold(mods, conv, bn):
    """BatchNorm folded into the conv in fp64 from the module's eval statistics, then cast to fp32."""
    w = mods[conv].weight.detach().double()
    if bn is None:
        return w.float(), mods[conv].bias.detach().float()
    m = mods[bn]
    scale = m.weight.detach().double() / torch.sqrt(m.running_var.detach().double() + m.eps)
    return (w * scale[:, None, None, None]).float(), (m.bias.detach().double() - m.running_mean.detach().double() * scale).float()


def _conv_bound(ref, R, K, rounded):
    """Output rounding to TF32 (where the output is rounded) plus fp32 accumulation."""
    return (2.0 ** -11 * ref.abs() if rounded else 0) + conv_acc_bound(ref, R, K)


def _within(what, got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = torch.nan_to_num(err / bound, nan=float("inf"))
    worst = ratio.max().item()
    assert worst <= 1.0, (f"{what}: {int((ratio > 1).sum())} of {ratio.numel()} elements outside the bound, worst "
                          f"|err|/bound {worst:.3g} (max |err| {err.max().item():.3g})")
    return worst


def _bits_equal(what, got, ref):
    got, ref = got.contiguous().view(torch.int32), ref.float().contiguous().view(torch.int32)
    bad = int((got != ref).sum())
    assert bad == 0, f"{what}: {bad} of {got.numel()} elements differ from the bit-exact reference"
    return 0.0


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _upsample_ref(src):
    """nn.UpsamplingBilinear2d(scale_factor=2) of NHWC `src` in fp64, with ATen's fp32 source coordinates:
    scale = (in-1)/(out-1), src = scale*dst, l1 = src - floor(src), l0 = 1 - l1."""
    def axis(n):
        scale = torch.tensor(float(n - 1), dtype=torch.float32) / torch.tensor(float(2 * n - 1), dtype=torch.float32)
        s = scale.to(src.device) * torch.arange(2 * n, dtype=torch.float32, device=src.device)
        i0 = s.floor()
        l1 = s - i0
        i0 = i0.long()
        return i0, (i0 + 1).clamp(max=n - 1), (1 - l1).double(), l1.double()

    y0, y1, hy0, hy1 = axis(src.shape[1])
    x0, x1, wx0, wx1 = axis(src.shape[2])
    s = src.double()
    rows = lambda yi: wx0[None, :, None] * s[:, yi][:, :, x0] + wx1[None, :, None] * s[:, yi][:, :, x1]
    return hy0[None, :, None, None] * rows(y0) + hy1[None, :, None, None] * rows(y1)


class _Guarded:
    """A tensor inside a larger allocation whose margins hold GUARD_BYTE."""

    def __init__(self, shape, dtype):
        nbytes = int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size()
        self.buf = torch.full((2 * GUARD + nbytes,), GUARD_BYTE, dtype=torch.uint8, device=DEV)
        self.t = self.buf[GUARD:GUARD + nbytes].view(dtype).view(shape)

    def margins_intact(self):
        return bool((self.buf[:GUARD] == GUARD_BYTE).all() and (self.buf[-GUARD:] == GUARD_BYTE).all())


class _StageRun:
    def __init__(self, net, trunk, x, seg, ver):
        self.net, self.trunk, self.x, self.seg, self.ver = net, trunk, x, seg, ver
        self.ctot = seg + ver
        self.b, _, self.h, self.w = x.shape
        self.mods = dict(net.named_modules())
        self.table = bs.stages(trunk, seg, ver, self.b, self.h, self.w)
        self.L = _native.lib()
        self.handle = net._prepare_native(DEV)
        self.num_stages = self.L.pvnet_backbone_handle_num_stages(self.handle)
        assert [s.name for s in self.table] == [self.L.pvnet_backbone_handle_stage_name(self.handle, i).decode()
                                                for i in range(self.num_stages)], "stage table is stale"
        n = ctypes.c_size_t()
        _native.check(self.L.pvnet_backbone_workspace_bytes(self.handle, self.b, self.h, self.w, ctypes.byref(n)),
                      "pvnet_backbone_workspace_bytes")
        self.at, total = bs.layout(trunk, self.b, self.h, self.w)
        assert n.value == total + 256, "workspace layout of tests/backbone_stages.py is stale"
        self.nbytes = n.value
        raw = torch.full((self.nbytes + 256,), 0xFF, dtype=torch.uint8, device=DEV)
        shift = (-raw.data_ptr()) % 256
        self._raw, self.ws = raw, raw[shift:shift + self.nbytes]
        self.worst, self.acc = {}, {}

    # ---------------------------------------------------------------- outputs and regions
    def set_outputs(self, pixel_major, mask_dtype):
        b, h, w, c = self.b, self.h, self.w, self.ctot
        self.pixel_major = pixel_major
        self.out = _Guarded([b, h, w, c] if pixel_major else [b, c, h, w], torch.float32)
        self.mask = _Guarded([b, h, w], mask_dtype)
        _native.check(self.L.pvnet_backbone_set_output_layout(self.handle, int(pixel_major)), "set_output_layout")

    def region(self, r, base=None):
        """The region's elements as a strided view, NHWC; fp32 data viewed as int32."""
        if r.buf == "out":
            t = self.out.t.view(torch.int32)
            return t if self.pixel_major else _nhwc(t)
        if r.buf == "mask":
            return self.mask.t[..., None]
        n, h, w = r.grid
        start = self.at[r.buf] // 4 + r.off
        wsi = (self.ws if base is None else base).view(torch.int32)
        return wsi[start:start + n * h * w * r.cs].view(n, h, w, r.cs)[..., r.co:r.co + r.cc]

    def f32(self, r, n):
        """Image n of a workspace region as fp32 [1, H, W, cc]."""
        return self.region(r)[n:n + 1].contiguous().view(torch.float32)

    # ---------------------------------------------------------------- one stage
    def run(self, i):
        st = self.table[i]
        for r in st.writes:
            t = self.region(r)
            t.fill_(255 if t.dtype == torch.uint8 else -1)
        snap, osnap, msnap = self.ws.clone(), self.out.buf.clone(), self.mask.buf.clone()
        mptr = self.mask.t.data_ptr()
        _native.check(self.L.pvnet_backbone_run_stage(
            self.handle, i, self.x.data_ptr(), self.b, self.h, self.w, self.out.t.data_ptr(), mptr,
            self.mask.t.element_size(), self.ws.data_ptr(), self.nbytes,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), f"run_stage({st.name})")
        torch.cuda.synchronize()
        ws_writes = [r for r in st.writes if r.buf not in ("out", "mask")]
        # (a) nothing outside the stage's regions changed
        got = [self.region(r).clone() for r in ws_writes]
        for r in ws_writes:
            self.region(r).copy_(self.region(r, snap))
        bad = self._first_difference(snap)
        for r, g in zip(ws_writes, got):
            self.region(r).copy_(g)
        assert bad is None, f"{st.name}: wrote outside its output region, into {bad}"
        writes_out = any(r.buf == "out" for r in st.writes)
        if writes_out:
            assert self.out.margins_intact() and self.mask.margins_intact(), f"{st.name}: wrote past `out` or the mask"
        else:
            assert torch.equal(self.out.buf, osnap) and torch.equal(self.mask.buf, msnap), f"{st.name}: touched `out` or the mask"
        del snap, osnap, msnap
        if not st.writes:
            return False
        # (b) fully written
        for r in st.writes:
            t = self.region(r)
            left = int((t == (255 if t.dtype == torch.uint8 else -1)).sum())
            assert left == 0, f"{st.name}: {left} elements of {r.buf} [{r.co}, {r.co + r.cc}) never written"
        # (c) TF32 invariant
        if st.kind in ("conv", "stem"):
            for r in st.reads:
                assert not (self.region(r) & 0x1FFF).any(), f"{st.name}: tensor-core input {r.buf} is not TF32-valued"
        for r in ws_writes:
            if r.buf != "R0":
                assert not (self.region(r) & 0x1FFF).any(), f"{st.name}: output {r.buf} is not TF32-valued"
        # (d) values, one image at a time
        worst = 0.0
        for n in range(self.b):
            worst = max(worst, getattr(self, "_check_" + st.kind)(st, n))
        self.worst[st.name] = max(worst, self.worst.get(st.name, 0.0))
        return True

    def _first_difference(self, snap, chunk=1 << 26):
        a, b = self.ws.view(torch.int32), snap.view(torch.int32)
        for s in range(0, a.numel(), chunk):
            if not torch.equal(a[s:s + chunk], b[s:s + chunk]):
                k = s + int(torch.nonzero(a[s:s + chunk] != b[s:s + chunk])[0, 0])
                byte = 4 * k
                names = [name for name in self.at if self.at[name] <= byte]
                return f"{names[-1]} at float {(byte - self.at[names[-1]]) // 4}" if names else f"byte {byte}"
        return None

    # ---------------------------------------------------------------- references
    def _conv_input(self, st, n):
        return torch.cat([self.f32(r, n) for r in st.reads], 3)

    def _conv_ref(self, st, inp, n):
        """(the layer in fp64, R: the same sum over absolute values, before the activation)."""
        conv = self.mods[st.conv]
        w, b = _fold(self.mods, st.conv, st.bn)
        xq, wq = _nchw(_trunc(inp[..., :conv.in_channels])).double(), _r(w).double()
        y = _nhwc(F.conv2d(xq, wq, None, conv.stride, conv.padding, conv.dilation)) + b.double()
        R = _nhwc(F.conv2d(xq.abs(), wq.abs(), None, conv.stride, conv.padding, conv.dilation)) + b.double().abs()
        if st.res is not None:
            res = self.f32(st.res, n).double()
            y, R = y + res, R + res.abs()
        if st.act == "relu":
            y = y.clamp_min(0)
        elif st.act == "leaky":
            y = torch.where(y > 0, y, 0.1 * y)
        return y, R

    def _K(self, st):
        """Products per output element."""
        w = self.mods[st.conv].weight
        return w.shape[1] * w.shape[2] * w.shape[3]

    def _note_acc(self, st, got, ref, R, rounded):
        """Records max (|got - ref| - rounding) / R: how close the accumulation comes to the R term."""
        err = (got.double() - ref).abs() - (2.0 ** -11 * ref.abs() if rounded else 0)
        r = float(torch.where(err > 0, err / R, torch.zeros_like(err)).max())
        self.acc[st.name] = max(r, self.acc.get(st.name, 0.0))

    def _check_pack(self, st, n):
        rx = _nhwc(_r(self.x[n:n + 1]))
        h2, w2 = self.h // 2, self.w // 2
        img = F.pad(rx, (0, 5))
        s2d = rx.reshape(1, h2, 2, w2, 2, 3).permute(0, 1, 3, 2, 4, 5).reshape(1, h2, w2, 12)
        _bits_equal(f"{st.name}: space-to-depth image", self.region(st.writes[0])[n:n + 1], F.pad(s2d, (0, 4)))
        return _bits_equal(f"{st.name}: image slice", self.region(st.writes[-1])[n:n + 1], img)

    def _check_stem(self, st, n):
        x = _nhwc(self.x[n:n + 1])
        ref, R = self._conv_ref(st, _r(x), n)
        got = self.f32(st.writes[0], n)
        self._note_acc(st, got, ref, R, True)
        return _within(st.name, got, ref, _conv_bound(ref, R, self._K(st), True))

    def _check_pool(self, st, n):
        ref = _nhwc(self.mods[self.trunk.prefix + "maxpool"](_nchw(self.f32(st.reads[0], n))))
        return _bits_equal(st.name, self.region(st.writes[0])[n:n + 1], ref)

    def _check_up(self, st, n):
        src = self.f32(st.reads[0], n)
        ref = _upsample_ref(src)
        bound = 2.0 ** -11 * ref.abs() + 2.0 ** -20 * src.abs().max().item()
        return _within(st.name, self.f32(st.writes[0], n), ref, bound)

    def _logits_got(self, n):
        o = self.out.t[n:n + 1]
        return o if self.pixel_major else _nhwc(o)

    def _check_mask(self, st, n):
        logits = self._logits_got(n)[..., :self.seg]
        assert torch.equal(self.mask.t[n:n + 1].long(), torch.argmax(logits, -1)), \
            f"{st.name}: mask is not torch.argmax of the stage's own logits"

    def _head_weights(self):
        """convraw.3 as packed: rounded to TF32 at raw_dim 32 (the fused head's MMA reads it), fp32 at raw_dim 64."""
        w, b = _fold(self.mods, "convraw.3", None)
        w = w.reshape(w.shape[0], -1)
        return (_r(w) if self.trunk.dims[4] == 32 else w).double(), b.double()

    def _check_conv(self, st, n):
        ref, R = self._conv_ref(st, self._conv_input(st, n), n)
        if st.writes[0].buf != "out":
            got = self.f32(st.writes[0], n)
            self._note_acc(st, got, ref, R, st.round_out)
            return _within(st.name, got, ref, _conv_bound(ref, R, self._K(st), st.round_out))
        # convraw.0 with convraw.3 + argmax in its epilogue: the head MMA reads r(a)
        W, bh = self._head_weights()
        logits = _r(ref.float()).double() @ W.T + bh
        bound = (2.0 ** -10 * ref.abs() + conv_acc_bound(ref, R, self._K(st))) @ W.abs().T + 1e-6
        worst = _within(f"{st.name} + fused head", self._logits_got(n), logits, bound)
        self._check_mask(st, n)
        return worst

    def _check_head(self, st, n):
        r0 = self.f32(st.reads[0], n).double()
        W, bh = self._head_weights()
        ref = r0 @ W.T + bh
        bound = 2.0 ** -18 * (r0.abs() @ W.abs().T) + 2.0 ** -23 * bh.abs()
        worst = _within(st.name, self._logits_got(n), ref, bound)
        self._check_mask(st, n)
        return worst


def _net(cls, ver, seg, dims, seed):
    net = cls(ver, seg, *dims)
    net.load_state_dict(seeded_state_dict(net, seed=seed))
    return net.to(DEV).eval()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_every_stage_against_its_own_layer(case):
    name, cls, ver, seg, dims, (b, h, w) = case
    x = torch.from_numpy(np.random.default_rng(h * w + b).standard_normal((b, 3, h, w), dtype=np.float32)).to(DEV)
    try:
        with torch.no_grad():
            run = _StageRun(_net(cls, ver, seg, dims, seed=21), NETS[cls]._replace(dims=dims), x, seg, ver)
            run.set_outputs(*OUTPUT_FORMS[0])
            checked = 0
            for i, st in enumerate(run.table):
                if any(r.buf == "out" for r in st.writes):
                    for form in OUTPUT_FORMS:        # the stage that writes `out` and the mask, in every form
                        run.set_outputs(*form)
                        run.run(i)
                    checked += 1
                else:
                    checked += run.run(i)
    finally:
        torch.cuda.synchronize()
    idle = 1 if dims[4] == 32 and seg + ver <= 32 else 0        # the head, when convraw.0 carries it
    assert checked == run.num_stages - idle
    print(f"\n[stages {name}] worst |err|/bound per stage: " +
          ", ".join(f"{k}: {v:.2g}" for k, v in run.worst.items()))
    kinds = {}
    for st in run.table:
        if st.name in run.worst:
            kind = st.kind if st.kind != "conv" else "conv " + ("1x1" if run._K(st) == run.mods[st.conv].in_channels
                                                                 else "3x3")
            kinds[kind] = max(kinds.get(kind, 0.0), run.worst[st.name])
    print(f"[stages {name}] worst |err|/bound per kind: " + ", ".join(f"{k}: {v:.2g}" for k, v in kinds.items()))
    print(f"[stages {name}] max (|err| - rounding) / R per conv: " +
          ", ".join(f"{k} (K={run._K(st)}): {run.acc[k]:.2g}" for st in run.table for k in [st.name] if k in run.acc))


# ---------------------------------------------------------------------------------------------- argmax ties
@pytest.mark.parametrize("ver,seg,groups", [(18, 10, [(0, 1), (5, 6), (2, 9)]), (34, 3, [(1, 2)])],
                         ids=["fused head", "k_head"])
def test_head_argmax_ties(ver, seg, groups):
    """Seg channels in tie groups (same convraw.3 row and bias) give bit-equal logits -- the same products summed in
    the same order -- and the mask is the lowest index of the winning group, torch.argmax's first maximum.  The
    fused head's groups cross each boundary of its argmax: {0, 1} within a lane, {5, 6} across lanes, {2, 9}
    across lanes and 8-channel blocks.  Every other seg channel is biased far down."""
    net = Resnet18_8s(ver, seg)
    net.load_state_dict(seeded_state_dict(net, seed=4))
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        wt, bias = net.convraw[3].weight, net.convraw[3].bias
        bias[:seg] = -1e4
        for grp in groups:
            row, b0 = torch.randn(32, generator=g) * 0.3, torch.randn(1, generator=g).item() * 0.1
            for c in grp:
                wt[c, :, 0, 0] = row
                bias[c] = b0
    net.to(DEV).eval()
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((2, 3, 64, 96), dtype=np.float32)).to(DEV)
    for pixel_major, mask_dtype in OUTPUT_FORMS:
        with torch.no_grad():
            out, mask = net.forward_native(x, with_mask=True, mask_dtype=mask_dtype, pixel_major=pixel_major)
        logits = (out.permute(0, 3, 1, 2) if pixel_major else out)[:, :seg]
        for grp in groups:
            for c in grp[1:]:
                assert torch.equal(logits[:, c].view(torch.int32), logits[:, grp[0]].view(torch.int32)), \
                    f"tied channels {grp[0]} and {c} differ"
        assert torch.equal(mask.long(), torch.argmax(logits, 1))
        winners = torch.unique(mask.long()).tolist()
        assert set(winners) <= {min(grp) for grp in groups}
        assert len(winners) == len(groups), f"every tie group should win somewhere, winners {winners}"
