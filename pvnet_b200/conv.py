"""Host helpers for the tensor-core convolution primitive (pvnet_conv2d_nhwc).

Weight packing (done once at load time, not on the hot path): PyTorch's
[Cout,Cin,kh,kw] conv weight with an eval-mode BatchNorm folded in
(w' = w * gamma/sqrt(var+eps), b' = beta - mean*gamma/sqrt(var+eps)) becomes the
K-major [Cout][kh*kw][Cin] matrix the kernel's weight tensor map reads, rounded to TF32.
"""
from __future__ import annotations

import ctypes

import torch
from torch.autograd.function import once_differentiable

from . import _native

ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2
MODE_AUTO, MODE_PER_TAP, MODE_COLUMN = 0, 1, 2


def set_mode(mode: int):
    """Test hook (pvnet_conv_set_mode): which kernel pvnet_conv2d_nhwc runs for layers both kernels support."""
    _native.check(_native.lib().pvnet_conv_set_mode(int(mode)), "pvnet_conv_set_mode")


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


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _workspace(dev, query_fn_name, *args):
    """A uint8 workspace on `dev` (from the caching allocator, at least 16 bytes) of the size the C ABI's
    `query_fn_name(*args, size_t *bytes)` reports."""
    n = ctypes.c_size_t()
    _native.check(getattr(_native.lib(), query_fn_name)(*args, ctypes.byref(n)), query_fn_name)
    return torch.empty(max(n.value, 16), dtype=torch.uint8, device=dev)


def conv2d_nhwc(inp, in_co, cin, w_packed, bias, out, out_co, cout, ksize, stride=1, dilation=1, act=ACT_NONE,
                res=None, res_co=0, round_out=False):
    """inp [b,H,W,in_cs] / out [b,Ho,Wo,out_cs] / res [b,Ho,Wo,res_cs]: contiguous NHWC fp32
    CUDA tensors; the conv reads channels [in_co,in_co+cin) and writes [out_co,out_co+cout)."""
    b, H, W, in_cs = inp.shape
    with torch.cuda.device(inp.device):
        _native.check(_native.lib().pvnet_conv2d_nhwc(
            _p(inp), in_cs, in_co, cin, _p(w_packed), _p(bias), _p(res), 0 if res is None else res.shape[3], res_co,
            _p(out), out.shape[3], out_co, cout, b, H, W, ksize, stride, dilation, act, int(round_out),
            _stream(inp.device)), "pvnet_conv2d_nhwc")
    return out


# ----------------------------------------------------------------------------- training (autograd)
def pack_dgrad_weight(w: torch.Tensor, n: int | None = None, tf32: bool = True) -> torch.Tensor:
    """[Cout,Cin,k,k] -> the data-gradient operand [n][k*k][cin_padded(Cout)]: taps flipped (kh,kw) ->
    (k-1-kh,k-1-kw), Cout and Cin swapped, rounded to TF32; n (default Cin) keeps the first n input channels.
    pvnet_conv2d_nhwc(dY, this, bias 0, act none, same dilation and padding) is then conv2d_input of a stride-1
    convolution (of a stride-2 one on the zero-inserted dY)."""
    wt = w.detach().flip(2, 3).transpose(0, 1)
    return pack_weight(wt if n is None else wt[:n], tf32=tf32)


def conv2d_nhwc_wgrad(inp, in_co, cin, dout, dout_co, cout, ksize, dilation=1):
    """pvnet_conv2d_nhwc_wgrad: inp [b,H,W,in_cs] and dout [b,H,W,dout_cs] contiguous NHWC fp32 on one device
    -> dW [cout,cin,ksize,ksize] fp32 (workspace from the caching allocator, current stream)."""
    b, H, W, in_cs = inp.shape
    dev = inp.device
    with torch.cuda.device(dev):
        ws = _workspace(dev, "pvnet_conv2d_nhwc_wgrad_workspace_bytes", cin, cout, b, H, W, ksize)
        dw = torch.empty(cout, cin, ksize, ksize, dtype=torch.float32, device=dev)
        _native.check(_native.lib().pvnet_conv2d_nhwc_wgrad(
            _p(inp), in_cs, in_co, cin, _p(dout), dout.shape[3], dout_co, cout, _p(dw), b, H, W, ksize, dilation,
            _p(ws), ws.numel(), _stream(dev)), "pvnet_conv2d_nhwc_wgrad")
    return dw


def zero_insert2x(inp, out=None):
    """pvnet_zero_insert2x_nhwc: inp [b,h,w,C] contiguous NHWC -> [b,2h,2w,C] with inp at the even pixels, 0 elsewhere."""
    b, h, w, C = inp.shape
    if out is None:
        out = torch.empty(b, 2 * h, 2 * w, C, dtype=torch.float32, device=inp.device)
    with torch.cuda.device(inp.device):
        _native.check(_native.lib().pvnet_zero_insert2x_nhwc(
            _p(inp), C, 0, C, _p(out), out.shape[3], 0, b, 2 * h, 2 * w, _stream(inp.device)),
            "pvnet_zero_insert2x_nhwc")
    return out


def _nhwc(t):
    """[b,C,H,W] -> its [b,H,W,C] view, after making the storage channels_last."""
    return t.contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1)


class Conv2dNHWC(torch.autograd.Function):
    """One bias-free convolution of a [b,C,H,W] channels_last tensor (physically NHWC) with a torch
    [Cout,Cin,k,k] weight, Cin <= C (the weight is zero-extended over the input's extra channels).  padding =
    dilation*(k-1)/2, the only padding Resnet18_8s uses.  Forward: pvnet_conv2d_nhwc.  Backward: the data gradient
    as pvnet_conv2d_nhwc of dY with pack_dgrad_weight (only input channels [0, dgrad_channels) get one; the rest
    are zero) and pvnet_conv2d_nhwc_wgrad; a stride-2 layer first zero-inserts dY.  Runs on the input's device and
    its current stream."""

    @staticmethod
    def forward(ctx, x, weight, stride, dilation, dgrad_channels):
        b, C, H, W = x.shape
        cout, cin, k, _ = weight.shape
        if not x.is_cuda or x.dtype != torch.float32 or weight.dtype != torch.float32:
            raise ValueError("Conv2dNHWC needs float32 CUDA tensors")
        if cin > C:
            raise ValueError(f"weight has {cin} input channels, the input {C}")
        xh = _nhwc(x)
        out = torch.empty(b, cout, H // stride, W // stride, dtype=torch.float32, device=x.device,
                          memory_format=torch.channels_last)
        wp = pack_weight(weight.detach(), cin_pad=cin_padded(C))
        bias = torch.zeros(cout, dtype=torch.float32, device=x.device)
        conv2d_nhwc(xh, 0, C, wp, bias, out.permute(0, 2, 3, 1), 0, cout, k, stride, dilation)
        ctx.save_for_backward(xh, weight)
        ctx.stride, ctx.dilation, ctx.dgrad_channels = stride, dilation, dgrad_channels
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        xh, weight = ctx.saved_tensors
        b, H, W, C = xh.shape
        cout, cin, k, _ = weight.shape
        gyh = _nhwc(gy.float())
        if ctx.stride == 2:
            gyh = zero_insert2x(gyh)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            n = C if ctx.dgrad_channels is None else ctx.dgrad_channels
            dx = torch.empty(b, C, H, W, dtype=torch.float32, device=xh.device, memory_format=torch.channels_last)
            if n < C:
                dx[:, n:].zero_()
            bias = torch.zeros(n, dtype=torch.float32, device=xh.device)
            conv2d_nhwc(gyh, 0, cout, pack_dgrad_weight(weight, n), bias, dx.permute(0, 2, 3, 1), 0, n, k, 1,
                        ctx.dilation)
        if ctx.needs_input_grad[1]:
            dw = conv2d_nhwc_wgrad(xh, 0, C, gyh, 0, cout, k, ctx.dilation)
            if cin < C:
                dw = dw[:, :cin].contiguous()
        return dx, dw, None, None, None


def conv2d_train(x, weight, stride=1, dilation=1, dgrad_channels=None):
    """Conv2dNHWC.apply: the native convolution under autograd (see Conv2dNHWC)."""
    return Conv2dNHWC.apply(x, weight, stride, dilation, dgrad_channels)


class Upsample2xCatNHWC(torch.autograd.Function):
    """torch.cat([F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=True), *rest], 1) as one
    channels_last tensor, for [b,C,h,w] `low` and [b,Ci,2h,2w] `rest` (C and C + sum Ci multiples of 4).  Forward:
    pvnet_upsample2x_nhwc writes the upsampled channels straight into the concatenated buffer (bit for bit torch's
    CUDA forward), and the `rest` tensors are copied behind them.  Backward: `low` gets pvnet_upsample2x_backward_nhwc
    of the gradient's first C channels, read in place (the terms of torch's backward in a fixed order, without
    atomics, so identical run to run); each rest[i] gets its channel slice of the gradient, as cat's backward gives
    it.  Runs on the input's device and its current stream.

    With `buf` given the concatenated buffer is the caller's: a channels_last [b,Cb,2h,2w] float32 tensor that needs
    no gradient, whose channels behind the first C + sum Ci the caller has filled (forward_train: the stem writes
    convraw.0's image and pad channels, or conv2s.0's x_ds and pad channels in Resnet50_8s_2o).  The upsampled
    channels and the `rest` tensors are written into it in place, and it is returned, marked dirty; its other
    channels are not copied in either direction."""

    @staticmethod
    def forward(ctx, low, buf, *rest):
        b, C, h, w = low.shape
        widths = [C] + [r.shape[1] for r in rest]
        if buf is None:
            if not low.is_cuda or low.dtype != torch.float32 or any(r.dtype != torch.float32 for r in rest):
                raise ValueError("Upsample2xCatNHWC needs float32 CUDA tensors")
            if any(r.shape[0] != b or r.shape[2:] != (2 * h, 2 * w) for r in rest):
                raise ValueError(f"every concatenated tensor must be [{b}, C, {2 * h}, {2 * w}]")
            if C % 4 or sum(widths) % 4:
                raise ValueError(f"C and the concatenated width must be multiples of 4, got {widths}")
            buf = torch.empty(b, sum(widths), 2 * h, 2 * w, dtype=torch.float32, device=low.device,
                              memory_format=torch.channels_last)
        else:
            _check_float_cuda("Upsample2xCatNHWC", low, buf)
            if buf.dim() != 4 or buf.shape[0] != b or tuple(buf.shape[2:]) != (2 * h, 2 * w) or buf.shape[1] < C or \
                    not buf.is_contiguous(memory_format=torch.channels_last):
                raise ValueError(f"buf must be a channels_last [{b}, >= {C}, {2 * h}, {2 * w}] tensor, got "
                                 f"{tuple(buf.shape)}")
            if buf.requires_grad:
                raise ValueError("Upsample2xCatNHWC: buf gets no gradient, so it must not require one")
            if rest and (any(r.dtype != torch.float32 or r.shape[0] != b or r.shape[2:] != (2 * h, 2 * w)
                             for r in rest) or C % 4 or sum(widths) > buf.shape[1]):
                raise ValueError(f"every concatenated tensor must be float32 [{b}, C, {2 * h}, {2 * w}], C a multiple "
                                 f"of 4, and all {widths} channels must fit in buf's {buf.shape[1]}")
            ctx.mark_dirty(buf)
        dev = low.device
        lh = _nhwc(low)
        with torch.cuda.device(dev):
            _native.check(_native.lib().pvnet_upsample2x_nhwc(
                _p(lh), C, _p(buf), buf.shape[1], 0, b, h, w, _stream(dev)), "pvnet_upsample2x_nhwc")
        co = C
        for r in rest:
            buf[:, co:co + r.shape[1]].copy_(r)
            co += r.shape[1]
        ctx.widths = widths
        return buf

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        widths = ctx.widths
        b, _, H, W = gy.shape
        C, h, w = widths[0], H // 2, W // 2
        grads = [None] * (len(widths) + 1)          # low, buf, *rest
        if ctx.needs_input_grad[0]:
            gyh = _nhwc(gy.float())
            dev = gyh.device
            dlow = torch.empty(b, C, h, w, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
            with torch.cuda.device(dev):
                _native.check(_native.lib().pvnet_upsample2x_backward_nhwc(
                    _p(gyh), gyh.shape[3], 0, C, _p(dlow), b, h, w, _stream(dev)), "pvnet_upsample2x_backward_nhwc")
            grads[0] = dlow
        co = C
        for k, c in enumerate(widths[1:], 2):
            if ctx.needs_input_grad[k]:
                grads[k] = gy[:, co:co + c]
            co += c
        return tuple(grads)


def upsample2x_cat(low, *rest):
    """Upsample2xCatNHWC.apply: cat([F.interpolate(low, x2, bilinear, align_corners=True), *rest], 1) on the native
    kernels under autograd (see Upsample2xCatNHWC)."""
    return Upsample2xCatNHWC.apply(low, None, *rest)


def upsample2x_into(low, buf, *rest):
    """Upsample2xCatNHWC.apply with the caller's buffer: the upsampled `low`, then `rest`, written into the first
    channels of `buf` under autograd, `buf` returned."""
    return Upsample2xCatNHWC.apply(low, buf, *rest)


# ----------------------------------------------------------------------------- train-mode BatchNorm (autograd)
FORM_ACT, FORM_ADD_RELU, FORM_ADD_BN_RELU = 0, 1, 2


def act_of(module) -> int:
    """The activation code of an nn.ReLU / nn.LeakyReLU(0.1) / nn.Identity module (anything else: ValueError)."""
    if isinstance(module, torch.nn.ReLU):
        return ACT_RELU
    if isinstance(module, torch.nn.LeakyReLU) and module.negative_slope == 0.1:
        return ACT_LEAKY
    if isinstance(module, torch.nn.Identity):
        return ACT_NONE
    raise ValueError(f"no native activation for {module!r} (ReLU, LeakyReLU(0.1) or Identity)")


class BatchNormState:
    """One nn.BatchNorm2d call as the native kernels take it, decided the way nn.BatchNorm2d.forward decides: batch
    statistics when the module is training (or has no running statistics), an update of running_mean/running_var
    when it also tracks them, the factor `momentum` or 1/num_batches_tracked (momentum=None), and
    num_batches_tracked.add_(1) exactly when the module would do it (at construction, i.e. once per forward call).
    It also owns the fp64 statistics [3][C] (mean, biased variance, invstd) and fp32 scale/shift [2][C] that the
    forward writes and the backward reads."""

    def __init__(self, bn, device):
        if not isinstance(bn, torch.nn.modules.batchnorm._BatchNorm):
            raise ValueError(f"expected a BatchNorm module, got {type(bn).__name__}")
        factor = 0.0 if bn.momentum is None else float(bn.momentum)
        if bn.training and bn.track_running_stats and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
            if bn.momentum is None:
                factor = 1.0 / float(bn.num_batches_tracked)      # a host read, as in nn.BatchNorm2d
        self.batch_stats = bn.training or (bn.running_mean is None and bn.running_var is None)
        use_buffers = not bn.training or bn.track_running_stats
        self.running_mean = bn.running_mean if use_buffers else None
        self.running_var = bn.running_var if use_buffers else None
        self.factor, self.eps = factor, float(bn.eps)
        C = bn.num_features
        for t in (bn.weight, bn.bias, self.running_mean, self.running_var):
            if t is not None and (t.dtype != torch.float32 or t.device != torch.device(device) or not t.is_contiguous()
                                  or t.numel() != C):
                raise ValueError("BatchNorm parameters and buffers must be contiguous float32 [C] on the input's device")
        self.saved = torch.empty(3, C, dtype=torch.float64, device=device)
        self.coef = torch.empty(2, C, dtype=torch.float32, device=device)

    def params(self, weight=None, bias=None):
        return _native.BatchNormParams(
            None if weight is None else weight.data_ptr(), None if bias is None else bias.data_ptr(),
            None if self.running_mean is None else self.running_mean.data_ptr(),
            None if self.running_var is None else self.running_var.data_ptr(),
            int(self.batch_stats), self.factor, self.eps, self.saved.data_ptr(), self.coef.data_ptr())


def _bn_check(t, C, shape=None):
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 4:
        raise ValueError("the native BatchNorm needs float32 CUDA [b,C,H,W] tensors")
    if t.shape[1] != C or (shape is not None and t.shape != shape):
        raise ValueError(f"expected {C} channels{'' if shape is None else ' and shape ' + str(tuple(shape))}, "
                         f"got {tuple(t.shape)}")


def _bn_operand(t, C, shape=None):
    _bn_check(t, C, shape)
    return _nhwc(t)


def batchnorm_forward(form, act, xh, zh, st, weight, bias, st_z=None, weight_z=None, bias_z=None):
    """pvnet_batchnorm_act_forward on NHWC views xh (and zh) -> y [b,C,H,W] channels_last; st / st_z are the
    BatchNormStates (their running statistics are updated in place, their saved/coef written)."""
    b, H, W, C = xh.shape
    dev = xh.device
    with torch.cuda.device(dev):
        ws = _workspace(dev, "pvnet_batchnorm_workspace_bytes", form, C, b * H * W)
        y = torch.empty(b, C, H, W, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        p = st.params(weight, bias)
        pz = None if st_z is None else ctypes.byref(st_z.params(weight_z, bias_z))
        _native.check(_native.lib().pvnet_batchnorm_act_forward(
            form, act, _p(xh), _p(zh), b * H * W, C, ctypes.byref(p), pz, _p(y), _p(ws), ws.numel(), _stream(dev)),
            "pvnet_batchnorm_act_forward")
    return y


def batchnorm_backward(form, act, gyh, xh, zh, st, weight, st_z=None, weight_z=None, param_grads=(True, True)):
    """pvnet_batchnorm_act_backward -> (dx, dz, dweight, dbias, dweight_z, dbias_z): dx, dz [b,C,H,W] channels_last
    (dz None for form 0), the parameter gradients [C] (None where the BatchNorm has no affine parameters or
    param_grads says they are not wanted)."""
    b, H, W, C = xh.shape
    dev = xh.device
    new = lambda: torch.empty(b, C, H, W, dtype=torch.float32, device=dev, memory_format=torch.channels_last)  # noqa
    vec = lambda w, want: None if w is None or not want else torch.empty(C, dtype=torch.float32, device=dev)  # noqa
    with torch.cuda.device(dev):
        ws = _workspace(dev, "pvnet_batchnorm_workspace_bytes", form, C, b * H * W)
        dx = new()
        dz = None if form == FORM_ACT else new()
        dw, db = vec(weight, param_grads[0]), vec(weight, param_grads[1])
        dwz = dbz = None
        if form == FORM_ADD_BN_RELU:
            dwz, dbz = vec(weight_z, param_grads[0]), vec(weight_z, param_grads[1])
        p = st.params(weight)
        pz = None if st_z is None else ctypes.byref(st_z.params(weight_z))
        _native.check(_native.lib().pvnet_batchnorm_act_backward(
            form, act, _p(gyh), _p(xh), _p(zh), b * H * W, C, ctypes.byref(p), pz, _p(dx), _p(dz), _p(dw), _p(db),
            _p(dwz), _p(dbz), _p(ws), ws.numel(), _stream(dev)), "pvnet_batchnorm_act_backward")
    return dx, dz, dw, db, dwz, dbz


class BatchNormActNHWC(torch.autograd.Function):
    """act(BatchNorm2d(x)) for a [b,C,H,W] float32 CUDA tensor (C a multiple of 4; made channels_last if it is not),
    with act none, ReLU or LeakyReLU(0.1): the `conv -> BatchNorm2d -> act` tail of Resnet18_8s's layers.  Forward:
    pvnet_batchnorm_act_forward (fp64 batch statistics over a fixed partition, the running-stat update, then one
    pass y = act(fma(x, scale, shift))).  Backward: pvnet_batchnorm_act_backward (the mask recomputed from x, fp64
    per-channel sums in a fixed order, dx = a*g + b*x + c), identical run to run.  `weight` and `bias` are the module's
    own parameters (they get gradients), `state` a BatchNormState built from the module for this call.  Saves x only
    (plus the [C] statistics).  Runs on the input's device and its current stream."""

    @staticmethod
    def forward(ctx, x, weight, bias, state, act):
        xh = _bn_operand(x, state.coef.shape[1])
        y = batchnorm_forward(FORM_ACT, act, xh, None, state, weight, bias)
        ctx.save_for_backward(xh, weight)
        ctx.state, ctx.act = state, act
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        xh, weight = ctx.saved_tensors
        dx, _, dw, db, _, _ = batchnorm_backward(FORM_ACT, ctx.act, _nhwc(gy.float()), xh, None, ctx.state, weight,
                                                 param_grads=ctx.needs_input_grad[1:3])
        return dx, dw, db, None, None


class BatchNormAddReluNHWC(torch.autograd.Function):
    """relu(bn(a) + skip) -- a BasicBlock's tail -- or, with a second BatchNorm, relu(bn(a) + bn_z(z)) -- the tail of
    a block with a downsample, both BatchNorms applied in one pass.  Forward pvnet_batchnorm_act_forward, backward
    pvnet_batchnorm_act_backward (form 1 or 2, see BatchNormActNHWC); the skip gets g = dy*relu'(pre) itself, z the
    data gradient of bn_z.  Saves a and the skip / z, tensors the block's convolutions keep anyway."""

    @staticmethod
    def forward(ctx, a, weight, bias, state, z, weight_z, bias_z, state_z):
        C = state.coef.shape[1]
        ah = _bn_operand(a, C)
        zh = _bn_operand(z, C, a.shape)
        form = FORM_ADD_RELU if state_z is None else FORM_ADD_BN_RELU
        y = batchnorm_forward(form, ACT_RELU, ah, zh, state, weight, bias, state_z, weight_z, bias_z)
        ctx.save_for_backward(ah, zh, weight, weight_z)
        ctx.state, ctx.state_z, ctx.form = state, state_z, form
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        ah, zh, weight, weight_z = ctx.saved_tensors
        n = ctx.needs_input_grad
        dx, dz, dw, db, dwz, dbz = batchnorm_backward(
            ctx.form, ACT_RELU, _nhwc(gy.float()), ah, zh, ctx.state, weight, ctx.state_z, weight_z,
            param_grads=(n[1] or n[5], n[2] or n[6]))
        return dx, dw if n[1] else None, db if n[2] else None, None, dz, dwz if n[5] else None, \
            dbz if n[6] else None, None


class BatchSizeError(ValueError, RuntimeError):
    """Batch statistics over a single value per channel.  A ValueError, as nn.BatchNorm2d raises it; also a
    RuntimeError, the class the C ABI's argument check has always reported it with."""


def _bn_batch_check(state, x):
    """nn.BatchNorm2d's _verify_batch_size, at the same point: after the module counted the batch, before any
    statistic or running buffer is touched."""
    if state.batch_stats and x.shape[0] * x.shape[2] * x.shape[3] == 1:
        raise BatchSizeError(f"expected more than one value per channel when training, got input size "
                             f"{tuple(x.shape)}")


def bn_act(bn, x, act=ACT_NONE):
    """act(bn(x)) on the native kernels under autograd, following the module's training flag, momentum, eps and
    track_running_stats (see BatchNormActNHWC, BatchNormState)."""
    _bn_check(x, bn.num_features)                 # before the state counts a batch
    state = BatchNormState(bn, x.device)
    _bn_batch_check(state, x)
    return BatchNormActNHWC.apply(x, bn.weight, bn.bias, state, act)


def bn_add_relu(bn, a, skip, bn_skip=None):
    """relu(bn(a) + skip), or relu(bn(a) + bn_skip(skip)) when bn_skip is given, on the native kernels under
    autograd (see BatchNormAddReluNHWC)."""
    _bn_check(a, bn.num_features)
    _bn_check(skip, bn.num_features, a.shape)
    state = BatchNormState(bn, a.device)
    _bn_batch_check(state, a)                     # bn raises before bn_skip runs, as in BasicBlock.forward
    if bn_skip is None:
        return BatchNormAddReluNHWC.apply(a, bn.weight, bn.bias, state, skip, None, None, None)
    return BatchNormAddReluNHWC.apply(a, bn.weight, bn.bias, state, skip, bn_skip.weight, bn_skip.bias,
                                      BatchNormState(bn_skip, a.device))


# ----------------------------------------------------------------------------- stem, max-pool and head (autograd)
def stem_s2d_index(device=None) -> torch.Tensor:
    """[256] int64 on `device` (default CPU): for entry (ty, tx, ch) of pack_stem_s2d's [4][4][16] layout, the index
    into conv1's weight flattened per output channel as [3][7][7] (c*49 + kh*7 + kw, kh = 2ty+py-1, kw = 2tx+px-1,
    ch = (py*2+px)*3+c), or 147 where the entry is a zero (kh or kw outside 0..6, or ch >= 12).  147 entries are a
    bijection onto the weights; it maps the packed weights one way and folds the s2d weight gradient back the other.
    Built with device arithmetic, so no host-to-device copy (and no stream synchronisation) is involved: the training
    stem can run inside a CUDA-graph capture."""
    i = torch.arange(256, dtype=torch.int64, device=device)
    ty, tx, ch = i // 64, (i // 16) % 4, i % 16
    par, c = ch // 3, ch % 3
    kh, kw = 2 * ty + par // 2 - 1, 2 * tx + par % 2 - 1
    ok = (ch < 12) & (kh >= 0) & (kh <= 6) & (kw >= 0) & (kw <= 6)
    return torch.where(ok, c * 49 + kh * 7 + kw, torch.full_like(i, 147))


_STEM_INDEX = {}                 # (device type, index) -> stem_s2d_index on that device


def _stem_index_on(device) -> torch.Tensor:
    """stem_s2d_index(device), built once per device.  Inside a CUDA-graph capture an index not yet cached is built
    for that call only (its memory would belong to the graph's pool)."""
    key = (device.type, device.index)
    idx = _STEM_INDEX.get(key)
    if idx is None:
        idx = stem_s2d_index(device)
        if not (device.type == "cuda" and torch.cuda.is_current_stream_capturing()):
            _STEM_INDEX[key] = idx
    return idx


def pack_stem_s2d_train(w: torch.Tensor) -> torch.Tensor:
    """pack_stem_s2d as one gather on w's device (the values are identical): [64,3,7,7] -> [64][4][4][16],
    TF32-rounded."""
    cout = w.shape[0]
    flat = torch.cat([w.reshape(cout, 147), w.new_zeros(cout, 1)], 1)
    return round_tf32(torch.index_select(flat, 1, _stem_index_on(w.device)).reshape(cout, 4, 4, 16))


def _check_float_cuda(what, *ts):
    for t in ts:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
            raise ValueError(f"{what} needs float32 CUDA tensors")


def norm3(mean, std):
    """ToTensor + Normalize constants (sequences of numbers or CPU tensors; a CUDA tensor would cost a synchronising
    read) as the two ctypes float[3] pvnet_stem_s2d_nhwc takes for a uint8 image; ValueError unless each has exactly
    three values."""
    vals = []
    for name, v in (("mean", mean), ("std", std)):
        v = [float(t) for t in (v.flatten().tolist() if isinstance(v, torch.Tensor) else v)]
        if len(v) != 3:
            raise ValueError(f"{name} must have 3 values (one per colour channel), got {len(v)}")
        vals.append((ctypes.c_float * 3)(*v))
    return vals


class StemS2dNHWC(torch.autograd.Function):
    """conv1 of Resnet18_8s (weight [64,3,7,7], stride 2, padding 3, no bias) of an image that needs no gradient, in
    either of two forms (H, W even):
    * a [b,3,H,W] float32 CUDA image, with mean and std None;
    * a raw uint8 [b,H,W,3] CUDA image with the Normalize constants mean and std (3 values each), normalised on the
      device as torchvision's ToTensor + Normalize compute it on the CPU ((u/255 - mean)/std, three correctly rounded
      fp32 ops).  Every result is the float form's for the normalised image.
    Forward: pvnet_stem_s2d_nhwc, the eval path's tensor-core form -- the 2x2 space-to-depth image S, TF32-rounded,
    and the 4x4 stride-1 convolution with the weights packed by pack_stem_s2d_train -- into a channels_last
    [b,64,H/2,W/2].  In the same pass it writes the fp32 image, unrounded, into channels [co, co+3) of `img` (a
    [b,C,H,W] channels_last float32 buffer that gets no gradient; the 5 channels behind it get zeros, the others are
    not touched): convraw.0's concatenated input.  With half=True `img` is a [b,C,H/2,W/2] buffer instead and gets
    x_ds = F.interpolate(image, scale_factor=0.5, mode='bilinear') (torch's CUDA arithmetic, bit for bit; DESIGN.md
    §21) in those channels: conv2s.0's input in Resnet50_8s_2o.  With img None (a caller that wants conv1 alone)
    those channels go to a scratch buffer.  Backward: the weight gradient only (pvnet_stem_s2d_wgrad: the 4x4
    gradient on S, all 16 taps per CTA, folded back to [64,3,7,7]).  Saves S only.  Runs on the input's device and
    its current stream."""

    @staticmethod
    def forward(ctx, x, weight, img, co, mean, std, half):
        _check_float_cuda("StemS2dNHWC", weight, *([] if img is None else [img]))
        is_u8 = x.dtype == torch.uint8
        if is_u8:
            if not x.is_cuda:
                raise ValueError(f"StemS2dNHWC needs a uint8 CUDA image, got one on {x.device}")
            if mean is None or std is None:
                raise ValueError("StemS2dNHWC: a uint8 image needs mean and std (the Normalize constants)")
            if x.dim() != 4 or x.shape[3] != 3 or x.shape[1] % 2 or x.shape[2] % 2:
                raise ValueError(f"StemS2dNHWC needs a uint8 x [b,H,W,3] with H, W even, got {tuple(x.shape)}")
            b, H, W, _ = x.shape
            mean3, std3 = norm3(mean, std)
        else:
            _check_float_cuda("StemS2dNHWC", x)
            if x.requires_grad:
                raise ValueError("StemS2dNHWC: the image gets no gradient, so it must not require one")
            if mean is not None or std is not None:
                raise ValueError("StemS2dNHWC: mean and std apply to a uint8 image; a float image is already "
                                 "normalised")
            if x.dim() != 4 or x.shape[1] != 3 or x.shape[2] % 2 or x.shape[3] % 2:
                raise ValueError(f"StemS2dNHWC needs a float x [b,3,H,W] with H, W even, got {tuple(x.shape)}")
            b, _, H, W = x.shape
            mean3 = std3 = None
        if tuple(weight.shape) != (64, 3, 7, 7):
            raise ValueError(f"StemS2dNHWC needs weight [64,3,7,7], got {tuple(weight.shape)}")
        Hi, Wi = (H // 2, W // 2) if half else (H, W)
        if img is None:
            img, co = torch.empty(b, 8, Hi, Wi, dtype=torch.float32, device=x.device,
                                  memory_format=torch.channels_last), 0
        if img.dim() != 4 or img.shape[0] != b or tuple(img.shape[2:]) != (Hi, Wi) or \
                not img.is_contiguous(memory_format=torch.channels_last):
            raise ValueError(f"img must be a channels_last [{b},C,{Hi},{Wi}] buffer, got {tuple(img.shape)}")
        if img.requires_grad:
            raise ValueError("StemS2dNHWC: img gets no gradient, so it must not require one")
        dev = x.device
        xc = x.contiguous()
        s2d = torch.empty(b, H // 2, W // 2, 16, dtype=torch.float32, device=dev)
        out = torch.empty(b, 64, H // 2, W // 2, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        w4 = pack_stem_s2d_train(weight.detach())
        bias = torch.zeros(64, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            fn = "pvnet_stem_s2d_half_nhwc" if half else "pvnet_stem_s2d_nhwc"
            _native.check(getattr(_native.lib(), fn)(
                _p(xc), int(is_u8), mean3, std3, _p(w4), _p(bias), _p(s2d), _p(out), _p(img), img.shape[1], co, b, H,
                W, _stream(dev)), fn)
        ctx.save_for_backward(s2d)
        ctx.hw = (H, W)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        if not ctx.needs_input_grad[1]:
            return None, None, None, None, None, None, None
        s2d, = ctx.saved_tensors
        b = s2d.shape[0]
        H, W = ctx.hw
        dev = s2d.device
        gyh = _nhwc(gy.float())
        with torch.cuda.device(dev):
            ws = _workspace(dev, "pvnet_stem_s2d_wgrad_workspace_bytes", b, H, W)
            dw = torch.empty(64, 3, 7, 7, dtype=torch.float32, device=dev)
            _native.check(_native.lib().pvnet_stem_s2d_wgrad(_p(s2d), _p(gyh), _p(dw), b, H, W, _p(ws), ws.numel(),
                                                             _stream(dev)), "pvnet_stem_s2d_wgrad")
        return None, dw, None, None, None, None, None


def stem_train(x, weight, img=None, co=0, mean=None, std=None):
    """StemS2dNHWC.apply: conv1 (7x7/2, pad 3, no bias) on the native kernels under autograd, of a float image or of a
    raw uint8 image normalised on the device; it also fills convraw.0's image and pad channels [co, co+8) of `img`
    when one is given (see StemS2dNHWC)."""
    return StemS2dNHWC.apply(x, weight, img, co, mean, std, False)


def stem_train_half(x, weight, img=None, co=0, mean=None, std=None):
    """stem_train for Resnet50_8s_2o: channels [co, co+8) of an H/2 x W/2 `img` get x_ds and 5 zeros, conv2s.0's image
    and pad channels (see StemS2dNHWC, half=True)."""
    return StemS2dNHWC.apply(x, weight, img, co, mean, std, True)


class MaxPool3x3s2NHWC(torch.autograd.Function):
    """nn.MaxPool2d(3, stride=2, padding=1) of a [b,C,H,W] float32 CUDA tensor (C a multiple of 4, H and W even; made
    channels_last if it is not) -> channels_last [b,C,H/2,W/2].  Forward: pvnet_maxpool3x3s2_nhwc, torch's argmax rule
    (NaN wins, ties to the first in row-major order), with a uint8 window code per output instead of int64 indices.
    Backward: pvnet_maxpool3x3s2_backward_nhwc, a gather in ATen's order without atomics.  Saves the codes only."""

    @staticmethod
    def forward(ctx, x):
        _check_float_cuda("MaxPool3x3s2NHWC", x)
        if x.dim() != 4 or x.shape[1] % 4 or x.shape[2] % 2 or x.shape[3] % 2:
            raise ValueError(f"MaxPool3x3s2NHWC needs [b,C,H,W] with C a multiple of 4 and H, W even, got "
                             f"{tuple(x.shape)}")
        b, C, H, W = x.shape
        dev = x.device
        xh = _nhwc(x)
        out = torch.empty(b, C, H // 2, W // 2, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        code = torch.empty(b, H // 2, W // 2, C, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _native.check(_native.lib().pvnet_maxpool3x3s2_nhwc(_p(xh), _p(out), _p(code), b, H, W, C, _stream(dev)),
                          "pvnet_maxpool3x3s2_nhwc")
        ctx.save_for_backward(code)
        ctx.hw = (H, W)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gy):
        code, = ctx.saved_tensors
        b, _, _, C = code.shape
        H, W = ctx.hw
        dev = code.device
        gyh = _nhwc(gy.float())
        dx = torch.empty(b, C, H, W, dtype=torch.float32, device=dev, memory_format=torch.channels_last)
        with torch.cuda.device(dev):
            _native.check(_native.lib().pvnet_maxpool3x3s2_backward_nhwc(_p(gyh), _p(code), _p(dx), b, H, W, C,
                                                                         _stream(dev)),
                          "pvnet_maxpool3x3s2_backward_nhwc")
        return dx


def maxpool_train(x):
    """MaxPool3x3s2NHWC.apply: nn.MaxPool2d(3, 2, 1) on the native kernels under autograd."""
    return MaxPool3x3s2NHWC.apply(x)


class Head1x1NCHW(torch.autograd.Function):
    """The 1x1 convolution with bias convraw.3 of a [b,Cin,H,W] float32 CUDA tensor (Cin a multiple of 32; made
    channels_last if it is not) -> a contiguous NCHW [b,Cout,H,W].  Forward: pvnet_head1x1_nchw, exact fp32 (one fmaf
    chain per output from the bias).  Backward: pvnet_head1x1_backward, the input gradient as fmaf chains and the
    weight and bias gradients as fp64 sums in a fixed order, rounded once (identical run to run); the parameter
    gradients are skipped when the parameters need none.  Saves the input and the weight."""

    @staticmethod
    def forward(ctx, y, weight, bias):
        _check_float_cuda("Head1x1NCHW", y, weight, bias)
        cout, cin = weight.shape[:2]
        if y.dim() != 4 or y.shape[1] != cin or tuple(weight.shape[2:]) != (1, 1) or tuple(bias.shape) != (cout,):
            raise ValueError(f"Head1x1NCHW needs y [b,{cin},H,W], weight [Cout,Cin,1,1] and bias [Cout], got "
                             f"{tuple(y.shape)}, {tuple(weight.shape)}, {tuple(bias.shape)}")
        b, _, H, W = y.shape
        dev = y.device
        yh = _nhwc(y)
        w2 = weight.detach().reshape(cout, cin).contiguous()
        out = torch.empty(b, cout, H, W, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _native.check(_native.lib().pvnet_head1x1_nchw(_p(yh), _p(w2), _p(bias.detach().contiguous()), _p(out), b,
                                                           H, W, cin, cout, _stream(dev)), "pvnet_head1x1_nchw")
        ctx.save_for_backward(yh, weight)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        yh, weight = ctx.saved_tensors
        b, H, W, cin = yh.shape
        cout = weight.shape[0]
        dev = yh.device
        need_y, need_w, need_b = ctx.needs_input_grad
        g = gout.float().contiguous()
        w2 = weight.detach().reshape(cout, cin).contiguous()
        dy = torch.empty(b, cin, H, W, dtype=torch.float32, device=dev,
                         memory_format=torch.channels_last) if need_y else None
        dw = torch.empty(cout, cin, dtype=torch.float32, device=dev) if need_w else None
        db = torch.empty(cout, dtype=torch.float32, device=dev) if need_b else None
        with torch.cuda.device(dev):
            ws = _workspace(dev, "pvnet_head1x1_backward_workspace_bytes", b, H, W, cin, cout) if need_w or need_b \
                else None
            _native.check(_native.lib().pvnet_head1x1_backward(
                _p(g), _p(yh), _p(w2), _p(dy), _p(dw), _p(db), b, H, W, cin, cout, _p(ws),
                0 if ws is None else ws.numel(), _stream(dev)), "pvnet_head1x1_backward")
        return dy, None if dw is None else dw.view(cout, cin, 1, 1), db


def head_train(y, weight, bias):
    """Head1x1NCHW.apply: convraw.3 (1x1 with bias) on the native kernels under autograd, as a contiguous NCHW
    tensor."""
    return Head1x1NCHW.apply(y, weight, bias)


def pack_head3x3(w: torch.Tensor) -> torch.Tensor:
    """[1,C,3,3] -> [9][C] fp32 (tap ky*3+kx, then channel; not rounded): the score head's operand
    (pvnet_head3x3_nchw, pvnet_backbone_create_detector's last slot)."""
    return w.detach().reshape(w.shape[1], 9).t().contiguous()


class Head3x3NCHW(torch.autograd.Function):
    """The detectors' score head, a 3x3 convolution with padding 1, bias and one output channel (Resnet18_8s_detector's
    fc, Resnet18_8s_detector_v2's out_conv), of a [b,C,H,W] float32 CUDA tensor (C a multiple of 32, at most 512; made
    channels_last if it is not) -> a contiguous [b,1,H,W].  Forward: pvnet_head3x3_nchw, exact fp32 (one fmaf chain
    per output from the bias in a fixed (chunk, tap, channel) order).  Backward: pvnet_head3x3_backward, the input
    gradient as fmaf chains over the taps and the weight and bias gradients as fp64 sums in a fixed order, rounded once
    (identical run to run); the parameter gradients are skipped when the parameters need none.  Saves the input and
    the weight."""

    @staticmethod
    def forward(ctx, y, weight, bias):
        _check_float_cuda("Head3x3NCHW", y, weight, bias)
        C = weight.shape[1]
        if y.dim() != 4 or y.shape[1] != C or tuple(weight.shape) != (1, C, 3, 3) or tuple(bias.shape) != (1,):
            raise ValueError(f"Head3x3NCHW needs y [b,{C},H,W], weight [1,C,3,3] and bias [1], got "
                             f"{tuple(y.shape)}, {tuple(weight.shape)}, {tuple(bias.shape)}")
        b, _, H, W = y.shape
        dev = y.device
        yh = _nhwc(y)
        w9 = pack_head3x3(weight)
        out = torch.empty(b, 1, H, W, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _native.check(_native.lib().pvnet_head3x3_nchw(_p(yh), _p(w9), _p(bias.detach().contiguous()), _p(out), b,
                                                           H, W, C, _stream(dev)), "pvnet_head3x3_nchw")
        ctx.save_for_backward(yh, weight)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, gout):
        yh, weight = ctx.saved_tensors
        b, H, W, C = yh.shape
        dev = yh.device
        need_y, need_w, need_b = ctx.needs_input_grad
        g = gout.float().contiguous()
        w9 = pack_head3x3(weight)
        dy = torch.empty(b, C, H, W, dtype=torch.float32, device=dev,
                         memory_format=torch.channels_last) if need_y else None
        dw = torch.empty(9, C, dtype=torch.float32, device=dev) if need_w else None
        db = torch.empty(1, dtype=torch.float32, device=dev) if need_b else None
        with torch.cuda.device(dev):
            ws = _workspace(dev, "pvnet_head3x3_backward_workspace_bytes", b, H, W, C) if need_w or need_b else None
            _native.check(_native.lib().pvnet_head3x3_backward(
                _p(g), _p(yh), _p(w9), _p(dy), _p(dw), _p(db), b, H, W, C, _p(ws), 0 if ws is None else ws.numel(),
                _stream(dev)), "pvnet_head3x3_backward")
        return dy, None if dw is None else dw.t().reshape(1, C, 3, 3), db


def head3x3_train(y, weight, bias):
    """Head3x3NCHW.apply: a detector's 3x3 one-channel score head on the native kernels under autograd."""
    return Head3x3NCHW.apply(y, weight, bias)
