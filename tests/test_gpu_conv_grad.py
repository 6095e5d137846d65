"""Native convolution backward on the H100: pvnet_conv2d_nhwc_wgrad, the data gradient through pvnet_conv2d_nhwc with
pack_dgrad_weight, zero insertion for the stride-2 layers, the Conv2dNHWC autograd Function and
Resnet18_8s.forward_train.

Per layer the reference is the fp64 operation on the operands as the MMA sees them (activations and gradients
TF32-valued, weights as packed), bounded by |got - ref| <= 1e-5 * R with R the same operation on absolute values."""
import copy

import numpy as np
import pytest
import torch
from torch.nn.grad import conv2d_input

from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s
from tests import conv_grad_cases as cg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def _check(got, ref, absref, what):
    err = (got.double() - ref).abs()
    bound = 1e-5 * absref
    worst = float((err - bound).max().detach())
    assert worst <= 0, f"{what}: max |got-ref| {float(err.max()):.3e}, exceeds 1e-5 R by {worst:.3e}"


def _case(row, b, hw, seed):
    name, cin, cout, k, stride, dil, _ = row
    g = torch.Generator(device=DEV).manual_seed(seed)
    ho, wo = hw
    cbuf = cg.buffer_channels(name, cin)
    x = pc.round_tf32(torch.randn(b, cbuf, ho * stride, wo * stride, device=DEV, generator=g))
    if cg.is_convraw(name):
        x[:, cin:] = 0
    dy = pc.round_tf32(torch.randn(b, cout, ho, wo, device=DEV, generator=g))
    w = torch.randn(cout, cin, k, k, device=DEV, generator=g) * 0.1
    return x, dy, w


def _dgrad_native(dy, w, n, stride, dil):
    k = w.shape[2]
    gy = _nhwc(dy)
    if stride == 2:
        gy = pc.zero_insert2x(gy)
    b, H, W, cout = gy.shape
    out = torch.full((b, H, W, n), float("nan"), device=DEV)
    pc.conv2d_nhwc(gy, 0, cout, pc.pack_dgrad_weight(w, n), torch.zeros(n, device=DEV), out, 0, n, k, 1, dil)
    return out.permute(0, 3, 1, 2)


def _wgrad_native(x, dy, k, stride, dil):
    gy = _nhwc(dy)
    if stride == 2:
        gy = pc.zero_insert2x(gy)
    return pc.conv2d_nhwc_wgrad(_nhwc(x), 0, x.shape[1], gy, 0, dy.shape[1], k, dil)


def _layer_check(row, b, hw, seed, co=None, ci=None):
    name, cin, cout, k, stride, dil, _ = row
    x, dy, w = _case(row, b, hw, seed)
    n = cg.dgrad_channels(name, cin)
    pad = cg.pad_of(k, dil)
    # data gradient: the weights as packed (TF32), in fp64
    packed = pc.pack_dgrad_weight(w, n)
    wq = cg.unpack_dgrad(packed, n, cout, k).flip(2, 3).transpose(0, 1).double()     # back to [Cout, n, k, k]
    got = _dgrad_native(dy, w, n, stride, dil)
    shape = (b, n, x.shape[2], x.shape[3])
    ref = conv2d_input(shape, wq, dy.double(), stride=stride, padding=pad, dilation=dil)
    absref = conv2d_input(shape, wq.abs(), dy.double().abs(), stride=stride, padding=pad, dilation=dil)
    assert torch.isfinite(got).all()
    _check(got, ref, absref, f"{name} dgrad")
    # weight gradient (optionally on a channel window, reference only: the kernel computes all of dW)
    dw = _wgrad_native(x, dy, k, stride, dil)
    assert dw.shape == (cout, x.shape[1], k, k)
    co = slice(None) if co is None else co
    ci = slice(None) if ci is None else ci
    xd, dyd = x[:, ci].double(), dy[:, co].double()
    ref = cg.wgrad_stride1_form(xd, dyd, k, stride, dil)
    absref = cg.wgrad_stride1_form(xd.abs(), dyd.abs(), k, stride, dil)
    _check(dw[co, ci], ref, absref, f"{name} wgrad")


@pytest.mark.parametrize("row", cg.ROWS, ids=[r[0] for r in cg.ROWS])
def test_layer_reduced(row):
    # 9 x 13 output pixels: partial 32-pixel K-blocks, image borders inside blocks, batch 3
    _layer_check(row, 3, (9, 13), 10)


def test_convraw0_full_resolution():
    row = [r for r in cg.ROWS if r[0] == "convraw.0"][0]
    _layer_check(row, 2, (480, 640), 11)


def test_layer4_full_batch16():
    row = [r for r in cg.ROWS if r[0] == "layer4.1.conv1"][0]
    # all of dW is computed; the fp64 reference covers a window across the 128-channel tile edges
    _layer_check(row, 16, (60, 80), 12, co=slice(96, 224), ci=slice(96, 224))


def test_wgrad_workspace_stays_bounded():
    # the split planner keeps the partial tiles to at most 128 MB and a modest split count, at the largest shapes:
    # Resnet18_8s's, and the deep networks' fc.0 over 2048 channels (a 28 MB dW), their widest 1x1 convs, the 1x1
    # convs at 1/4 resolution (stride 2: the zero-inserted grid), the 896- and 512-channel decoder inputs and convraw.0
    import ctypes
    from pvnet_b200 import _native
    for cin, cout, b, h, w, k in ((512, 512, 32, 60, 80, 3), (40, 32, 32, 480, 640, 3), (64, 64, 32, 120, 160, 3),
                                  (2048, 384, 32, 60, 80, 3), (2048, 512, 32, 60, 80, 1), (512, 2048, 32, 60, 80, 1),
                                  (1024, 2048, 32, 60, 80, 1), (64, 256, 32, 120, 160, 1), (256, 64, 32, 120, 160, 1),
                                  (256, 512, 32, 120, 160, 1), (896, 256, 32, 60, 80, 3), (512, 128, 32, 120, 160, 3),
                                  (72, 64, 32, 480, 640, 3)):
        n = ctypes.c_size_t()
        with torch.cuda.device(DEV):
            _native.check(_native.lib().pvnet_conv2d_nhwc_wgrad_workspace_bytes(cin, cout, b, h, w, k, ctypes.byref(n)),
                          "pvnet_conv2d_nhwc_wgrad_workspace_bytes")
        splits = n.value // (cout * cin * k * k * 4)
        assert n.value <= 128 << 20 and 1 <= splits <= 512, (cin, cout, n.value, splits)


def test_channel_offsets_and_strides():
    g = torch.Generator(device=DEV).manual_seed(3)
    b, H, W, cin, cout = 2, 10, 14, 64, 128
    x = pc.round_tf32(torch.randn(b, H, W, 80, device=DEV, generator=g))
    dy = pc.round_tf32(torch.randn(b, H, W, 140, device=DEV, generator=g))
    dw_slices = pc.conv2d_nhwc_wgrad(x, 8, cin, dy, 4, cout, 3, 2)
    dw_dense = pc.conv2d_nhwc_wgrad(x[..., 8:8 + cin].contiguous(), 0, cin, dy[..., 4:4 + cout].contiguous(), 0,
                                    cout, 3, 2)
    assert torch.equal(dw_slices, dw_dense)
    # zero insertion into a channel slice of a wider buffer: the neighbours stay as they were
    src = torch.randn(b, H // 2, W // 2, 32, device=DEV, generator=g)
    buf = torch.full((b, H, W, 48), float("nan"), device=DEV)
    torch.cuda.synchronize()
    import ctypes
    from pvnet_b200 import _native
    _native.check(_native.lib().pvnet_zero_insert2x_nhwc(
        ctypes.c_void_p(src.data_ptr()), 32, 0, 32, ctypes.c_void_p(buf.data_ptr()), 48, 8, b, H, W,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pvnet_zero_insert2x_nhwc")
    assert torch.isnan(buf[..., :8]).all() and torch.isnan(buf[..., 40:]).all()
    ref = cg.zero_insert(src.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    assert torch.equal(buf[..., 8:40], ref)
    # the data gradient written into a slice (pvnet_conv2d_nhwc's out_co) leaves the other channels alone
    w = torch.randn(cout, cin, 3, 3, device=DEV, generator=g)
    out = torch.full((b, H, W, 96), float("nan"), device=DEV)
    pc.conv2d_nhwc(dy[..., :cout].contiguous(), 0, cout, pc.pack_dgrad_weight(w), torch.zeros(cin, device=DEV), out,
                   32, cin, 3, 1, 1)
    assert torch.isnan(out[..., :32]).all() and torch.isfinite(out[..., 32:]).all()


def test_backward_is_deterministic():
    for row in (cg.ROWS[4], cg.ROWS[16], cg.ROWS[23]):
        name, cin, cout, k, stride, dil, _ = row
        x, dy, w = _case(row, 4, (30, 40), 5)
        x = x.contiguous(memory_format=torch.channels_last).requires_grad_()
        w = w.requires_grad_()
        y = pc.conv2d_train(x, w, stride, dil, cg.dgrad_channels(name, cin))
        r1 = torch.autograd.grad(y, (x, w), dy, retain_graph=True)
        r2 = torch.autograd.grad(y, (x, w), dy)
        assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1]), name


def test_function_matches_layer_reference():
    # the autograd Function end to end on a stride-2 layer, against torch's fp64 conv on the same TF32 operands
    row = cg.ROWS[4]
    name, cin, cout, k, stride, dil, _ = row
    x, dy, w = _case(row, 2, (9, 13), 6)
    w = pc.round_tf32(w)
    xl = x.contiguous(memory_format=torch.channels_last).requires_grad_()
    wl = w.clone().requires_grad_()
    y = pc.conv2d_train(xl, wl, stride, dil)
    assert y.is_contiguous(memory_format=torch.channels_last)
    gx, gw = torch.autograd.grad(y, (xl, wl), dy)
    xd, wd = x.double().requires_grad_(), w.double().requires_grad_()
    yd = torch.nn.functional.conv2d(xd, wd, stride=stride, padding=cg.pad_of(k, dil), dilation=dil)
    ya = torch.nn.functional.conv2d(xd.detach().abs(), wd.detach().abs(), stride=stride, padding=1)
    _check(y, yd.detach(), ya, "forward")
    rx, rw = torch.autograd.grad(yd, (xd, wd), dy.double())
    torch.testing.assert_close(gx.double(), rx, rtol=0, atol=1e-4 * float(rx.abs().max()))
    torch.testing.assert_close(gw.double(), rw, rtol=0, atol=1e-4 * float(rw.abs().max()))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _training_targets(b, h, w, K, seed):
    """A disc mask per image, keypoints inside the image, the vertex field and 0/1 weights: what train() feeds."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    masks = [((yy - rng.uniform(0.3, 0.7) * h) ** 2 + (xx - rng.uniform(0.3, 0.7) * w) ** 2 < (0.25 * h) ** 2)
             for _ in range(b)]
    mask = torch.from_numpy(np.stack(masks).astype(np.int64)).to(DEV)
    hc = np.concatenate([rng.uniform([0, 0], [w, h], (b, K, 2)), np.ones((b, K, 1))], 2)
    field = nu.vertex_targets(mask, torch.from_numpy(hc).to(DEV))
    return mask, field, mask[:, None].float()


def test_forward_train_against_fp64_module():
    # one training step's loss -- the reference's cross-entropy + normalised smooth-L1 torch expressions, in each
    # copy's own dtype -- and backward(): outputs, every parameter gradient and the updated running statistics
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    ref = copy.deepcopy(net).double()
    tf32 = copy.deepcopy(net)
    b, h, w = 2, 128, 160
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    mask, field, wgt = _training_targets(b, h, w, 9, 2)

    def run(m, fwd, dtype):
        seg, ver = fwd(m)(x.to(dtype))
        loss_seg = torch.nn.functional.cross_entropy(seg, mask)
        loss_ver = nu._smooth_l1_torch(ver, field.to(dtype), wgt.to(dtype), 1.0, True).mean()
        (loss_seg + loss_ver).backward()
        return seg.detach(), ver.detach()

    out_n = run(net, lambda m: m.forward_train, torch.float32)
    out_r = run(ref, lambda m: m._forward_torch, torch.float64)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        out_t = run(tf32, lambda m: m._forward_torch, torch.float32)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    rows = [("seg_pred", out_n[0], out_t[0], out_r[0]), ("ver_pred", out_n[1], out_t[1], out_r[1])]
    pn, pt, pr = dict(net.named_parameters()), dict(tf32.named_parameters()), dict(ref.named_parameters())
    rows += [(f"grad {k}", pn[k].grad, pt[k].grad, pr[k].grad) for k in pr]
    bn, bt, br = dict(net.named_buffers()), dict(tf32.named_buffers()), dict(ref.named_buffers())
    rows += [(k, bn[k], bt[k], br[k]) for k in br if "running" in k]
    # Outputs and running statistics are held to 5e-3.  The parameter gradients cannot be: with TF32 operands the
    # torch graph itself is up to 1.7e-1 from fp64 on them (printed beside ours; the deep layers' gradients follow
    # the forward's TF32 error through every BatchNorm backward), so each is held to 1.5 x torch's own error.
    bad = []
    for what, a, t, r in rows:
        e, et = _rel(a, r), _rel(t, r)
        print(f"{what}: native {e:.2e}  torch TF32 graph {et:.2e}")
        if e > (max(5e-3, 1.5 * et) if what.startswith("grad ") else 5e-3):
            bad.append((what, e, et))
    assert all(torch.equal(bn[k], br[k].to(bn[k].dtype)) for k in br if k.endswith("num_batches_tracked"))
    assert not bad, bad


def test_forward_train_single_head_gradient_and_losses():
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    b, h, w = 2, 64, 96
    x = torch.randn(b, 3, h, w, device=DEV)
    seg, ver = net.forward_train(x)
    assert seg.shape == (b, 2, h, w) and ver.shape == (b, 18, h, w)
    base = nu._one_output(seg, ver)
    assert base is not None and base.is_contiguous()
    rng = np.random.default_rng(0)
    mask = torch.from_numpy((rng.random((b, h, w)) < 0.3).astype(np.int64)).to(DEV)
    hc = np.concatenate([rng.uniform([0, 0], [w, h], (b, 9, 2)), np.ones((b, 9, 1))], 2)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, torch.from_numpy(hc).to(DEV),
                                                                 mask[:, None].float())
    loss = ls.mean() + lv.mean()
    node = loss.grad_fn
    seen, stack = set(), [node]
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        assert "SliceBackward" not in type(n).__name__, "the head gradient goes through a slice"
        stack += [f for f, _ in n.next_functions]
    loss.backward()
    for name, p in net.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), name


def test_forward_train_rejects_image_with_grad():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    x = torch.randn(1, 3, 64, 64, device=DEV, requires_grad=True)
    with pytest.raises(ValueError):
        net.forward_train(x)
