"""The stem, max-pool and head of Resnet18_8s.forward_train on the H100: pvnet_stem_s2d_nhwc / pvnet_stem_s2d_wgrad
against fp64 on the operands as the tensor cores see them, pvnet_maxpool3x3s2_nhwc / _backward against torch's CUDA
max-pool, pvnet_head1x1_nchw / _backward against oracle/stem_pool_head_oracle.py bit for bit, and forward_train's
graph and a training step without cuDNN."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_weight

from oracle import stem_pool_head_oracle as so
from pvnet_b200 import _native
from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _check(got, ref, absref, what):
    err = (got.double() - ref).abs()
    worst = float((err - 1e-5 * absref).max().detach())
    assert worst <= 0, f"{what}: max |got-ref| {float(err.max()):.3e}, exceeds 1e-5 R by {worst:.3e}"


# ----------------------------------------------------------------------------- stem
# 16400 x 8 x 8: b*H/2 = 65600 rows, more than one launch of the space-to-depth pack
@pytest.mark.parametrize("b,H,W", [(16, 480, 640), (1, 6, 10), (2, 34, 50), (16400, 8, 8)])
def test_stem_forward_and_weight_gradient_against_fp64(b, H, W):
    g = torch.Generator(device=DEV).manual_seed(H + W + b)
    x = torch.randn(b, 3, H, W, device=DEV, generator=g)
    w = (0.1 * torch.randn(64, 3, 7, 7, device=DEV, generator=g)).requires_grad_()
    y = pc.stem_train(x, w)
    assert y.shape == (b, 64, H // 2, W // 2) and y.is_contiguous(memory_format=torch.channels_last)
    xq, wq = pc.round_tf32(x).double(), pc.round_tf32(w.detach()).double()
    ref = F.conv2d(xq, wq, stride=2, padding=3)
    _check(y, ref, F.conv2d(xq.abs(), wq.abs(), stride=2, padding=3), "stem forward")
    del ref
    dy = torch.randn(b, 64, H // 2, W // 2, device=DEV, generator=g)
    (dw,) = torch.autograd.grad(y, w, dy)
    dq = _trunc_tf32(dy).double()
    ref = conv2d_weight(xq, (64, 3, 7, 7), dq, stride=2, padding=3)
    _check(dw, ref, conv2d_weight(xq.abs(), (64, 3, 7, 7), dq.abs(), stride=2, padding=3), "stem wgrad")


def test_stem_weight_gradient_run_to_run_and_frozen():
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(4, 3, 96, 128, device=DEV, generator=g)
    w = torch.randn(64, 3, 7, 7, device=DEV, generator=g).requires_grad_()
    y = pc.stem_train(x, w)
    dy = torch.randn_like(y)
    r1 = torch.autograd.grad(y, w, dy, retain_graph=True)[0]
    r2 = torch.autograd.grad(y, w, dy)[0]
    assert torch.equal(r1, r2)
    with pytest.raises(ValueError):
        pc.stem_train(x.requires_grad_(), w)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    net.resnet18_8s.conv1.weight.requires_grad_(False)
    seg, ver = net.forward_train(torch.randn(1, 3, 64, 96, device=DEV))
    (seg.sum() + ver.square().mean()).backward()
    assert net.resnet18_8s.conv1.weight.grad is None
    assert net.resnet18_8s.bn1.weight.grad is not None


def test_stem_and_wgrad_bad_arguments_return_a_status():
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_stem_s2d_wgrad_workspace_bytes(2, 7, 8, ctypes.byref(n)) == -1
    assert b"even" in L.pvnet_last_error()
    mean3 = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    for is_u8, m in ((0, None), (1, mean3)):            # a float image, a uint8 image
        assert L.pvnet_stem_s2d_nhwc(None, is_u8, m, m, None, None, None, None, None, 8, 0, 1, 8, 8, None) == -1
        assert b"null" in L.pvnet_last_error()


# ----------------------------------------------------------------------------- max-pool
def _pool_input(kind, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "relu":
        x = torch.relu(torch.randn(4, 64, 60, 80, device=DEV, generator=g))
    elif kind == "coarse":
        x = torch.randint(-2, 3, (2, 8, 14, 18), device=DEV, generator=g).float()
    elif kind == "ninf":
        x = torch.randn(2, 8, 12, 16, device=DEV, generator=g)
        x[:, :, :3, :3] = -float("inf")
        x[:, :4, 5:8, 7:10] = -float("inf")
    else:
        x = torch.randn(2, 8, 12, 16, device=DEV, generator=g)
        x.view(-1)[torch.randint(0, x.numel(), (60,), device=DEV, generator=g)] = float("nan")
    return x.contiguous(memory_format=torch.channels_last)


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("kind", ["relu", "coarse", "ninf", "nan"])
def test_maxpool_forward_and_backward_equal_torch(kind):
    x = _pool_input(kind).requires_grad_()
    y = pc.maxpool_train(x)
    ref, ind = F.max_pool2d(x, 3, 2, 1, return_indices=True)
    assert y.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(_bits(y), _bits(ref))
    g = torch.randn(ref.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    # A window with no winner (all -inf): torch's CPU kernel and this one take its first in-image element as the
    # argmax (tests/test_stem_pool_head_cpu.py); torch's CUDA channels_last kernel records another index, so those
    # windows' gradients are left out of the comparison.
    empty = ref.detach() == -float("inf")
    if empty.any():
        print(f"torch CUDA channels_last argmax of an all -inf window: {int(ind[empty][0])}")
        g = g.masked_fill(empty, 0.0)
    (gx,) = torch.autograd.grad(y, x, g)
    (rx,) = torch.autograd.grad(ref, x, g)
    assert torch.equal(_bits(gx), _bits(rx))


@pytest.mark.parametrize("kind", ["relu", "ninf", "nan"])
def test_maxpool_codes_are_uint8_and_match_the_oracle(kind):
    x = _pool_input(kind, 1)
    b, C, H, W = x.shape
    xh = x.permute(0, 2, 3, 1)
    out = torch.empty(b, H // 2, W // 2, C, device=DEV)
    code = torch.empty(b, H // 2, W // 2, C, dtype=torch.uint8, device=DEV)
    _native.check(_native.lib().pvnet_maxpool3x3s2_nhwc(xh.data_ptr(), out.data_ptr(), code.data_ptr(), b, H, W, C,
                                                        None), "maxpool")
    g = torch.randn(out.shape, device=DEV)
    din = torch.empty_like(xh.contiguous())
    _native.check(_native.lib().pvnet_maxpool3x3s2_backward_nhwc(g.data_ptr(), code.data_ptr(), din.data_ptr(), b, H,
                                                                 W, C, None), "maxpool backward")
    torch.cuda.synchronize()
    ro, rc = so.maxpool_forward(xh.cpu().numpy())
    assert code.dtype == torch.uint8 and np.array_equal(code.cpu().numpy(), rc)
    assert np.array_equal(out.cpu().numpy().view(np.int32), ro.view(np.int32))
    assert np.array_equal(din.cpu().numpy(), so.maxpool_backward(g.cpu().numpy(), rc, H, W))


# ----------------------------------------------------------------------------- head
def _head_case(cout, seed, b=2, H=37, W=61, cin=32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    y = torch.randn(b, cin, H, W, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    w = (0.2 * torch.randn(cout, cin, 1, 1, device=DEV, generator=g)).requires_grad_()
    bias = torch.randn(cout, device=DEV, generator=g).requires_grad_()
    return y.requires_grad_(), w, bias


@pytest.mark.parametrize("cout", [20, 36, 3])
@pytest.mark.parametrize("strided", [False, True])
def test_head_bit_identical_to_oracle(cout, strided):
    y, w, bias = _head_case(cout, cout)
    out = pc.head_train(y, w, bias)
    b, cin, H, W = y.shape
    assert out.shape == (b, cout, H, W) and out.is_contiguous()
    yn = y.detach().permute(0, 2, 3, 1).reshape(-1, cin).cpu().numpy()
    wn = w.detach().reshape(cout, cin).cpu().numpy()
    ref = so.head_forward(yn, wn, bias.detach().cpu().numpy())
    assert np.array_equal(out.detach().permute(0, 2, 3, 1).reshape(-1, cout).cpu().numpy(), ref)
    if strided:          # a gradient that is not NCHW-contiguous: channels_last, and a slice of a wider tensor
        gw = torch.randn(b, 2 * cout, H, W, device=DEV).contiguous(memory_format=torch.channels_last)
        gout = gw[:, ::2]
    else:
        gout = torch.randn(b, cout, H, W, device=DEV)
    r1 = torch.autograd.grad(out, (y, w, bias), gout, retain_graph=True)
    r2 = torch.autograd.grad(out, (y, w, bias), gout)
    assert all(torch.equal(p, q) for p, q in zip(r1, r2))
    gy, gwt, gb = r1
    gn = gout.permute(0, 2, 3, 1).reshape(-1, cout).cpu().numpy()
    assert np.array_equal(gy.permute(0, 2, 3, 1).reshape(-1, cin).cpu().numpy(), so.head_dy(gn, wn))
    dw, db = so.head_param_sums(gn, yn)
    assert np.array_equal(gwt.reshape(cout, cin).cpu().numpy(), dw) and np.array_equal(gb.cpu().numpy(), db)
    exact_w = gn.astype(np.float64).T @ yn.astype(np.float64)
    exact_b = gn.astype(np.float64).sum(0)
    for got, exact in ((dw, exact_w), (db, exact_b)):
        ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
        assert (np.abs(got.astype(np.float64) - exact) <= ulp).all()


def test_head_skips_parameter_gradients_when_frozen():
    y, w, bias = _head_case(20, 1)
    w.requires_grad_(False)
    bias.requires_grad_(False)
    out = pc.head_train(y, w, bias)
    gout = torch.randn_like(out)
    (gy,) = torch.autograd.grad(out, y, gout)
    b, cin, H, W = y.shape
    gn = gout.permute(0, 2, 3, 1).reshape(-1, 20).cpu().numpy()
    ref = so.head_dy(gn, w.reshape(20, cin).cpu().numpy())
    assert np.array_equal(gy.permute(0, 2, 3, 1).reshape(-1, cin).cpu().numpy(), ref)


def test_cuda_graph_capture_and_replay():
    # the three Functions, forward and backward, captured in one CUDA graph and replayed on new inputs: bit for bit the
    # eager calls (nothing in them synchronises the stream or copies from the host)
    g = torch.Generator(device=DEV).manual_seed(21)
    xs = torch.randn(2, 3, 64, 96, device=DEV, generator=g)
    w1 = torch.randn(64, 3, 7, 7, device=DEV, generator=g).requires_grad_()
    ys = torch.randn(2, 32, 64, 96, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    wh = torch.randn(20, 32, 1, 1, device=DEV, generator=g).requires_grad_()
    bh = torch.randn(20, device=DEV, generator=g).requires_grad_()
    gs = torch.randn(2, 20, 64, 96, device=DEV, generator=g)

    def step():
        s = pc.stem_train(xs, w1)
        p = pc.maxpool_train(torch.relu(s))
        y = ys.detach().requires_grad_()
        h = pc.head_train(y, wh, bh)
        return (s, p, h) + torch.autograd.grad((p.sum(), h), (w1, y, wh, bh), (None, gs))
    # warm-up, capture and the eager reference all on one side stream (the leaves' gradient nodes keep their stream)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    side.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        outs = step()
    for seed in (22, 23):
        gg = torch.Generator(device=DEV).manual_seed(seed)
        xs.copy_(torch.randn(xs.shape, device=DEV, generator=gg))
        ys.copy_(torch.randn(ys.shape, device=DEV, generator=gg))
        gs.copy_(torch.randn(gs.shape, device=DEV, generator=gg))
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in outs]
        with torch.cuda.stream(side):
            eager = step()
        side.synchronize()
        for u, v in zip(got, eager):
            assert torch.equal(u, v)


def test_forward_train_step_does_not_synchronise():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    x = torch.randn(2, 3, 64, 96, device=DEV)
    seg, ver = net.forward_train(x)                  # first call: one-time setup (kernel attributes)
    (seg.sum() + ver.square().mean()).backward()
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        seg, ver = net.forward_train(x)
        (seg.sum() + ver.square().mean()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert torch.isfinite(net.resnet18_8s.conv1.weight.grad).all()


# ----------------------------------------------------------------------------- forward_train
def _node_names(t):
    names, seen, stack = [], set(), [t.grad_fn]
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        names.append(type(n).__name__)
        stack += [f for f, _ in n.next_functions]
    return names


def test_forward_train_graph_has_no_torch_layers():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    seg, _ = net.forward_train(torch.randn(1, 3, 64, 96, device=DEV))
    names = _node_names(seg)
    for bad in ("ConvolutionBackward0", "CudnnConvolutionBackward0", "MaxPool2DWithIndicesBackward0", "CloneBackward0"):
        assert bad not in names, bad
    for one in ("StemS2dNHWCBackward", "MaxPool3x3s2NHWCBackward", "Head1x1NCHWBackward"):
        assert names.count(one) == 1, one
    assert names.count("BatchNormActNHWCBackward") == 14 and names.count("BatchNormAddReluNHWCBackward") == 8
    assert names.count("Upsample2xCatNHWCBackward") == 3 and names.count("CatBackward0") == 1


def test_forward_train_rejects_other_module_shapes():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    x = torch.randn(1, 3, 64, 64, device=DEV)
    for attr, mod in (("maxpool", torch.nn.MaxPool2d(3, 2, 1, ceil_mode=True)),
                      ("conv1", torch.nn.Conv2d(3, 64, 7, 2, 3, bias=True))):
        m = copy.deepcopy(net).to(DEV)
        setattr(m.resnet18_8s, attr, mod.to(DEV))
        with pytest.raises(ValueError):
            m.forward_train(x)
    m = copy.deepcopy(net)
    m.convraw[3] = torch.nn.Conv2d(32, 20, 1, 1, bias=False).to(DEV)
    with pytest.raises(ValueError):
        m.forward_train(x)


def _step(net, x, mask, hc, wgt):
    seg, ver = net.forward_train(x)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
    (ls.mean() + lv.mean()).backward()
    return seg.detach(), ver.detach()


def test_step_without_cudnn_is_identical():
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    twin = copy.deepcopy(net)
    b, h, w = 2, 128, 160
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    rng = np.random.default_rng(0)
    mask = torch.from_numpy((rng.random((b, h, w)) < 0.3).astype(np.int64)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [w, h], (b, 9, 2)), np.ones((b, 9, 1))], 2)).to(DEV)
    wgt = mask[:, None].float()
    out_a = _step(net, x, mask, hc, wgt)
    with torch.backends.cudnn.flags(enabled=False):
        out_b = _step(twin, x, mask, hc, wgt)
    assert all(torch.equal(p, q) for p, q in zip(out_a, out_b))
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k
