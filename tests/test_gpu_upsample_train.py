"""Bilinear x2 upsampling for training on the H100: pvnet_upsample2x_nhwc (bit for bit torch's CUDA forward on a
channels_last tensor), pvnet_upsample2x_backward_nhwc (ATen's terms in a fixed order, checked bit for bit against
oracle/upsample_oracle.py and against torch's atomic backward within the reordering bound), the Upsample2xCatNHWC
autograd Function, and a deterministic Resnet18_8s.forward_train step under torch.use_deterministic_algorithms(True)."""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import upsample_oracle as uo
from pvnet_b200 import _native
from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STAGES = [(2, 128, 60, 80), (2, 64, 120, 160), (2, 32, 240, 320)]
ODD = [(1, 16, 1, 1), (2, 16, 3, 7), (1, 32, 13, 9)]


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _forward(x, out, co):
    """x [b,h,w,C] dense NHWC -> out [b,2h,2w,cs] at channel co."""
    b, h, w, C = x.shape
    _native.check(_native.lib().pvnet_upsample2x_nhwc(ctypes.c_void_p(x.data_ptr()), C, ctypes.c_void_p(out.data_ptr()),
                                                      out.shape[3], co, b, h, w, _stream()), "pvnet_upsample2x_nhwc")


def _backward(dy, co, C):
    """dy [b,2h,2w,cs] read at channels [co, co+C) -> dX [b,h,w,C]."""
    b, H, W, cs = dy.shape
    dx = torch.full((b, H // 2, W // 2, C), float("nan"), device=DEV)
    _native.check(_native.lib().pvnet_upsample2x_backward_nhwc(ctypes.c_void_p(dy.data_ptr()), cs, co, C,
                                                               ctypes.c_void_p(dx.data_ptr()), b, H // 2, W // 2,
                                                               _stream()), "pvnet_upsample2x_backward_nhwc")
    return dx


def _torch_up(t):
    return F.interpolate(t, scale_factor=2, mode="bilinear", align_corners=True)


@pytest.mark.parametrize("b,C,h,w", STAGES + ODD)
def test_forward_bit_identical_to_torch(b, C, h, w):
    g = torch.Generator(device=DEV).manual_seed(C * 1000 + h)
    x = torch.randn(b, C, h, w, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    ref = _torch_up(x).permute(0, 2, 3, 1)
    out = torch.full((b, 2 * h, 2 * w, C + 8), float("nan"), device=DEV)
    _forward(x.permute(0, 2, 3, 1), out, 4)
    torch.cuda.synchronize()
    assert torch.equal(out[..., 4:4 + C], ref)
    assert torch.isnan(out[..., :4]).all() and torch.isnan(out[..., 4 + C:]).all(), "neighbouring channels written"


@pytest.mark.parametrize("b,C,h,w", ODD + [(1, 4, 2, 5), (2, 4, 15, 20), (1, 8, 4, 1)])
def test_backward_equals_oracle(b, C, h, w):
    g = torch.Generator(device=DEV).manual_seed(C * 100 + h * 10 + w)
    buf = torch.randn(b, 2 * h, 2 * w, C + 12, device=DEV, generator=g)
    dx = _backward(buf, 8, C)
    ref = uo.upsample2x_backward(buf[..., 8:8 + C].cpu().numpy())
    assert np.array_equal(dx.cpu().numpy().view(np.int32), ref.view(np.int32))


@pytest.mark.parametrize("b,C,h,w", STAGES + ODD)
def test_backward_within_reordering_of_torch(b, C, h, w):
    """torch's backward adds the same terms with atomics in some order: each element (at most 16 terms) differs from
    ours by at most the bound on reordering its fp32 sum, 2 * 15 * 2^-24 * sum |terms|."""
    g = torch.Generator(device=DEV).manual_seed(C + h + w)
    x = torch.randn(b, C, h, w, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    x.requires_grad_()
    gy = torch.randn(b, C, 2 * h, 2 * w, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    _torch_up(x).backward(gy)
    ref = x.grad.permute(0, 2, 3, 1)
    gh = gy.permute(0, 2, 3, 1).contiguous()
    got = _backward(gh, 0, C)
    absb = _backward(gh.abs(), 0, C)
    err = (got - ref).abs()
    assert (err <= 31 * 2.0 ** -24 * absb + 1e-37).all(), float((err / absb.clamp_min(1e-30)).max())


def test_backward_run_to_run_full_resolution():
    b, C, h, w = 8, 32, 240, 320
    g = torch.Generator(device=DEV).manual_seed(5)
    dy = torch.randn(b, 2 * h, 2 * w, 40, device=DEV, generator=g)
    a = _backward(dy, 0, C)
    c = _backward(dy, 0, C)
    assert torch.equal(a, c)
    assert torch.isfinite(a).all()


def test_bad_arguments_return_a_status():
    x = torch.zeros(1, 4, 4, 8, device=DEV)
    out = torch.zeros(1, 8, 8, 8, device=DEV)
    L = _native.lib()
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)   # noqa: E731
    assert L.pvnet_upsample2x_nhwc(p(x), 6, p(out), 8, 0, 1, 4, 4, _stream()) != 0            # C not a multiple of 4
    assert L.pvnet_upsample2x_nhwc(p(x), 8, p(out), 8, 4, 1, 4, 4, _stream()) != 0            # slice past the end
    assert L.pvnet_upsample2x_nhwc(p(x, 4), 8, p(out), 8, 0, 1, 4, 4, _stream()) != 0         # misaligned
    assert L.pvnet_upsample2x_backward_nhwc(p(out), 8, 2, 4, p(x), 1, 4, 4, _stream()) != 0   # offset
    assert L.pvnet_upsample2x_backward_nhwc(None, 8, 0, 4, p(x), 1, 4, 4, _stream()) != 0
    assert L.pvnet_upsample2x_backward_nhwc(p(out), 8, 0, 4, p(x), 0, 4, 4, _stream()) != 0   # empty batch
    with pytest.raises(RuntimeError):
        _native.check(L.pvnet_upsample2x_nhwc(p(x), 6, p(out), 8, 0, 1, 4, 4, _stream()), "pvnet_upsample2x_nhwc")


def test_upsample2x_cat_values_gradients_and_node():
    g = torch.Generator(device=DEV).manual_seed(3)
    cl = torch.channels_last
    low = torch.randn(2, 32, 30, 40, device=DEV, generator=g).contiguous(memory_format=cl).requires_grad_()
    r1 = torch.randn(2, 4, 60, 80, device=DEV, generator=g).contiguous(memory_format=cl).requires_grad_()
    r2 = torch.randn(2, 8, 60, 80, device=DEV, generator=g).contiguous(memory_format=cl)
    out = pc.upsample2x_cat(low, r1, r2)
    assert type(out.grad_fn).__name__ == "Upsample2xCatNHWCBackward"
    assert out.is_contiguous(memory_format=cl) and out.shape == (2, 44, 60, 80)
    ref = torch.cat([_torch_up(low), r1, r2], 1)
    assert torch.equal(out, ref)
    gy = torch.randn(out.shape, device=DEV, generator=g).contiguous(memory_format=cl)
    out.backward(gy)
    assert torch.equal(r1.grad, gy[:, 32:36])
    assert r2.grad is None
    dlow = _backward(gy.permute(0, 2, 3, 1).contiguous(), 0, 32).permute(0, 3, 1, 2)
    assert torch.equal(low.grad, dlow)
    # a gradient that is not channels_last gives the same result
    low.grad = None
    pc.upsample2x_cat(low, r1, r2).backward(gy.contiguous())
    assert torch.equal(low.grad, dlow)


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


def test_forward_train_graph_has_no_torch_upsampling():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    seg, _ = net.forward_train(torch.randn(1, 3, 64, 96, device=DEV))
    names = _node_names(seg)
    assert not [n for n in names if "Upsample" in n and n != "Upsample2xCatNHWCBackward"]
    assert names.count("Upsample2xCatNHWCBackward") == 3
    assert names.count("CatBackward0") == 1, "only conv8s's input is a plain concatenation"


def test_forward_train_outputs_and_statistics_unchanged(monkeypatch):
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    ref = copy.deepcopy(net)
    x = torch.randn(2, 3, 128, 160, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    out_n = net.forward_train(x)
    monkeypatch.setattr(pc, "upsample2x_cat", lambda low, *rest: torch.cat([_torch_up(low), *rest], 1))
    out_t = ref.forward_train(x)
    assert torch.equal(out_n[0], out_t[0]) and torch.equal(out_n[1], out_t[1])
    bn, bt = dict(net.named_buffers()), dict(ref.named_buffers())
    for k in bn:
        assert torch.equal(bn[k], bt[k]), k


def _step(net, opt, x, mask, hc):
    opt.zero_grad()
    seg, ver = net.forward_train(x)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, mask[:, None].float())
    (ls.mean() + lv.mean()).backward()
    opt.step()


def test_deterministic_training_step():
    b, h, w, K = 2, 128, 160, 9
    torch.manual_seed(0)
    nets = [Resnet18_8s(ver_dim=2 * K, seg_dim=2).to(DEV).train()]
    nets.append(copy.deepcopy(nets[0]))
    opts = [torch.optim.Adam(n.parameters(), lr=1e-3) for n in nets]
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    rng = np.random.default_rng(2)
    mask = torch.from_numpy((rng.random((b, h, w)) < 0.3).astype(np.int64)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [w, h], (b, K, 2)), np.ones((b, K, 1))], 2)).to(DEV)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for net, opt in zip(nets, opts):
            _step(net, opt, x, mask, hc)
        torch.cuda.synchronize()
        (pa, pb) = (dict(n.named_parameters()) for n in nets)
        for k in pa:
            assert torch.equal(pa[k], pb[k]), k
            assert torch.equal(pa[k].grad, pb[k].grad), f"grad {k}"
        (ba, bb) = (dict(n.named_buffers()) for n in nets)
        for k in ba:
            assert torch.equal(ba[k], bb[k]), k
        sa, sb = opts[0].state_dict()["state"], opts[1].state_dict()["state"]
        assert sa.keys() == sb.keys() and len(sa) == len(pa)
        for i in sa:
            for k in sa[i]:
                assert torch.equal(sa[i][k], sb[i][k]), (i, k)
        # the flag does not swap the native upsampling for anything else (torch 2.11 replaces its own F.interpolate
        # by a decomposition into index and elementwise ops in this mode)
        seg, _ = nets[0].forward_train(x)
        assert _node_names(seg).count("Upsample2xCatNHWCBackward") == 3
    finally:
        torch.use_deterministic_algorithms(prev)
