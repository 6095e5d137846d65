"""The compact training input on the H100 (DESIGN.md §18): the uint8 stem pack (pvnet_stem_s2d_u8_nhwc) against
torch's normalisation, a forward_train(uint8, mean, std) step against the float path bit for bit, the losses with
vertex_weights=None against the loader's mask.unsqueeze(1).float(), CUDA-graph replay, no synchronisation,
deterministic mode, and the C ABI's refusals."""
import copy
import ctypes

import numpy as np
import pytest
import torch

from pvnet_b200 import _native
from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s
from tests.train_u8_oracle import IMAGENET_MEAN, IMAGENET_STD, pack_u8

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# 1100 x 120 x 8: b*H/2 = 66000 rows, more than one launch of the pack (its grid.y is limited to 65535).  A whole step
# at that shape is out of reach for the float path too: the decoder's upsampling launches b*h rows of blocks
# (pvnet_upsample2x_nhwc, 66000 for up2storaw), so the step cases stop at the first three and the chunked pack is
# compared with the float path's stem (S, its convolution and convraw.0's image channels) on its own.
SHAPES = [(2, 480, 640), (3, 72, 104), (4, 8, 8), (1100, 120, 8)]
STEP_SHAPES = SHAPES[:3]


def _u8(b, H, W, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, 256, (b, H, W, 3), dtype=torch.uint8, device=DEV, generator=g)


def _normalised(u8):
    """torch's own ToTensor + Normalize on CUDA, with 255 as a CUDA tensor so that torch runs a tensor division, the
    operation the loader's ToTensor runs on the CPU (ATen may turn a division by a Python scalar into a multiplication
    by its reciprocal, which differs in the last bit for some bytes)."""
    mean = torch.tensor(IMAGENET_MEAN, device=DEV).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD, device=DEV).view(1, 3, 1, 1)
    x = u8.permute(0, 3, 1, 2).float().div(torch.tensor(255.0, device=DEV))
    return x.sub(mean).div(std).contiguous()


def _stem_u8(u8, w4, img, co):
    b, H, W, _ = u8.shape
    s2d = torch.full((b, H // 2, W // 2, 16), float("nan"), device=DEV)
    out = torch.empty(b, H // 2, W // 2, 64, device=DEV)
    mean3, std3 = pc.norm3(IMAGENET_MEAN, IMAGENET_STD)
    _native.check(_native.lib().pvnet_stem_s2d_u8_nhwc(
        u8.data_ptr(), mean3, std3, w4.data_ptr(), torch.zeros(64, device=DEV).data_ptr(), s2d.data_ptr(),
        out.data_ptr(), img.data_ptr(), img.shape[3], co, b, H, W,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pvnet_stem_s2d_u8_nhwc")
    return s2d, out


@pytest.mark.parametrize("b,H,W", SHAPES)
def test_pack_equals_torch_normalisation(b, H, W):
    u8 = _u8(b, H, W, H + W + b)
    w = 0.1 * torch.randn(64, 3, 7, 7, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    w4 = pc.pack_stem_s2d_train(w)
    img = torch.full((b, H, W, 40), float("nan"), device=DEV)
    s2d, out = _stem_u8(u8, w4, img, 32)
    x = _normalised(u8)
    xr = pc.round_tf32(x)
    want_s = torch.zeros(b, H // 2, W // 2, 16, device=DEV)
    for py in range(2):
        for px in range(2):
            ch = (py * 2 + px) * 3
            want_s[..., ch:ch + 3] = xr[:, :, py::2, px::2].permute(0, 2, 3, 1)
    assert torch.equal(s2d, want_s)
    assert torch.equal(img[..., 32:35], x.permute(0, 2, 3, 1))               # unrounded, as the float path's cat
    pad = img[..., 35:40]
    assert torch.equal(pad, torch.zeros_like(pad)) and not torch.signbit(pad).any()
    assert torch.isnan(img[..., :32]).all()                                     # the decoder's channels untouched
    # the convolution: the float path's stem on the normalised image
    s2d_f = torch.empty_like(s2d)
    out_f = torch.empty_like(out)
    _native.check(_native.lib().pvnet_stem_s2d_nhwc(
        x.data_ptr(), w4.data_ptr(), torch.zeros(64, device=DEV).data_ptr(), s2d_f.data_ptr(), out_f.data_ptr(), b,
        H, W, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pvnet_stem_s2d_nhwc")
    assert torch.equal(s2d_f, s2d) and torch.equal(out_f, out)
    if b * H * W <= 3 * 72 * 104:                                               # the numpy restatement, and the CPU
        S, buf = pack_u8(u8.cpu().numpy(), IMAGENET_MEAN, IMAGENET_STD, np.full((b, H, W, 40), np.nan, np.float32),
                         32)
        assert S.tobytes() == s2d.cpu().numpy().tobytes()
        assert buf[..., 32:].tobytes() == img[..., 32:].cpu().numpy().tobytes()


def _batch(b, H, W, seed):
    rng = np.random.default_rng(seed)
    mask = torch.from_numpy((rng.random((b, H, W)) < 0.3).astype(np.int64)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [W, H], (b, 9, 2)), np.ones((b, 9, 1))], 2)).to(DEV)
    return _u8(b, H, W, seed), mask, hc


def _step(net, x, mask, hc, wgt, **kw):
    seg, ver = net.forward_train(x, **kw)
    ls, lv, pr, rc = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
    (ls.mean() + lv.mean()).backward()
    return [seg.detach(), ver.detach(), ls.detach(), lv.detach(), pr, rc]


def _assert_same_state(net, twin):
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k


@pytest.mark.parametrize("b,H,W", STEP_SHAPES)
def test_uint8_step_equals_the_float_step(b, H, W):
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    twin = copy.deepcopy(net)
    u8, mask, hc = _batch(b, H, W, b + H)
    got = _step(net, u8, mask, hc, None, mean=IMAGENET_MEAN, std=IMAGENET_STD)       # the compact form
    want = _step(twin, _normalised(u8), mask, hc, mask.unsqueeze(1).float())         # the loader's form
    for i, (u, v) in enumerate(zip(got, want)):
        assert torch.equal(u, v), i
    _assert_same_state(net, twin)
    assert int(net.resnet18_8s.bn1.num_batches_tracked) == 1


def _loss_case(dtype, b, h, w, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    K = 4
    seg = torch.randn(b, 3, h, w, device=DEV, generator=g)                    # three classes: a value 2 is valid
    ver = torch.randn(b, 2 * K, h, w, device=DEV, generator=g)
    m = torch.randint(0, 2, (b, h, w), device=DEV, generator=g)
    m[0, 1, :5] = 2                                                            # weighs 2, and is no keypoint pixel
    mask = (m > 0) if dtype == torch.bool else m.to(dtype)
    field = torch.randn(b, 2 * K, h, w, device=DEV, generator=g)
    hc = torch.cat([torch.rand(b, K, 2, device=DEV, generator=g) * torch.tensor([w, h], device=DEV),
                    torch.ones(b, K, 1, device=DEV)], 2).double()
    return seg, ver, mask, field, hc


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
@pytest.mark.parametrize("h,w", [(64, 96), (37, 53)])
def test_losses_with_none_weights_equal_the_mask_weights(dtype, h, w):
    seg, ver, mask, field, hc = _loss_case(dtype, 3, h, w, h + w)
    wm = mask.unsqueeze(1).float()
    with torch.no_grad():
        for fn, tgt in ((nu.seg_vertex_losses, field), (nu.seg_vertex_losses_from_keypoints, hc)):
            for u, v in zip(fn(seg, ver, mask, tgt, None), fn(seg, ver, mask, tgt, wm)):
                assert torch.equal(u, v), fn.__name__
    for fn, tgt in ((nu.seg_vertex_training_losses, field), (nu.seg_vertex_training_losses_from_keypoints, hc)):
        res = []
        for wgt in (None, wm):
            s, v = seg.clone().requires_grad_(), ver.clone().requires_grad_()
            out = fn(s, v, mask, tgt, wgt)
            gs, gv = torch.rand(2, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
            res.append(list(out) + list(torch.autograd.grad((out[0], out[1]), (s, v), (gs, gv))))
        for i, (u, v) in enumerate(zip(*res)):
            assert torch.equal(u, v), (fn.__name__, i)
    # one output tensor (forward_train's form): the gradient is written once, with the mask's weights as well
    base = torch.cat([seg, ver], 1).requires_grad_()
    res = []
    for wgt in (None, wm):
        out = nu.seg_vertex_training_losses_from_keypoints(base[:, :3], base[:, 3:], mask, hc, wgt)
        res.append(list(out) + [torch.autograd.grad(out[0].sum() + out[1].sum(), base)[0]])
    for u, v in zip(*res):
        assert torch.equal(u, v)


def test_cuda_graph_capture_and_replay_of_a_uint8_step():
    torch.manual_seed(1)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    params = [p for p in net.parameters()]
    b, H, W = 2, 64, 96
    u8, mask, hc = _batch(b, H, W, 3)

    def step():
        seg, ver = net.forward_train(u8, mean=IMAGENET_MEAN, std=IMAGENET_STD)
        ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
        return [seg.detach(), ver.detach(), ls.detach(), lv.detach()] + \
            list(torch.autograd.grad(ls.mean() + lv.mean(), params))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    side.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        outs = step()
    for seed in (4, 5):
        u2, m2, h2 = _batch(b, H, W, seed)
        u8.copy_(u2)
        mask.copy_(m2)
        hc.copy_(h2)
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in outs]
        with torch.cuda.stream(side):
            eager = step()
        side.synchronize()
        for i, (u, v) in enumerate(zip(got, eager)):
            assert torch.equal(u, v), i


def test_uint8_step_does_not_synchronise_and_is_deterministic():
    torch.manual_seed(2)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    twin = copy.deepcopy(net)
    u8, mask, hc = _batch(2, 64, 96, 6)
    kw = dict(mean=IMAGENET_MEAN, std=IMAGENET_STD)
    _step(copy.deepcopy(net), u8, mask, hc, None, **kw)                         # one-time setup (kernel attributes)
    probe = copy.deepcopy(net)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _step(probe, u8, mask, hc, None, **kw)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = _step(net, u8, mask, hc, None, **kw)
        bb = _step(twin, u8, mask, hc, None, **kw)
    finally:
        torch.use_deterministic_algorithms(prev)
    for u, v in zip(a, bb):
        assert torch.equal(u, v)
    _assert_same_state(net, twin)


def test_forward_train_uint8_graph_has_no_float_image_or_cat():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    seg, _ = net.forward_train(_u8(1, 64, 96, 0), mean=IMAGENET_MEAN, std=IMAGENET_STD)
    names, seen, stack = [], set(), [seg.grad_fn]
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        names.append(type(n).__name__)
        stack += [f for f, _ in n.next_functions]
    assert names.count("StemS2dU8NHWCBackward") == 1 and "StemS2dNHWCBackward" not in names
    assert names.count("Upsample2xIntoNHWCBackward") == 1 and names.count("Upsample2xCatNHWCBackward") == 2
    assert names.count("CatBackward0") == 1                                     # conv8s's cat[xfc, x8s] only


def test_bad_arguments_return_invalid():
    L = _native.lib()
    u8 = torch.zeros(2 * 8 * 8 * 3 + 2, dtype=torch.uint8, device=DEV)
    f = torch.zeros(1 << 16, device=DEV)
    mean3, std3 = pc.norm3(IMAGENET_MEAN, IMAGENET_STD)
    _, zero3 = pc.norm3(IMAGENET_MEAN, [0.2, 0.0, 0.2])
    p = f.data_ptr()

    def call(img=u8.data_ptr(), m=mean3, s=std3, w4=p, out=p, buf=p, cs=40, co=32, b=2, H=8, W=8):
        return L.pvnet_stem_s2d_u8_nhwc(img, m, s, w4, p, p, out, buf, cs, co, b, H, W, None)
    cases = [
        (dict(img=None), b"null"), (dict(buf=None), b"null"), (dict(b=0), b"positive"),
        (dict(W=7), b"even"), (dict(H=9), b"even"), (dict(img=u8.data_ptr() + 1), b"aligned"),
        (dict(out=p + 4), b"aligned"), (dict(co=30), b"multiples of 4"), (dict(co=36), b"channel stride"),
        (dict(cs=38, co=28), b"multiples of 4"), (dict(s=zero3), b"std"),
    ]
    for kw, text in cases:
        assert call(**kw) == -1, kw
        assert text in L.pvnet_last_error(), (kw, L.pvnet_last_error())
    # the losses: a NULL vertex_weights with strides is refused as before (both NULL take the weights from the mask)
    s4 = (ctypes.c_int64 * 4)(20 * 64, 64, 8, 1)
    s3 = (ctypes.c_int64 * 3)(64, 8, 1)
    rc = L.pvnet_seg_vertex_losses(p, s4, p, 8, s3, p, s4, p, s4, None, s4, 2, 8, 8, 2, 18, 1.0, 1, p, p, p, p, p,
                                   1 << 20, None)
    assert rc == -1 and b"null" in L.pvnet_last_error()
