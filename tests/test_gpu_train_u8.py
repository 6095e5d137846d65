"""The compact training input on the H100 (DESIGN.md §18): the stem pack (pvnet_stem_s2d_nhwc) of a uint8 image against
torch's normalisation and of a float image against the image itself, a forward_train(uint8, mean, std) step against the
float path bit for bit, the losses with
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


def _stem(x, w4, img, co):
    """pvnet_stem_s2d_nhwc of a uint8 [b,H,W,3] image (ImageNet constants) or a float [b,3,H,W] one -> (S, out);
    img [b,H,W,cs] gets the image and pad channels at co."""
    is_u8 = x.dtype == torch.uint8
    b, H, W = (x.shape[0], *x.shape[1:3]) if is_u8 else (x.shape[0], *x.shape[2:])
    s2d = torch.full((b, H // 2, W // 2, 16), float("nan"), device=DEV)
    out = torch.empty(b, H // 2, W // 2, 64, device=DEV)
    mean3, std3 = pc.norm3(IMAGENET_MEAN, IMAGENET_STD) if is_u8 else (None, None)
    _native.check(_native.lib().pvnet_stem_s2d_nhwc(
        x.data_ptr(), int(is_u8), mean3, std3, w4.data_ptr(), torch.zeros(64, device=DEV).data_ptr(), s2d.data_ptr(),
        out.data_ptr(), img.data_ptr(), img.shape[3], co, b, H, W,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "pvnet_stem_s2d_nhwc")
    return s2d, out


def _s2d(x):
    """The space-to-depth image of a float [b,3,H,W] image, TF32-rounded: what the pack writes as S."""
    b, _, H, W = x.shape
    xr = pc.round_tf32(x)
    want = torch.zeros(b, H // 2, W // 2, 16, device=DEV)
    for py in range(2):
        for px in range(2):
            ch = (py * 2 + px) * 3
            want[..., ch:ch + 3] = xr[:, :, py::2, px::2].permute(0, 2, 3, 1)
    return want


@pytest.mark.parametrize("b,H,W", SHAPES)
def test_uint8_pack_equals_torch_normalisation(b, H, W):
    u8 = _u8(b, H, W, H + W + b)
    w = 0.1 * torch.randn(64, 3, 7, 7, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    w4 = pc.pack_stem_s2d_train(w)
    img = torch.full((b, H, W, 40), float("nan"), device=DEV)
    s2d, out = _stem(u8, w4, img, 32)
    x = _normalised(u8)
    assert torch.equal(s2d, _s2d(x))
    assert torch.equal(img[..., 32:35], x.permute(0, 2, 3, 1))               # unrounded, as the float path's cat
    pad = img[..., 35:40]
    assert torch.equal(pad, torch.zeros_like(pad)) and not torch.signbit(pad).any()
    assert torch.isnan(img[..., :32]).all()                                     # the decoder's channels untouched
    # the float stem on the normalised image: the same S, convolution and image slice (bits, NaNs included)
    img_f = torch.full_like(img, float("nan"))
    s2d_f, out_f = _stem(x, w4, img_f, 32)
    assert torch.equal(s2d_f, s2d) and torch.equal(out_f, out)
    assert torch.equal(img_f.view(torch.int32), img.view(torch.int32))
    if b * H * W <= 3 * 72 * 104:                                               # the numpy restatement, and the CPU
        S, buf = pack_u8(u8.cpu().numpy(), IMAGENET_MEAN, IMAGENET_STD, np.full((b, H, W, 40), np.nan, np.float32),
                         32)
        assert S.tobytes() == s2d.cpu().numpy().tobytes()
        assert buf[..., 32:].tobytes() == img[..., 32:].cpu().numpy().tobytes()


@pytest.mark.parametrize("b,H,W", SHAPES)
def test_float_pack_writes_the_image_unrounded(b, H, W):
    # the float stem's image slice is the image itself, bit for bit (a negative zero and values that S rounds
    # included), then 5 zeros with no sign bit; every other channel is left as it was
    g = torch.Generator(device=DEV).manual_seed(H + W + b + 1)
    x = torch.randn(b, 3, H, W, device=DEV, generator=g)
    x.view(-1)[:3] = torch.tensor([-0.0, 1.0 + 2.0 ** -20, -(1.0 + 2.0 ** -11)], device=DEV)
    w4 = pc.pack_stem_s2d_train(0.1 * torch.randn(64, 3, 7, 7, device=DEV, generator=g))
    img = torch.full((b, H, W, 48), float("nan"), device=DEV)
    s2d, out = _stem(x, w4, img, 36)
    assert torch.equal(s2d, _s2d(x))
    bits = lambda t: t.contiguous().view(torch.int32)  # noqa: E731
    assert torch.equal(bits(img[..., 36:39]), bits(x.permute(0, 2, 3, 1)))
    pad = img[..., 39:44]
    assert torch.equal(pad, torch.zeros_like(pad)) and not torch.signbit(pad).any()
    assert torch.isnan(img[..., :36]).all() and torch.isnan(img[..., 44:]).all()
    # the convolution is the one the eval path runs on S
    want = torch.empty_like(out)
    pc.conv2d_nhwc(s2d, 0, 16, w4, torch.zeros(64, device=DEV), want, 0, 64, 4)
    assert torch.equal(out, want)


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


def test_forward_train_uint8_graph_is_the_float_graph():
    # both inputs run one stem Function and one upsampling Function: no float image, no image copy and no cat for
    # convraw.0's input on either path
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    u8 = _u8(1, 64, 96, 0)
    names = _node_names(net.forward_train(u8, mean=IMAGENET_MEAN, std=IMAGENET_STD)[0])
    assert names.count("StemS2dNHWCBackward") == 1 and names.count("Upsample2xCatNHWCBackward") == 3
    assert names.count("CatBackward0") == 1                                     # conv8s's cat[xfc, x8s] only
    assert sorted(names) == sorted(_node_names(net.forward_train(_normalised(u8))[0]))


def test_bad_arguments_return_invalid_for_both_image_forms():
    L = _native.lib()
    u8 = torch.zeros(2 * 8 * 8 * 3 + 2, dtype=torch.uint8, device=DEV)
    f = torch.zeros(1 << 16, device=DEV)
    mean3, std3 = pc.norm3(IMAGENET_MEAN, IMAGENET_STD)
    _, zero3 = pc.norm3(IMAGENET_MEAN, [0.2, 0.0, 0.2])
    p = f.data_ptr()

    def call(img=u8.data_ptr(), is_u8=1, m=mean3, s=std3, w4=p, out=p, buf=p, cs=40, co=32, b=2, H=8, W=8):
        return L.pvnet_stem_s2d_nhwc(img, is_u8, m, s, w4, p, p, out, buf, cs, co, b, H, W, None)
    flt = dict(img=p, is_u8=0, m=None, s=None)
    cases = [
        (dict(img=None), b"null"), (dict(buf=None), b"null"), (dict(b=0), b"positive"),
        (dict(W=7), b"even"), (dict(H=9), b"even"), (dict(img=u8.data_ptr() + 1), b"aligned"),
        (dict(out=p + 4), b"aligned"), (dict(co=30), b"multiples of 4"), (dict(co=36), b"channel stride"),
        (dict(cs=38, co=28), b"multiples of 4"), (dict(s=zero3), b"std"), (dict(m=None), b"mean"),
        # a float image: mean and std NULL, 8-byte aligned, and the same checks of the image slice
        (dict(flt, s=std3), b"NULL"), (dict(flt, img=p + 4), b"aligned"), (dict(flt, buf=None), b"null"),
        (dict(flt, co=36), b"channel stride"), (dict(flt, H=6, W=5), b"even"),
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
