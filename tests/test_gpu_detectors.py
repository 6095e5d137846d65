"""GPU: Resnet18_8s_detector and Resnet18_8s_detector_v2 on the native kernels.  The eval forward against the
reference's fp32 golden and the torch graph at 480x640 (the bound of test_gpu_deep_backbones.py: 3x cuDNN-TF32's own
deviation, floor 3e-3 of the range); the trunk stages bit for bit Resnet18_8s's; the score head, eval stage and
training kernels, against fp64 with the fp32 chain's bound, byte-identical run to run; forward_train against an fp64
module (output, every gradient, every running statistic; v2's gradients reach only what it uses); seeded steps
deterministic; uint8 input; weight updates, DataParallel, pickling and the errors."""
import copy
import ctypes
import gc
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from pvnet_b200 import _native
from pvnet_b200 import conv as pc
from pvnet_b200 import model_repository as mr
from pvnet_b200.optim import Adam
from tests.detectors import (DETECTOR_CLASSES, buffer_offsets, detector, detector_buffers, detector_golden,
                             head3x3_fp64)
from tests.helpers import seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


class _tf32:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = self.on
        torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


def _net(name, seed=1):
    return detector(name, seed).to(DEV).eval()


def _stage_names(handle):
    lib = _native.lib()
    return [lib.pvnet_backbone_handle_stage_name(handle, i).decode()
            for i in range(lib.pvnet_backbone_handle_num_stages(handle))]


def _buffer(net, bufs, i, b, h, w):
    """Buffer i of the net's workspace as [b, H>>level, W>>level, ch] float32."""
    ws = next(iter(net._nat.workspaces.values()))
    level, ch = bufs[i]
    off = buffer_offsets(bufs, b, h, w)[0][i]
    return ws[off:off + ((b * h * w) >> (2 * level)) * ch * 4].view(torch.float32).view(b, h >> level, w >> level, ch)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_native_vs_reference_golden(name):
    x, gold = detector_golden(name)
    net = _net(name)
    xd = torch.from_numpy(x).to(DEV)
    with torch.no_grad():
        got = net(xd)
        with _tf32(True):
            t = net._forward_torch(xd)
    g = torch.from_numpy(gold).to(DEV)
    e_cudnn = (t - g).abs().max().item()
    err = (got - g).abs().max().item()
    scale = g.abs().max().item()
    print(f"\n[{name} vs reference fp32 golden] max abs err {err:.3e}, range {scale:.3f}; cuDNN-TF32 {e_cudnn:.3e}")
    assert got.shape == g.shape and err <= max(3.0 * e_cudnn, 3e-3 * scale)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_native_vs_torch_graph_fullsize(name):
    net = _net(name, seed=3)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        with _tf32(False):
            r = net._forward_torch(x)
        with _tf32(True):
            t = net._forward_torch(x)
        got = net.forward_native(x)
    scale = r.abs().max().item()
    e, et = (got - r).abs().max().item(), (t - r).abs().max().item()
    print(f"\n[{name} 480x640] native {e / scale:.2e}, cuDNN-TF32 {et / scale:.2e} of the range")
    assert got.shape == (2, 1, 60, 80) and e <= max(3.0 * et, 3e-3 * scale)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_trunk_stages_are_resnet18_8s_bit_for_bit(name):
    """With the same trunk weights, the detector's plan and Resnet18_8s's leave the same bits in S, the stem's output
    and layer2's (v2) / layer4's (v1) output, which every trunk stage feeds."""
    b, h, w = 2, 64, 96
    det = _net(name, seed=4)
    r18 = mr.Resnet18_8s(18, 2)
    pre = det._prefix
    sd = seeded_state_dict(r18, seed=4)
    sd.update({"resnet18_8s." + k[len(pre):]: v for k, v in det.state_dict().items()
               if k.startswith(pre) and not k.startswith(pre + "fc")})
    r18.load_state_dict(sd)
    r18 = r18.to(DEV).eval()
    x = torch.randn(b, 3, h, w, device=DEV)
    lib = _native.lib()
    cut = len(_stage_names(det._prepare_native(torch.device(DEV)))) - 1          # every stage before the head
    for net in (det, r18):
        handle = net._prepare_native(torch.device(DEV))
        assert _stage_names(handle)[1:cut] == _stage_names(det._prepare_native(torch.device(DEV)))[1:cut]
        with torch.no_grad():
            net.run_stages(x, torch.empty(b, 20, h, w, device=DEV), None, 0, cut)
    torch.cuda.synchronize()
    dbufs = detector_buffers(det._last_stage)
    # Resnet18_8s's buffers (backbone.cu generate): S, C1, R0, C2, U2, P; layer1 A B C4 U4; layer2 A D B C8 U8;
    # layer3 A D B E; layer4 A D B E
    rbufs = [(1, 16), (0, 40), (0, 32), (1, 128), (1, 32), (2, 64), (2, 64), (2, 64), (2, 192), (2, 64),
             (3, 128), (3, 128), (3, 128), (3, 384), (3, 128)] + [(3, 256)] * 4 + [(3, 512)] * 4
    feat = _buffer(det, dbufs, len(dbufs) - 1, b, h, w)
    ref = _buffer(r18, rbufs, 13, b, h, w)[..., 256:] if det._last_stage == 2 else _buffer(r18, rbufs, 22, b, h, w)
    pairs = (("S", _buffer(det, dbufs, 0, b, h, w), _buffer(r18, rbufs, 0, b, h, w)),
             ("stem", _buffer(det, dbufs, 1, b, h, w), _buffer(r18, rbufs, 3, b, h, w)[..., 64:]),
             ("layer1", _buffer(det, dbufs, 5, b, h, w), _buffer(r18, rbufs, 8, b, h, w)[..., 128:]),
             ("last stage", feat, ref))
    for what, a, r in pairs:
        print(what, tuple(a.shape), tuple(r.shape), (a - r).abs().max().item(), r.abs().max().item())
    assert feat.abs().sum() > 0
    assert all(torch.equal(a, r) for _, a, r in pairs)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_score_stage_against_fp64(name):
    """The eval plan's head stage, from the buffer the stage before it left, against fp64 with the bound of one fp32
    fmaf chain of 9C+1 terms; two runs are byte-identical."""
    net = _net(name, seed=5)
    b, h, w = 2, 72, 104                                  # H/8 = 9, W/8 = 13
    x = torch.randn(b, 3, h, w, device=DEV)
    handle = net._prepare_native(torch.device(DEV))
    n = len(_stage_names(handle))
    outs = []
    with torch.no_grad():
        for _ in range(2):
            out = torch.full((b, 1, h // 8, w // 8), float("nan"), device=DEV)
            net.run_stages(x, out, None, 0, n)
            outs.append(out)
        torch.cuda.synchronize()
        bufs = detector_buffers(net._last_stage)
        feat = _buffer(net, bufs, len(bufs) - 1, b, h, w).permute(0, 3, 1, 2)
    hd = net.get_submodule(net._score_slot)
    ref, R = head3x3_fp64(feat, hd.weight, hd.bias)
    err = ((outs[0].double() - ref).abs() / R).max().item()
    print(f"\n{name} score stage: max |err| / R = {err:.2e}")
    assert err <= (9 * feat.shape[1] + 1) * 2.0 ** -24
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], net.forward_native(x))


@pytest.mark.parametrize("C,shape", [(512, (2, 9, 13)), (128, (3, 33, 41)), (32, (1, 8, 8))])
def test_training_head_against_fp64(C, shape):
    """pvnet_b200.conv.head3x3_train: forward, data gradient (an fmaf chain of 9 terms) and the fp64 weight and bias
    sums, against fp64; two runs are byte-identical."""
    b, H, W = shape
    g = torch.Generator(device=DEV).manual_seed(C)
    y = torch.randn(b, C, H, W, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(1, C, 3, 3, device=DEV, generator=g) * 0.05)
    bias = torch.randn(1, device=DEV, generator=g)
    gout = torch.randn(b, 1, H, W, device=DEV, generator=g)
    runs = []
    for _ in range(2):
        yy, ww, bb = (t.clone().requires_grad_() for t in (y, wt, bias))
        out = pc.head3x3_train(yy, ww, bb)
        out.backward(gout)
        runs.append((out.detach(), yy.grad, ww.grad, bb.grad))
    assert all(torch.equal(p, q) for p, q in zip(*runs))
    out, dy, dw, db = runs[0]
    ref, R = head3x3_fp64(y, wt, bias)
    assert ((out.double() - ref).abs() / R).max().item() <= (9 * C + 1) * 2.0 ** -24
    yd, wd, bd = (t.double().requires_grad_() for t in (y, wt, bias))
    F.conv2d(yd, wd, bd, padding=1).backward(gout.double())
    dyR = F.conv_transpose2d(gout.double().abs(), wt.double().abs(), padding=1)
    assert ((dy.double() - yd.grad).abs() / dyR.clamp_min(1e-30)).max().item() <= 9 * 2.0 ** -24
    dwR = F.conv2d(y.double().abs().transpose(0, 1), gout.double().abs().transpose(0, 1), padding=1).transpose(0, 1)
    assert ((dw.double() - wd.grad).abs() / dwR).max().item() <= 2.0 ** -24 + 1e-12
    assert abs(db.double() - bd.grad).item() <= 2.0 ** -24 * gout.abs().sum().item() + 1e-12


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _labels(b, h, w, seed):
    return torch.from_numpy(np.random.default_rng(seed).random((b, 1, h, w)) < 0.3).float().to(DEV)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
@pytest.mark.parametrize("shape", [(2, 64, 96), (2, 264, 328)])
def test_forward_train_against_fp64_module(name, shape):
    torch.manual_seed(0)
    net = detector(name, seed=6).to(DEV).train()
    ref = copy.deepcopy(net).double()
    tf32 = copy.deepcopy(net)
    b, h, w = shape
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    lab = _labels(b, h // 8, w // 8, 2)

    def run(m, fwd, dtype):
        out = fwd(m)(x.to(dtype))
        F.binary_cross_entropy_with_logits(out, lab.to(dtype)).backward()
        return out.detach()

    out_n = run(net, lambda m: m.forward_train, torch.float32)
    out_r = run(ref, lambda m: m._forward_torch, torch.float64)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
        out_t = run(tf32, lambda m: m._forward_torch, torch.float32)
    assert out_n.shape == (b, 1, h // 8, w // 8)
    rows = [("out", out_n, out_t, out_r)]
    pn, pt, pr = dict(net.named_parameters()), dict(tf32.named_parameters()), dict(ref.named_parameters())
    used = [k for k in pr if pr[k].grad is not None]
    unused = [k for k in pr if pr[k].grad is None]
    for k in unused:
        assert pn[k].grad is None, k
    if name == "Resnet18_8s_detector_v2":
        assert all(k.startswith(("base_detector.resnet18_8s.layer3", "base_detector.resnet18_8s.layer4",
                                 "base_detector.resnet18_8s.fc")) for k in unused) and len(unused) > 0
        assert all(k.startswith(("out_conv", "base_detector.resnet18_8s.conv1", "base_detector.resnet18_8s.bn1",
                                 "base_detector.resnet18_8s.layer1", "base_detector.resnet18_8s.layer2"))
                   for k in used)
    else:
        assert not unused
    rows += [(f"grad {k}", pn[k].grad, pt[k].grad, pr[k].grad) for k in used]
    bn, bt, br = dict(net.named_buffers()), dict(tf32.named_buffers()), dict(ref.named_buffers())
    rows += [(k, bn[k], bt[k], br[k]) for k in br if "running" in k]
    bad = []
    for what, a, t, r in rows:
        e, et = _rel(a, r), _rel(t, r)
        print(f"{name} {shape} {what}: native {e:.2e}  torch TF32 graph {et:.2e}")
        if e > max(5e-3, 2 * et):
            bad.append((what, e, et))
    assert all(torch.equal(bn[k], br[k].to(bn[k].dtype)) for k in br if k.endswith("num_batches_tracked"))
    assert not bad, bad


def _step(net, opt, x, lab, **kw):
    out = net.forward_train(x, **kw)
    F.binary_cross_entropy_with_logits(out, lab).backward()
    if opt is not None:
        opt.step()
        opt.zero_grad()
    return out.detach()


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_seeded_steps_are_deterministic(name):
    b, h, w = 3, 64, 96
    lab = _labels(b, h // 8, w // 8, 5)
    results = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(7)
            net = detector(name, seed=7).to(DEV).train()
            opt = Adam([p for p in net.parameters()], lr=1e-3)
            for s in range(2):
                x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(10 + s))
                _step(net, opt, x, lab)
            results.append([t.detach().clone() for t in net.state_dict().values()])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(p, q) for p, q in zip(*results))


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_uint8_input_gives_the_float_inputs_bits(name):
    net = detector(name, seed=8).to(DEV).train()
    twin = copy.deepcopy(net)
    b, h, w = 2, 64, 96
    img = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (b, h, w, 3), dtype=np.uint8)).to(DEV)
    xf = ((img.permute(0, 3, 1, 2).float() / 255 - torch.tensor(MEAN, device=DEV).view(1, 3, 1, 1))
          / torch.tensor(STD, device=DEV).view(1, 3, 1, 1))
    lab = _labels(b, h // 8, w // 8, 4)
    assert torch.equal(_step(net, None, xf, lab), _step(twin, None, img, lab, mean=MEAN, std=STD))
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert (p.grad is None and q.grad is None) or torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k
    ev = _net(name, seed=8)
    with torch.no_grad():
        assert torch.equal(ev.forward_native(xf), ev.forward_native(img, mean=MEAN, std=STD))


def test_weight_updates_are_picked_up_including_the_base_of_v2():
    base = _net("Resnet18_8s_detector", seed=9)
    v2 = mr.Resnet18_8s_detector_v2(base).to(DEV).eval()
    x = torch.randn(1, 3, 64, 64, device=DEV)
    with torch.no_grad():
        a1, a2 = base(x).clone(), v2(x).clone()
        base.resnet18_8s.fc.bias.add_(1.0)
        v2.out_conv.bias.add_(1.0)
        b1, b2 = base(x), v2(x)
        assert torch.allclose(b1 - a1, torch.ones_like(a1), atol=2e-5 * max(1.0, a1.abs().max().item()))
        assert torch.allclose(b2 - a2, torch.ones_like(a2), atol=2e-5 * max(1.0, a2.abs().max().item()))
        assert base.native_pack_count() == 2 and v2.native_pack_count() == 2
        base.resnet18_8s.layer4[1].conv2.weight.mul_(2.0)   # not used by v2: no repack
        assert torch.equal(v2(x), b2) and v2.native_pack_count() == 2
        base.resnet18_8s.layer1[0].conv1.weight.mul_(0.5)   # used by v2: repacked
        c2 = v2(x)
        assert v2.native_pack_count() == 3 and not torch.equal(c2, b2)
        with _tf32(True):
            t = v2._forward_torch(x)
        assert (c2 - t).abs().max() <= 3e-3 * t.abs().max() + 1e-3


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_dataparallel_copies_and_pickle(name):
    net = _net(name, seed=3)
    x = torch.randn(2 * max(1, torch.cuda.device_count()), 3, 64, 96, device=DEV)
    ids = list(range(torch.cuda.device_count()))
    with torch.no_grad():
        out = net(x)
        assert out.shape == (x.shape[0], 1, 8, 12) and net.native_pack_count() == 1
        dp = nn.DataParallel(net, device_ids=ids)
        assert torch.equal(dp(x), out) and torch.equal(dp(x), out)
        assert net.native_pack_count() == len(ids)
        del dp
        gc.collect()
        assert torch.equal(copy.copy(net)(x), out)
        buf = io.BytesIO()
        torch.save(net, buf)
        buf.seek(0)
        loaded = torch.load(buf, weights_only=False)
        assert type(loaded) is type(net) and torch.equal(loaded(x), out) and loaded.native_pack_count() == 1
        assert torch.equal(net(x), out)


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_errors(name):
    net = _net(name)
    x = torch.randn(1, 3, 64, 64, device=DEV)
    for kw in (dict(with_mask=True), dict(pixel_major=True)):
        with pytest.raises(ValueError, match="score map"):
            net.forward_native(x, **kw)
    with pytest.raises(ValueError, match="multiples of 8"):
        net.forward_native(torch.randn(1, 3, 60, 64, device=DEV))
    tr = detector(name).to(DEV).train()
    with pytest.raises(ValueError, match="require grad"):
        tr.forward_train(x.clone().requires_grad_())
    with pytest.raises(ValueError, match="mean= and std="):
        tr.forward_train(x, mean=MEAN, std=STD)
    handle = net._prepare_native(torch.device(DEV))
    lib = _native.lib()
    n = ctypes.c_size_t()
    assert lib.pvnet_backbone_workspace_bytes(handle, 1, 64, 64, ctypes.byref(n)) == 0
    ws = torch.empty(n.value, dtype=torch.uint8, device=DEV)
    out = torch.empty(1, 1, 8, 8, device=DEV)
    mask = torch.empty(1, 8, 8, dtype=torch.int64, device=DEV)
    assert lib.pvnet_backbone_forward(handle, x.data_ptr(), 1, 64, 64, out.data_ptr(), mask.data_ptr(), 8,
                                      ws.data_ptr(), ws.numel(), None) == -1
    assert b"mask must be NULL" in lib.pvnet_last_error()
    slot = net._score_slot.split(".")
    parent = net.get_submodule(".".join(slot[:-1])) if len(slot) > 1 else net
    setattr(parent, slot[-1], nn.Conv2d(parent.get_submodule(slot[-1]).in_channels, 1, 1).to(DEV))
    tr = copy.deepcopy(net).train()
    with pytest.raises(ValueError, match="3x3 convolution to one channel"):
        tr.forward_train(x)
