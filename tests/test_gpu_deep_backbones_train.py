"""GPU: `forward_train` of Resnet34_8s and Resnet50_8s -- every layer on the native kernels, the Bottleneck blocks
included -- against the module graph in fp64, one step of the training losses and backward(); the uint8 input;
seeded steps under torch.use_deterministic_algorithms(True); and the train-mode BatchNorm block tails (forms 1 and 2)
at 2048 channels, forward and backward, against an fp64 restatement.

Tolerance, following test_gpu_conv_grad.py's argument for Resnet18_8s: the convolutions run with TF32 operands, and
through 36 or 53 layers the torch graph with cuDNN-TF32 is itself 0.5-2e-2 (relative L2) from fp64 on the outputs of
one step, more on some gradients: the deep layers carry the forward's TF32 error through every BatchNorm backward.  So
every output, parameter gradient and running statistic is held to 2x torch-TF32's own error on the same step, at
least 5e-3.  Two TF32 computations that sum in different orders land at errors of the same size, not the same
values, hence 2x rather than 1x; a dropped tap, block or BatchNorm term moves a row by far more."""
import copy

import numpy as np
import pytest
import torch

from pvnet_b200 import conv as pc
from pvnet_b200 import model_repository as mr
from pvnet_b200 import net_utils as nu
from pvnet_b200.optim import Adam
from tests.deep_backbones import DEEP_BACKBONE_CLASSES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _targets(b, h, w, K, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    masks = [((yy - rng.uniform(0.3, 0.7) * h) ** 2 + (xx - rng.uniform(0.3, 0.7) * w) ** 2 < (0.25 * h) ** 2)
             for _ in range(b)]
    mask = torch.from_numpy(np.stack(masks).astype(np.int64)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [w, h], (b, K, 2)), np.ones((b, K, 1))], 2)).to(DEV)
    return mask, hc


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_forward_train_against_fp64_module(name):
    torch.manual_seed(0)
    net = getattr(mr, name)(18, 2).to(DEV).train()
    ref = copy.deepcopy(net).double()
    tf32 = copy.deepcopy(net)
    b, h, w = 2, 64, 96
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    mask, hc = _targets(b, h, w, 9, 2)
    field, wgt = nu.vertex_targets(mask, hc), mask[:, None].float()

    def run(m, fwd, dtype):
        seg, ver = fwd(m)(x.to(dtype))
        loss_seg = torch.nn.functional.cross_entropy(seg, mask)
        loss_ver = nu._smooth_l1_torch(ver, field.to(dtype), wgt.to(dtype), 1.0, True).mean()
        (loss_seg + loss_ver).backward()
        return seg.detach(), ver.detach()

    out_n = run(net, lambda m: m.forward_train, torch.float32)
    out_r = run(ref, lambda m: m._forward_torch, torch.float64)
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=True):
        out_t = run(tf32, lambda m: m._forward_torch, torch.float32)
    rows = [("seg_pred", out_n[0], out_t[0], out_r[0]), ("ver_pred", out_n[1], out_t[1], out_r[1])]
    pn, pt, pr = dict(net.named_parameters()), dict(tf32.named_parameters()), dict(ref.named_parameters())
    rows += [(f"grad {k}", pn[k].grad, pt[k].grad, pr[k].grad) for k in pr]
    bn, bt, br = dict(net.named_buffers()), dict(tf32.named_buffers()), dict(ref.named_buffers())
    rows += [(k, bn[k], bt[k], br[k]) for k in br if "running" in k]
    assert len([r for r in rows if r[0].startswith("grad ")]) == len(list(ref.parameters()))
    bad = []
    for what, a, t, r in rows:
        e, et = _rel(a, r), _rel(t, r)
        print(f"{name} {what}: native {e:.2e}  torch TF32 graph {et:.2e}")
        if e > max(5e-3, 2 * et):
            bad.append((what, e, et))
    assert all(torch.equal(bn[k], br[k].to(bn[k].dtype)) for k in br if k.endswith("num_batches_tracked"))
    assert not bad, bad


def _step(net, opt, x, mask, hc, **kw):
    seg, ver = net.forward_train(x, **kw)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
    (ls.mean() + lv.mean()).backward()
    if opt is not None:
        opt.step()
        opt.zero_grad()
    return seg.detach(), ver.detach()


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_uint8_input_gives_the_float_inputs_bits(name):
    torch.manual_seed(0)
    net = getattr(mr, name)(18, 2).to(DEV).train()
    twin = copy.deepcopy(net)
    b, h, w = 2, 64, 96
    img = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (b, h, w, 3), dtype=np.uint8)).to(DEV)
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    # ToTensor + Normalize with 255 as a tensor: a true division, as the loader's ToTensor runs it (a Python-scalar
    # divisor may become a multiplication by its reciprocal, which differs in the last bit for some bytes)
    xf = img.permute(0, 3, 1, 2).float().div(torch.tensor(255.0, device=DEV)) \
        .sub(torch.tensor(mean, device=DEV).view(1, 3, 1, 1)).div(torch.tensor(std, device=DEV).view(1, 3, 1, 1)) \
        .contiguous()
    mask, hc = _targets(b, h, w, 9, 4)
    a = _step(net, None, xf, mask, hc)
    u = _step(twin, None, img, mask, hc, mean=mean, std=std)
    assert all(torch.equal(p, q) for p, q in zip(a, u))
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_seeded_steps_are_deterministic(name):
    b, h, w = 3, 64, 96
    mask, hc = _targets(b, h, w, 9, 5)
    results = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(7)
            net = getattr(mr, name)(18, 2).to(DEV).train()
            opt = Adam(net.parameters(), lr=1e-3)
            for s in range(2):
                x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(10 + s))
                _step(net, opt, x, mask, hc)
            results.append([t.detach().clone() for t in net.state_dict().values()])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(p, q) for p, q in zip(*results))


def _bn_fp64(form, x, z, bn, bz):
    """The block tails in fp64: relu(bn(x) + z), relu(bn(x) + bz(z)); batch statistics, running update."""
    return torch.relu(bn(x) + (z if form == 1 else bz(z)))


@pytest.mark.parametrize("form", [1, 2])
def test_batchnorm_at_2048_channels_against_fp64(form):
    """The block tails at Resnet50_8s's layer4 width (form 0 keeps its 1024-channel contract)."""
    C, b, h, w = 2048, 2, 6, 10
    g = torch.Generator(device=DEV).manual_seed(form)
    x = (torch.randn(b, C, h, w, device=DEV, generator=g) * 2 + 0.5).contiguous(memory_format=torch.channels_last)
    z = torch.randn(b, C, h, w, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(b, C, h, w, device=DEV, generator=g)
    bn, bz = torch.nn.BatchNorm2d(C).to(DEV).train(), torch.nn.BatchNorm2d(C).to(DEV).train()
    with torch.no_grad():
        for m in (bn, bz):
            m.weight.uniform_(0.5, 1.5, generator=g)
            m.bias.normal_(0, 0.1, generator=g)
            m.running_mean.normal_(0, 0.1, generator=g)
            m.running_var.uniform_(0.5, 1.5, generator=g)
    bn64, bz64 = copy.deepcopy(bn).double(), copy.deepcopy(bz).double()
    xn, zn = x.clone().requires_grad_(), z.clone().requires_grad_()
    y = pc.bn_add_relu(bn, xn, zn, bz if form == 2 else None)
    y.backward(dy)
    xd, zd = x.double().requires_grad_(), z.double().requires_grad_()
    yd = _bn_fp64(form, xd, zd, bn64, bz64)
    yd.backward(dy.double())
    rows = [("y", y, yd), ("dx", xn.grad, xd.grad), ("dgamma", bn.weight.grad, bn64.weight.grad),
            ("dbeta", bn.bias.grad, bn64.bias.grad), ("running_mean", bn.running_mean, bn64.running_mean),
            ("running_var", bn.running_var, bn64.running_var), ("dz", zn.grad, zd.grad)]
    if form == 2:
        rows += [("dgamma_z", bz.weight.grad, bz64.weight.grad), ("dbeta_z", bz.bias.grad, bz64.bias.grad),
                 ("running_var_z", bz.running_var, bz64.running_var)]
    for what, a, r in rows:
        e = (a.double() - r).abs().max().item() / max(r.abs().max().item(), 1e-30)
        assert e <= 2e-6, (what, e)
