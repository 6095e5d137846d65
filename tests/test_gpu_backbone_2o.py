"""GPU: Resnet50_8s_2o on the native kernels.  Eval: against the reference's fp32 golden and our torch graph at
480x640 (the bound of test_gpu_deep_backbones.py: 3x cuDNN-TF32's own deviation, floor 3e-3 of the range), both
output layouts and the mask; the image pack's x_ds slice and the training stem's bit for bit against F.interpolate
on CUDA, for float and uint8 images; the stages this decoder adds (conv2s.0 over two sources, the head at half
resolution) against fp64 restatements of their own layers.  Training: forward_train against the fp64 module (the
rule of test_gpu_deep_backbones_train.py), the uint8 input's bits and seeded deterministic steps.  Lifecycle: weight
updates, DataParallel, pickling, and the pose pipeline on the half-resolution field.  The trunk stages are
Resnet50_8s's plan (tests/test_backbone_2o_cpu.py), checked stage by stage in test_gpu_backbone_stages.py."""
import copy
import gc
import io

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from pvnet_b200 import conv as pc
from pvnet_b200 import model_repository as mr
from pvnet_b200 import net_utils as nu
from pvnet_b200.optim import Adam
from pvnet_b200.pipeline import PoseKeypointPipeline
from tests.deep_backbones import deep_backbone_input
from tests.helpers import GOLDEN, seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _net(seed=1, ver=18):
    net = mr.Resnet50_8s_2o(ver, 2)
    net.load_state_dict(seeded_state_dict(net, seed=seed))
    return net.to(DEV).eval()


class _tf32:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = self.on
        torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


def _normalise(img):
    """ToTensor + Normalize on the device with a true division by 255 (as test_gpu_deep_backbones_train.py)."""
    return img.permute(0, 3, 1, 2).float().div(torch.tensor(255.0, device=DEV)) \
        .sub(torch.tensor(MEAN, device=DEV).view(1, 3, 1, 1)).div(torch.tensor(STD, device=DEV).view(1, 3, 1, 1)) \
        .contiguous()


def _x_ds(x):
    return F.interpolate(x, scale_factor=0.5, mode="bilinear", align_corners=False)


def _ws_buffers(net, b, h, w):
    """The first four buffers of the half-resolution plan's workspace, in carve order: S [b,h/2,w/2,16],
    X [b,h/2,w/2,8], C2 [b,h/2,w/2,s4+64], U2 [b,h/2,w/2,s2]."""
    ws = next(iter(net._nat.workspaces.values()))
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    q = b * (h // 2) * (w // 2)
    out, off = [], 0
    for ch in (16, 8, net.conv2s[0].in_channels - 3, net.conv2s[0].out_channels):
        out.append(ws[off:off + q * ch * 4].view(torch.float32).view(b, h // 2, w // 2, ch))
        off = al(off + q * ch * 4)
    return out


def test_native_vs_reference_golden():
    z = np.load(f"{GOLDEN}/resnet50_8s_2o_ref.npz")
    x, gseg, gver = deep_backbone_input(), z["seg"], z["ver"]
    net = _net()
    xd = torch.from_numpy(x).to(DEV)
    with torch.no_grad():
        seg, ver = net(xd)
        with _tf32(True):
            t = torch.cat(net._forward_torch(xd), 1)
    assert seg.shape == (2, 2, 28, 40) and ver.shape == (2, 18, 28, 40)
    gold = torch.from_numpy(np.concatenate([gseg, gver], 1)).to(DEV)
    e_cudnn = (t - gold).abs().max().item()
    for what, got, ref in (("seg", seg, gseg), ("ver", ver, gver)):
        err = np.abs(got.cpu().numpy() - ref).max()
        scale = np.abs(ref).max()
        print(f"\n[Resnet50_8s_2o vs reference fp32 golden] {what}: max abs err {err:.3e}, range {scale:.3f}; "
              f"cuDNN-TF32: {e_cudnn:.3e}")
        assert err <= max(3.0 * e_cudnn, 3e-3 * scale)


def test_native_vs_torch_graph_fullsize_masks_and_layouts():
    net = _net(seed=3)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        with _tf32(False):
            rs, rv = net._forward_torch(x)
        with _tf32(True):
            ts, tv = net._forward_torch(x)
        out, mask = net.forward_native(x, with_mask=True)
        out8, mask8 = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8)
        pm, pmask = net.forward_native(x, with_mask=True, pixel_major=True)
    assert out.shape == (2, 20, 240, 320) and mask.shape == (2, 240, 320) and pm.shape == (2, 240, 320, 20)
    seg, ver = out[:, :2], out[:, 2:]
    e_seg = (seg - rs).abs().max().item() / rs.abs().max().item()
    e_ver = (ver - rv).abs().max().item() / rv.abs().max().item()
    c_seg = (ts - rs).abs().max().item() / rs.abs().max().item()
    c_ver = (tv - rv).abs().max().item() / rv.abs().max().item()
    assert torch.equal(mask, torch.argmax(seg, 1))
    assert torch.equal(out8, out) and torch.equal(mask8.long(), mask)
    assert torch.equal(pm, out.permute(0, 2, 3, 1)) and torch.equal(pmask, mask)
    flips = (mask != torch.argmax(rs, 1)).float().mean().item()
    flips_cudnn = (torch.argmax(ts, 1) != torch.argmax(rs, 1)).float().mean().item()
    print(f"\n[Resnet50_8s_2o vs torch fp32 graph] 480x640: rel err seg {e_seg:.3e}, ver {e_ver:.3e} (cuDNN-TF32: "
          f"{c_seg:.3e}, {c_ver:.3e}); argmax flips {flips * 100:.4f}% (cuDNN-TF32: {flips_cudnn * 100:.4f}%)")
    assert e_seg <= max(3 * c_seg, 3e-3) and e_ver <= max(3 * c_ver, 3e-3)
    assert flips <= max(3 * flips_cudnn, 1e-4), "argmax flip rate against the fp32 graph"


@pytest.mark.parametrize("shape", [(2, 56, 80), (3, 64, 272)])
def test_pack_x_ds_is_interpolate_bit_for_bit(shape):
    """The eval pack's X buffer is round_tf32(F.interpolate(x, 0.5)) on CUDA, and zeros behind it, for a float image
    and for a uint8 image normalised on the device; the uint8 forward equals the float forward on the normalised
    image."""
    b, h, w = shape
    net = _net(seed=2)
    img = torch.from_numpy(np.random.default_rng(7).integers(0, 256, (b, h, w, 3), dtype=np.uint8)).to(DEV)
    xf = _normalise(img)
    xn = torch.from_numpy(np.random.default_rng(8).standard_normal((b, 3, h, w), dtype=np.float32) * 2.5).to(DEV)
    with torch.no_grad():
        for x in (xn, xf):
            out = net.forward_native(x)
            X = _ws_buffers(net, b, h, w)[1]
            assert torch.equal(X[..., :3], pc.round_tf32(_x_ds(x)).permute(0, 2, 3, 1))
            assert not X[..., 3:].any()
        ou = net.forward_native(img, mean=MEAN, std=STD)
        X = _ws_buffers(net, b, h, w)[1]
        assert torch.equal(X[..., :3], pc.round_tf32(_x_ds(xf)).permute(0, 2, 3, 1))
        assert torch.equal(ou, out)


@pytest.mark.parametrize("u8", [False, True])
def test_training_stem_writes_x_ds_unrounded(u8):
    b, h, w = 2, 64, 96
    img = torch.from_numpy(np.random.default_rng(9).integers(0, 256, (b, h, w, 3), dtype=np.uint8)).to(DEV)
    xf = _normalise(img) if u8 else torch.randn(b, 3, h, w, device=DEV) * 3
    wgt = torch.randn(64, 3, 7, 7, device=DEV) * 0.1
    buf = torch.full((b, 200, h // 2, w // 2), 7.0, device=DEV).contiguous(memory_format=torch.channels_last)
    if u8:
        y = pc.stem_train_half(img, wgt, buf, 192, MEAN, STD)
        y_full = pc.stem_train(img, wgt, None, 0, MEAN, STD)
    else:
        y = pc.stem_train_half(xf, wgt, buf, 192)
        y_full = pc.stem_train(xf, wgt)
    assert torch.equal(buf[:, 192:195], _x_ds(xf))
    assert not buf[:, 195:].any() and bool((buf[:, :192] == 7.0).all())
    assert torch.equal(y, y_full)


def test_new_stages_against_their_own_layers():
    """conv2s.0 (C2 and X as two sources, folded BatchNorm, LeakyReLU, unrounded output) and the fp32 head at H/2 x W/2,
    each from the buffers the stage before it left, against fp64."""
    net = _net(seed=5)
    b, h, w = 2, 64, 96
    x = torch.randn(b, 3, h, w, device=DEV)
    L = net._prepare_native(torch.device(DEV))
    from pvnet_b200 import _native
    lib = _native.lib()
    n = lib.pvnet_backbone_handle_num_stages(L)
    names = [lib.pvnet_backbone_handle_stage_name(L, i).decode() for i in range(n)]
    k = names.index("conv2s.0")
    assert k == n - 2
    out = torch.empty(b, 20, h // 2, w // 2, device=DEV)
    mask = torch.empty(b, h // 2, w // 2, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        net.run_stages(x, out, mask, 0, k)
        torch.cuda.synchronize()
        _, X, C2, _ = (t.clone() for t in _ws_buffers(net, b, h, w))
        net.run_stages(x, out, mask, k, k + 1)
        torch.cuda.synchronize()
        U2 = _ws_buffers(net, b, h, w)[3].clone()
        net.run_stages(x, out, mask, k + 1, n)
        torch.cuda.synchronize()
    c, bn = net.conv2s[0], net.conv2s[1]
    wf, bf = pc.fold_bn(c.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
    wt = pc.round_tf32(wf).double()
    inp = torch.cat([C2, X[..., :3]], 3).permute(0, 3, 1, 2).double()
    ref = F.conv2d(inp, wt, bf.double(), padding=1)
    R = F.conv2d(inp.abs(), wt.abs(), bf.double().abs(), padding=1)
    ref = F.leaky_relu(ref, 0.1)
    got = U2.permute(0, 3, 1, 2).double()
    err = ((got - ref).abs() / R.clamp_min(1e-30)).max().item()
    print(f"\nconv2s.0: max |err| / R = {err:.2e}")
    assert err <= 1e-5
    hd = net.conv2s[3]
    hw = hd.weight.detach().double().reshape(20, -1)
    href = torch.einsum("bchw,oc->bohw", got, hw) + hd.bias.detach().double().view(1, -1, 1, 1)
    hR = torch.einsum("bchw,oc->bohw", got.abs(), hw.abs()) + hd.bias.detach().double().abs().view(1, -1, 1, 1)
    herr = ((out.double() - href).abs() / hR).max().item()
    print(f"conv2s.3 head: max |err| / R = {herr:.2e}")
    assert herr <= 64 * 2.0 ** -24
    assert torch.equal(mask, torch.argmax(out[:, :2], 1))


def test_shared_stages_are_resnet50_8s_bit_for_bit():
    """Every stage before conv2s.0 -- pack, stem, max-pool, the trunk, fc.0, conv8s.0, UP8, conv4s.0, UP4 -- is
    Resnet50_8s's plan (tests/test_gpu_backbone_stages.py checks those stage by stage): with the same weights both
    handles leave the same bits in C2 (up(conv4s), x2s), which every one of those stages feeds, and in S."""
    b, h, w = 2, 64, 96
    n2o, n50 = _net(seed=4), mr.Resnet50_8s(18, 2)
    n50.load_state_dict({k: v for k, v in n2o.state_dict().items() if not k.startswith("conv2s.")}
                        | {k: v for k, v in seeded_state_dict(n50, seed=4).items()
                           if k.startswith(("conv2s.", "convraw."))})
    n50 = n50.to(DEV).eval()
    x = torch.randn(b, 3, h, w, device=DEV)
    from pvnet_b200 import _native
    lib = _native.lib()
    cuts = []
    for net, ho in ((n2o, h // 2), (n50, h)):
        handle = net._prepare_native(torch.device(DEV))
        names = [lib.pvnet_backbone_handle_stage_name(handle, i).decode()
                 for i in range(lib.pvnet_backbone_handle_num_stages(handle))]
        cuts.append(names.index("conv2s.0"))
        with torch.no_grad():
            net.run_stages(x, torch.empty(b, 20, ho, ho * w // h, device=DEV), None, 0, cuts[-1])
    torch.cuda.synchronize()
    assert cuts[0] == cuts[1]
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    q, p1 = b * (h // 2) * (w // 2), b * h * w
    S2o, _, C2o, _ = _ws_buffers(n2o, b, h, w)
    ws = next(iter(n50._nat.workspaces.values()))
    off = al(q * 16 * 4) + al(p1 * 72 * 4) + al(p1 * 64 * 4)           # S, C1, R0
    C2r = ws[off:off + q * 192 * 4].view(torch.float32).view(b, h // 2, w // 2, 192)
    S2r = ws[:q * 16 * 4].view(torch.float32).view(b, h // 2, w // 2, 16)
    assert torch.equal(S2o, S2r) and torch.equal(C2o, C2r) and C2o.abs().sum() > 0


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


@pytest.mark.parametrize("shape", [(2, 64, 96), (2, 480, 640)])
def test_forward_train_against_fp64_module(shape):
    torch.manual_seed(0)
    net = mr.Resnet50_8s_2o(18, 2).to(DEV).train()
    ref = copy.deepcopy(net).double()
    tf32 = copy.deepcopy(net)
    b, h, w = shape
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    mask, hc = _targets(b, h // 2, w // 2, 9, 2)
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
    assert out_n[0].shape == (b, 2, h // 2, w // 2)
    rows = [("seg_pred", out_n[0], out_t[0], out_r[0]), ("ver_pred", out_n[1], out_t[1], out_r[1])]
    pn, pt, pr = dict(net.named_parameters()), dict(tf32.named_parameters()), dict(ref.named_parameters())
    rows += [(f"grad {k}", pn[k].grad, pt[k].grad, pr[k].grad) for k in pr]
    bn, bt, br = dict(net.named_buffers()), dict(tf32.named_buffers()), dict(ref.named_buffers())
    rows += [(k, bn[k], bt[k], br[k]) for k in br if "running" in k]
    assert len([r for r in rows if r[0].startswith("grad ")]) == len(list(ref.parameters()))
    bad = []
    for what, a, t, r in rows:
        e, et = _rel(a, r), _rel(t, r)
        print(f"Resnet50_8s_2o {shape} {what}: native {e:.2e}  torch TF32 graph {et:.2e}")
        if e > max(5e-3, 2 * et):
            bad.append((what, e, et))
    assert all(torch.equal(bn[k], br[k].to(bn[k].dtype)) for k in br if k.endswith("num_batches_tracked"))
    assert not bad, bad


def test_forward_train_rejects_a_changed_head():
    net = mr.Resnet50_8s_2o(18, 2).to(DEV).train()
    net.conv2s[3] = nn.Conv2d(64, 20, 1, 1, bias=False).to(DEV)
    with pytest.raises(ValueError, match=r"conv2s\[3\]"):
        net.forward_train(torch.randn(1, 3, 32, 32, device=DEV))


def _step(net, opt, x, mask, hc, **kw):
    seg, ver = net.forward_train(x, **kw)
    ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
    (ls.mean() + lv.mean()).backward()
    if opt is not None:
        opt.step()
        opt.zero_grad()
    return seg.detach(), ver.detach()


def test_uint8_input_gives_the_float_inputs_bits():
    torch.manual_seed(0)
    net = mr.Resnet50_8s_2o(18, 2).to(DEV).train()
    twin = copy.deepcopy(net)
    b, h, w = 2, 64, 96
    img = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (b, h, w, 3), dtype=np.uint8)).to(DEV)
    mask, hc = _targets(b, h // 2, w // 2, 9, 4)
    a = _step(net, None, _normalise(img), mask, hc)
    u = _step(twin, None, img, mask, hc, mean=MEAN, std=STD)
    assert all(torch.equal(p, q) for p, q in zip(a, u))
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k


def test_seeded_steps_are_deterministic():
    b, h, w = 3, 64, 96
    mask, hc = _targets(b, h // 2, w // 2, 9, 5)
    results = []
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            torch.manual_seed(7)
            net = mr.Resnet50_8s_2o(18, 2).to(DEV).train()
            opt = Adam(net.parameters(), lr=1e-3)
            for s in range(2):
                x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(10 + s))
                _step(net, opt, x, mask, hc)
            results.append([t.detach().clone() for t in net.state_dict().values()])
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(p, q) for p, q in zip(*results))


def test_weights_update_is_picked_up():
    net = _net(seed=9)
    x = torch.randn(1, 3, 64, 64, device=DEV)
    with torch.no_grad():
        a = net.forward_native(x).clone()
        net.conv2s[3].bias.add_(1.0)
        b = net.forward_native(x)
    assert torch.allclose(b - a, torch.ones_like(a), atol=2e-5 * max(1.0, a.abs().max().item()))
    assert net.native_pack_count() == 2


def test_dataparallel_copies_and_pickle():
    net = _net(seed=3)
    x = torch.randn(2 * max(1, torch.cuda.device_count()), 3, 64, 96, device=DEV)
    ids = list(range(torch.cuda.device_count()))
    with torch.no_grad():
        seg, ver = net(x)
        assert seg.shape[2:] == (32, 48) and net.native_pack_count() == 1
        dp = nn.DataParallel(net, device_ids=ids)
        s1, v1 = dp(x)
        s2, _ = dp(x)
        assert torch.equal(s1, seg) and torch.equal(v1, ver) and torch.equal(s2, seg)
        assert net.native_pack_count() == len(ids), "one pack per device"
        del dp
        gc.collect()
        shallow = copy.copy(net)
        assert torch.equal(shallow(x)[0], seg) and net.native_pack_count() == len(ids)
        buf = io.BytesIO()
        torch.save(net, buf)
        buf.seek(0)
        loaded = torch.load(buf, weights_only=False)
        assert type(loaded) is type(net) and torch.equal(loaded(x)[0], seg) and loaded.native_pack_count() == 1
        assert torch.equal(net(x)[0], seg)


def test_pose_pipeline_end_to_end():
    """The pipeline runs unchanged on the half-resolution field: keypoints in the 48 x 64 output grid's pixels."""
    net = _net(seed=3)
    pipe = PoseKeypointPipeline(net, round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=128)
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)).to(DEV)
    with torch.no_grad():
        kp, cov = pipe.step(img)
    assert kp.shape == (2, 9, 2) and cov.shape == (2, 9, 2, 2)
    assert torch.isfinite(kp).all()
