"""GPU: the native eval forward of Resnet34_8s and Resnet50_8s (the trunk-description plan of
pvnet_backbone_create_trunk, the k_head kernel at raw_dim 64) against the reference's fp32 golden outputs and our
torch graph, with the rule of test_gpu_backbone.py: every conv runs with TF32 operands, so the bound is 3x the
deviation cuDNN-TF32 itself shows on the same input (floor 3e-3 of the range); a dropped tap, block or wrong BN fold
moves the output by far more.  Also: the masks and the pixel-major layout, weight updates, DataParallel,
pickling, the pose pipeline, k_head bit for bit, and Resnet18_8s through the trunk creator byte for byte."""
import copy
import ctypes
import gc
import io
import types

import numpy as np
import pytest
import torch
from torch import nn

from pvnet_b200 import _native
from pvnet_b200 import model_repository as mr
from pvnet_b200.pipeline import PoseKeypointPipeline
from tests.deep_backbones import DEEP_BACKBONE_CLASSES, deep_backbone_golden
from tests.helpers import seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _net(name, seed=1, ver=18):
    net = getattr(mr, name)(ver, 2)
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


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_native_vs_reference_golden(name):
    x, gseg, gver = deep_backbone_golden(name)
    net = _net(name)
    xd = torch.from_numpy(x).to(DEV)
    with torch.no_grad():
        seg, ver = net(xd)
        with _tf32(True):
            t = torch.cat(net._forward_torch(xd), 1)
    gold = torch.from_numpy(np.concatenate([gseg, gver], 1)).to(DEV)
    e_cudnn = (t - gold).abs().max().item()
    for what, got, ref in (("seg", seg, gseg), ("ver", ver, gver)):
        err = np.abs(got.cpu().numpy() - ref).max()
        scale = np.abs(ref).max()
        print(f"\n[{name} vs reference fp32 golden] {what}: max abs err {err:.3e}, range {scale:.3f}; "
              f"cuDNN-TF32: {e_cudnn:.3e}")
        assert err <= max(3.0 * e_cudnn, 3e-3 * scale)


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_native_vs_torch_graph_fullsize_masks_and_layouts(name):
    net = _net(name, seed=3)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        with _tf32(False):
            rs, rv = net._forward_torch(x)
        with _tf32(True):
            ts, tv = net._forward_torch(x)
        out, mask = net.forward_native(x, with_mask=True)
        out8, mask8 = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8)
        pm, pmask = net.forward_native(x, with_mask=True, pixel_major=True)
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
    print(f"\n[{name} vs torch fp32 graph] 480x640: rel err seg {e_seg:.3e}, ver {e_ver:.3e} (cuDNN-TF32: {c_seg:.3e}, "
          f"{c_ver:.3e}); argmax flips {flips * 100:.4f}% (cuDNN-TF32: {flips_cudnn * 100:.4f}%)")
    assert e_seg <= max(3 * c_seg, 3e-3) and e_ver <= max(3 * c_ver, 3e-3)
    assert flips <= max(3 * flips_cudnn, 1e-4), "argmax flip rate against the fp32 graph"


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_weights_update_is_picked_up(name):
    net = _net(name, seed=9)
    x = torch.randn(1, 3, 64, 64, device=DEV)
    with torch.no_grad():
        a = net.forward_native(x).clone()
        net.convraw[3].bias.add_(1.0)
        b = net.forward_native(x)
    # the head sums 64 products in fp32 after its bias: each of the two chains rounds by at most 64 half-ulps of the
    # largest partial sum
    assert torch.allclose(b - a, torch.ones_like(a), atol=2e-5 * max(1.0, a.abs().max().item()))
    assert net.native_pack_count() == 2


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_dataparallel_copies_and_pickle(name):
    net = _net(name, seed=3)
    x = torch.randn(2 * max(1, torch.cuda.device_count()), 3, 64, 96, device=DEV)
    ids = list(range(torch.cuda.device_count()))
    with torch.no_grad():
        seg, ver = net(x)
        assert net.native_pack_count() == 1
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


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_pose_pipeline_end_to_end(name):
    net = _net(name, seed=3)
    pipe = PoseKeypointPipeline(net, round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=128)
    img = torch.from_numpy(np.random.default_rng(1).integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)).to(DEV)
    with torch.no_grad():
        kp, cov = pipe.step(img)
    assert kp.shape == (2, 9, 2) and cov.shape == (2, 9, 2, 2)
    assert torch.isfinite(kp).all()


def test_resnet18_through_the_trunk_creator_is_byte_identical():
    net = _net("Resnet18_8s", seed=3)
    twin = copy.deepcopy(net)
    twin._create_handle = types.MethodType(mr._Resnet8s._create_handle, twin)     # pvnet_backbone_create_trunk
    x = torch.from_numpy(np.random.default_rng(4).standard_normal((2, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        a, ma = net.forward_native(x, with_mask=True)
        b, mb = twin.forward_native(x, with_mask=True)
    L = _native.lib()
    h = twin._prepare_native(torch.device(DEV))
    assert L.pvnet_backbone_handle_num_convs(h) == 26
    assert torch.equal(a, b) and torch.equal(ma, mb)


def _fma32(a, b, c):
    """fmaf(a, b, c) correctly rounded, elementwise: the product is exact in fp64, the sum an fp64 two-sum; the fp32
    rounding is decided by the sum, or by the two-sum's error when the sum is an fp32 midpoint."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    back = r.astype(np.float64)
    nxt = np.nextafter(r, np.where(s > back, np.float32(np.inf), np.float32(-np.inf))).astype(np.float32)
    mid = (back + nxt.astype(np.float64)) / 2
    toward = np.sign(err) == np.sign(nxt.astype(np.float64) - back)
    return np.where((s == mid) & (err != 0) & toward, nxt, r)


@pytest.mark.parametrize("ties", [False, True])
def test_head_at_64_channels_is_exact_fp32(ties):
    """k_head<64> on the workspace's convraw.0 output (buffer R0, third in the carve order) against an fp32
    restatement, bit for bit; with identical seg rows every pixel ties and the mask is the first maximum, 0."""
    net = _net("Resnet34_8s", seed=6)
    if ties:
        with torch.no_grad():
            net.convraw[3].weight[1].copy_(net.convraw[3].weight[0])
            net.convraw[3].bias[1].copy_(net.convraw[3].bias[0])
    b, h, w = 2, 56, 80
    x = torch.randn(b, 3, h, w, device=DEV)
    L = _native.lib()
    handle = net._prepare_native(torch.device(DEV))
    nst = L.pvnet_backbone_handle_num_stages(handle)
    assert L.pvnet_backbone_handle_stage_name(handle, nst - 1).startswith(b"convraw.3")
    out = torch.empty(b, 20, h, w, device=DEV)
    mask = torch.empty(b, h, w, dtype=torch.int64, device=DEV)
    with torch.no_grad():
        net.run_stages(x, out, mask, 0, nst)
    torch.cuda.synchronize()
    ws = next(iter(net._nat.workspaces.values()))
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    p1 = b * h * w
    off = al(p1 // 4 * 16 * 4) + al(p1 * (64 + 8) * 4)
    r0 = ws[off:off + p1 * 64 * 4].view(torch.float32).view(p1, 64).cpu().numpy()
    wt = net.convraw[3].weight.detach().reshape(20, 64).cpu().numpy()
    acc = np.broadcast_to(net.convraw[3].bias.detach().cpu().numpy(), (p1, 20)).astype(np.float32)
    for j in range(64):
        acc = _fma32(r0[:, j:j + 1], wt[None, :, j], acc)
    ref = acc.reshape(b, h, w, 20).transpose(0, 3, 1, 2)
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    ref_mask = np.argmax(ref[:, :2], 1)
    assert np.array_equal(mask.cpu().numpy(), ref_mask)
    if ties:
        assert np.array_equal(ref[:, 0], ref[:, 1]) and not mask.any()
