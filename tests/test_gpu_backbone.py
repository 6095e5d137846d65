"""GPU: the native Resnet18_8s (wgmma convs) against (a) the golden outputs produced by the
REFERENCE classes on the CPU in true fp32, (b) our torch graph on the GPU with TF32 off.

Tolerance.  The native path computes every conv with TF32 inputs (10-bit mantissa) and fp32
accumulation -- what the reference's own cuDNN path does on this GPU under torch's default
`cudnn.allow_tf32=True`.  Through 26 layers this gives ~2e-3 of the output range.  The bound is 3x the
error cuDNN-TF32 itself shows on the same input in the same test (floor 3e-3 of the range, in case cuDNN
picks fp32 kernels for the small test shapes): a dropped K-block or tap in any layer, or a wrong BN fold,
moves the output by far more.  Argmax flips against the fp32 graph are bounded too."""

import numpy as np
import pytest
import torch

from pvnet_b200.model_repository import Resnet18_8s
from tests.helpers import backbone_golden, seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _net(ver, seed=1):
    net = Resnet18_8s(ver, 2)
    net.load_state_dict(seeded_state_dict(net, seed=seed))
    return net.to(DEV).eval()


class _tf32:
    """cudnn / matmul TF32 switches, restored on exit."""

    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = self.on
        torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


def _cudnn_tf32_error(net, x, ref):
    """max abs deviation of the torch graph under cuDNN-TF32 from `ref` (true fp32) on this input"""
    with torch.no_grad(), _tf32(True):
        t = torch.cat(net._forward_torch(x), 1)
    return (t - ref).abs().max().item()


@pytest.mark.parametrize("tag,ver", [("k9", 18), ("k17", 34)])
def test_native_vs_reference_golden(tag, ver):
    z = backbone_golden()
    net = _net(ver)
    x = torch.from_numpy(z[tag + "_x"]).to(DEV)
    with torch.no_grad():
        seg, v = net(x)
    torch.cuda.synchronize()
    gold = torch.from_numpy(np.concatenate([z[tag + "_seg"], z[tag + "_ver"]], 1)).to(DEV)
    e_cudnn = _cudnn_tf32_error(net, x, gold)
    for name, got, ref in (("seg", seg, z[tag + "_seg"]), ("ver", v, z[tag + "_ver"])):
        got = got.cpu().numpy()
        err = np.abs(got - ref).max()
        scale = np.abs(ref).max()
        print(f"\n[backbone vs reference fp32 golden] {tag} {name}: max abs err {err:.3e}, range {scale:.3f}, "
              f"rel {err / scale:.3e}; cuDNN-TF32 on the same input: {e_cudnn:.3e}")
        assert err <= max(3.0 * e_cudnn, 3e-3 * scale)


def test_native_vs_torch_graph_fullsize_and_mask():
    net = _net(18, seed=3)
    x = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        with _tf32(False):
            rs, rv = net._forward_torch(x)
        with _tf32(True):
            ts, tv = net._forward_torch(x)
        out, mask = net.forward_native(x, with_mask=True)
        out8, mask8 = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8)
    torch.cuda.synchronize()
    seg, ver = out[:, :2], out[:, 2:]
    e_seg = (seg - rs).abs().max().item() / rs.abs().max().item()
    e_ver = (ver - rv).abs().max().item() / rv.abs().max().item()
    c_seg = (ts - rs).abs().max().item() / rs.abs().max().item()
    c_ver = (tv - rv).abs().max().item() / rv.abs().max().item()
    # bit-exact argmax GIVEN our logits (the fused head's mask == torch.argmax of its own output)
    assert torch.equal(mask, torch.argmax(seg, 1))
    assert torch.equal(out8, out) and torch.equal(mask8.long(), mask)
    flips = (mask != torch.argmax(rs, 1)).float().mean().item()
    flips_cudnn = (torch.argmax(ts, 1) != torch.argmax(rs, 1)).float().mean().item()
    print(f"\n[backbone vs torch fp32 graph] 480x640: rel err seg {e_seg:.3e}, ver {e_ver:.3e} (cuDNN-TF32: {c_seg:.3e}, "
          f"{c_ver:.3e}); argmax pixels differing from the fp32 graph: {flips * 100:.4f}% (cuDNN-TF32: {flips_cudnn * 100:.4f}%)")
    assert e_seg <= max(3 * c_seg, 3e-3) and e_ver <= max(3 * c_ver, 3e-3)
    assert flips <= max(3 * flips_cudnn, 1e-4), "argmax flip rate against the fp32 graph"


def test_native_matches_cudnn_tf32_class():
    """The reference's default numerics on this GPU (cuDNN TF32) deviate from fp32 by about as
    much as the native path does."""
    net = _net(18, seed=5)
    x = torch.from_numpy(np.random.default_rng(1).standard_normal((1, 3, 240, 320), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        with _tf32(False):
            f32 = torch.cat(net._forward_torch(x), 1)
        with _tf32(True):
            tf32 = torch.cat(net._forward_torch(x), 1)
        ours = net.forward_native(x)
    scale = f32.abs().max().item()
    e_cudnn = (tf32 - f32).abs().max().item() / scale
    e_ours = (ours - f32).abs().max().item() / scale
    print(f"\n[tf32 class] rel err vs fp32: cuDNN-TF32 {e_cudnn:.3e}, native {e_ours:.3e}")
    assert e_ours < max(3 * e_cudnn, 3e-3)


def test_reference_view_roundtrip_into_vote():
    """forward -> argmax -> permuted view -> ransac_voting_layer_v3, as tools/demo.py:46-55."""
    from pvnet_b200 import ransac_voting_gpu as rv
    net = _net(18, seed=7)
    x = torch.randn(2, 3, 128, 160, device=DEV)
    with torch.no_grad():
        seg_pred, vertex_pred = net(x)
    vertex = vertex_pred.permute(0, 2, 3, 1)
    b, h, w, vn2 = vertex.shape
    vertex = vertex.view(b, h, w, vn2 // 2, 2)
    mask = torch.argmax(seg_pred, 1)
    kp = rv.ransac_voting_layer_v3(mask, vertex, 64, inlier_thresh=0.99)
    assert kp.shape == (2, 9, 2)


def test_weights_update_is_picked_up():
    net = _net(18, seed=9)
    x = torch.randn(1, 3, 64, 64, device=DEV)
    with torch.no_grad():
        a = net.forward_native(x).clone()
        net.convraw[3].bias.add_(1.0)
        b = net.forward_native(x)
    assert torch.allclose(b - a, torch.ones_like(a), atol=1e-5)


def test_odd_sizes_multiple_of_8():
    net = _net(18, seed=2)
    for h, w in [(72, 104), (256, 264)]:
        x = torch.randn(1, 3, h, w, device=DEV)
        with torch.no_grad():
            with _tf32(False):
                ref = torch.cat(net._forward_torch(x), 1)
            out = net.forward_native(x)
        assert (out - ref).abs().max().item() <= max(3 * _cudnn_tf32_error(net, x, ref), 3e-3 * ref.abs().max().item())
