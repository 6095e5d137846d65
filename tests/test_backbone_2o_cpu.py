"""CPU: Resnet50_8s_2o is the reference's graph -- the same state-dict keys and shapes in the same order and the same
eval outputs (tests/golden/resnet50_8s_2o_ref.npz, made by tests/golden/make_golden_backbone_2o.py from the reference
class) -- x_ds's rounding sequence, and the half-resolution plan of pvnet_backbone_create_trunk_2o: its stages and
slots as the module describes them, the trunk exactly Resnet50_8s's, the workspace without the full-resolution
buffers, and the arguments it rejects."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pvnet_b200 import _native
from pvnet_b200 import model_repository as mr
from tests.deep_backbones import deep_backbone_input
from tests.helpers import GOLDEN, seeded_state_dict

GOLD = np.load(os.path.join(GOLDEN, "resnet50_8s_2o_ref.npz"))
R50_BLOCKS = (3, 4, 6, 3)
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def _create_2o(kind=1, blocks=R50_BLOCKS, ver=18, seg=2, dims=(384, 256, 128, 64)):
    handle = ctypes.c_void_p()
    rc = _native.lib().pvnet_backbone_create_trunk_2o(kind, None if blocks is None else (ctypes.c_int * 4)(*blocks),
                                                      ver, seg, *dims, ctypes.byref(handle))
    return rc, handle


def _create_r50(ver=18, seg=2):
    handle = ctypes.c_void_p()
    assert _native.lib().pvnet_backbone_create_trunk(1, (ctypes.c_int * 4)(*R50_BLOCKS), ver, seg, 384, 256, 128, 64,
                                                     64, ctypes.byref(handle)) == 0
    return handle


def _stage_names(handle):
    L = _native.lib()
    return [L.pvnet_backbone_handle_stage_name(handle, i).decode() for i in range(L.pvnet_backbone_handle_num_stages(handle))]


def _workspace(handle, b, h, w):
    n = ctypes.c_size_t()
    assert _native.lib().pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)) == 0
    return n.value


def test_state_dict_matches_reference_and_loads_strictly():
    net = mr.Resnet50_8s_2o(18, 2)
    sd = net.state_dict()
    assert list(sd) == GOLD["keys"].tolist()
    assert [",".join(str(d) for d in t.shape) for t in sd.values()] == GOLD["shapes"].tolist()
    assert "conv2s.0.bias" not in sd and tuple(sd["conv2s.0.weight"].shape) == (64, 195, 3, 3)
    assert tuple(sd["conv2s.3.weight"].shape) == (20, 64, 1, 1) and "conv2s.3.bias" in sd
    assert not any(k.startswith("convraw.") for k in sd)
    ref_sd = {k: torch.zeros([int(d) for d in s.split(",")] if s else []) for k, s in zip(GOLD["keys"], GOLD["shapes"])}
    ref_sd.update(seeded_state_dict(net, seed=4))
    assert net.load_state_dict(ref_sd, strict=True)
    assert torch.equal(net.state_dict()["conv2s.3.weight"], ref_sd["conv2s.3.weight"])


def test_torch_graph_reproduces_reference_outputs():
    net = mr.Resnet50_8s_2o(18, 2)
    net.load_state_dict(seeded_state_dict(net, seed=1))
    net.eval()
    x = torch.from_numpy(deep_backbone_input())
    with torch.no_grad():
        seg, ver = net._forward_torch(x)
    assert seg.shape == (2, 2, 28, 40) and ver.shape == (2, 18, 28, 40)
    for got, ref in ((seg, GOLD["seg"]), (ver, GOLD["ver"])):
        assert np.abs(got.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


def test_shim_exports_the_class_by_name():
    from lib.networks.model_repository import Resnet50_8s_2o
    assert Resnet50_8s_2o is mr.Resnet50_8s_2o


def _blocks(x):
    x = np.asarray(x, dtype=np.float32)
    return x[:, :, 0::2, 0::2], x[:, :, 0::2, 1::2], x[:, :, 1::2, 0::2], x[:, :, 1::2, 1::2]


def x_ds_device(x):
    """The pack's x_ds (and torch's CUDA kernel's): h0*(w0*a + w1*b) + h1*(w0*c + w1*d), every weight 0.5."""
    a, b, c, d = _blocks(x)
    h = np.float32(0.5)
    return h * (h * a + h * b) + h * (h * c + h * d)


def x_ds_cpu(x):
    """torch's CPU kernel: the four terms with weight 0.25 summed left to right."""
    a, b, c, d = _blocks(x)
    q = np.float32(0.25)
    return ((q * a + q * b) + q * c) + q * d


def _inputs():
    rng = np.random.default_rng(5)
    normal = rng.standard_normal((3, 3, 48, 64), dtype=np.float32) * np.float32(2.5)
    u8 = rng.integers(0, 256, (3, 48, 64, 3), dtype=np.uint8)
    # ToTensor + Normalize in fp32: (u / 255 - mean) / std, three correctly rounded ops
    t = torch.from_numpy(u8).permute(0, 3, 1, 2).float().div(torch.tensor(255.0))
    t = t.sub(torch.tensor(MEAN).view(1, 3, 1, 1)).div(torch.tensor(STD).view(1, 3, 1, 1))
    return [("normal", normal), ("uint8 ImageNet-normalised", t.contiguous().numpy())]


@pytest.mark.parametrize("which", [0, 1])
def test_x_ds_rounding_sequences(which):
    """Both rounding sequences restated in numpy: torch's CPU order is F.interpolate on the CPU bit for bit; the
    device order (what the pack computes, and F.interpolate on CUDA, pinned by test_gpu_backbone_2o.py) rounds the two
    row means first.  The two differ in the last bit on about a quarter of the pixels; both are within two ulps of
    the largest of the four terms from the exact mean."""
    _, x = _inputs()[which]
    ref = F.interpolate(torch.from_numpy(x), scale_factor=0.5, mode="bilinear", align_corners=False).numpy()
    assert np.array_equal(x_ds_cpu(x).view(np.uint32), ref.view(np.uint32))
    dev = x_ds_device(x)
    a, b, c, d = (t.astype(np.float64) for t in _blocks(x))
    exact = (a + b + c + d) / 4
    big = np.maximum(np.maximum(np.abs(a), np.abs(b)), np.maximum(np.abs(c), np.abs(d))).astype(np.float32)
    ulp = np.spacing(big).astype(np.float64)
    assert np.all(np.abs(dev - exact) <= 2 * ulp) and np.all(np.abs(ref - exact) <= 2 * ulp)
    assert 0.05 < (dev != ref).mean() < 0.5


def test_handle_stages_and_slots_match_the_module():
    net = mr.Resnet50_8s_2o(18, 2)
    rc, h = _create_2o()
    assert rc == 0
    r50 = _create_r50()
    L = _native.lib()
    try:
        names, r50_names = _stage_names(h), _stage_names(r50)
        slots = net._slots()
        convs = [n for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)]
        assert L.pvnet_backbone_handle_num_convs(h) == len(slots) == len(convs) == 58
        assert sorted(c for c, _ in slots) == sorted(convs)
        assert [c for c, _ in slots[-4:]] == ["conv8s.0", "conv4s.0", "conv2s.0", "conv2s.3"]
        assert slots[:-4] == mr.Resnet50_8s(18, 2)._slots()[:-5]
        # the trunk's stages (pack, stem, pool, every block, fc.0) and conv8s.0 .. conv4s.0 are Resnet50_8s's
        k = r50_names.index("conv2s.0")
        assert names[:k] == r50_names[:k]
        assert names[k:] == ["conv2s.0", "conv2s.3 1x1 + argmax head (fp32)"]
        conv_stages = [n for n in names if not n.startswith(("image", "maxpool", "upsample", "conv2s.3"))]
        assert len(conv_stages) == len(slots) - 1
        assert L.pvnet_backbone_output_scale(h) == 2 and L.pvnet_backbone_output_scale(r50) == 1
        assert L.pvnet_backbone_output_scale(None) == -1
        assert net._out_scale == 2 and mr.Resnet50_8s._out_scale == 1
    finally:
        L.pvnet_backbone_destroy(h)
        L.pvnet_backbone_destroy(r50)


@pytest.mark.parametrize("b,hh,ww", [(16, 480, 640), (2, 56, 80)])
def test_workspace_drops_the_full_resolution_buffers(b, hh, ww):
    rc, h = _create_2o()
    r50 = _create_r50()
    L = _native.lib()
    try:
        n2o, n50 = _workspace(h, b, hh, ww), _workspace(r50, b, hh, ww)
    finally:
        L.pvnet_backbone_destroy(h)
        L.pvnet_backbone_destroy(r50)
    p1 = b * hh * ww
    c1, r0, x = p1 * (64 + 8) * 4, p1 * 64 * 4, p1 // 4 * 8 * 4     # C1, R0 gone; X [b,H/2,W/2,8] added
    # every buffer starts on a 256-byte boundary: the rest of the carve is the same up to that padding
    assert abs((n50 - n2o) - (c1 + r0 - x)) <= 3 * 256
    assert n50 - n2o >= c1 + r0 - x - 3 * 256 > 0
    print(f"\nworkspace at {b}x{hh}x{ww}: Resnet50_8s {n50} B, Resnet50_8s_2o {n2o} B")


@pytest.mark.parametrize("kind,blocks,ver,seg,dims,msg", [
    (1, R50_BLOCKS, 18, 2, (384, 256, 128, 16), b"multiples of 32"),
    (1, R50_BLOCKS, 18, 2, (384, 256, 128, 96), b"s2dim must be 32 or 64"),
    (1, R50_BLOCKS, 18, 2, (384, 256, 128, 128), b"s2dim must be 32 or 64"),
    (1, R50_BLOCKS, 18, 2, (384, 256, 128, 48), b"multiples of 32"),
    (2, R50_BLOCKS, 18, 2, (384, 256, 128, 64), b"block kind"),
    (1, None, 18, 2, (384, 256, 128, 64), b"null block counts"),
    (1, (3, 4, 0, 3), 18, 2, (384, 256, 128, 64), b"stage 3"),
    (1, R50_BLOCKS, 60, 8, (384, 256, 128, 64), b"seg_dim+ver_dim"),
])
def test_create_trunk_2o_rejects_bad_arguments(kind, blocks, ver, seg, dims, msg):
    rc, h = _create_2o(kind, blocks, ver, seg, dims)
    assert rc == -1 and not h.value
    assert msg in _native.lib().pvnet_last_error()


def test_create_trunk_2o_rejects_a_null_out_pointer():
    L = _native.lib()
    assert L.pvnet_backbone_create_trunk_2o(1, (ctypes.c_int * 4)(*R50_BLOCKS), 18, 2, 384, 256, 128, 64, None) == -1


@pytest.mark.parametrize("kind,s2dim", [(0, 32), (1, 32), (1, 64)])
def test_create_trunk_2o_accepts_both_block_kinds_and_head_widths(kind, s2dim):
    rc, h = _create_2o(kind, (2, 2, 2, 2), 18, 2, (256, 128, 64, s2dim))
    assert rc == 0
    _native.lib().pvnet_backbone_destroy(h)
