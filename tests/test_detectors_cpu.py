"""CPU: Resnet18_8s_detector and Resnet18_8s_detector_v2 are the reference's graphs -- the same state-dict keys and
shapes in the same order (reference checkpoints load strictly) and the same eval outputs on seeded weights
(tests/golden/resnet18_8s_detectors_ref.npz, made by tests/golden/make_golden_detectors.py from the reference
classes) -- and the decoder-less plan of pvnet_backbone_create_detector: its slots and stages as the modules describe
them, its workspace, and the arguments it rejects.  Also the score head's fixed summation order restated in numpy,
and the device rules: eval refuses the CPU, train mode runs torch."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from pvnet_b200 import _native
from pvnet_b200 import conv as pc
from pvnet_b200 import model_repository as mr
from tests.detectors import (DETECTOR_CLASSES, buffer_offsets, detector, detector_buffers, detector_golden,
                             detector_state_dict_shapes, head3x3_fp64)
from tests.helpers import seeded_state_dict


def _create(kind=0, blocks=(2, 2, 2, 2), last_stage=4):
    handle = ctypes.c_void_p()
    rc = _native.lib().pvnet_backbone_create_detector(kind, None if blocks is None else (ctypes.c_int * 4)(*blocks),
                                                      last_stage, ctypes.byref(handle))
    return rc, handle


def _stage_names(handle):
    L = _native.lib()
    return [L.pvnet_backbone_handle_stage_name(handle, i).decode()
            for i in range(L.pvnet_backbone_handle_num_stages(handle))]


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_state_dict_matches_reference_and_loads_strictly(name):
    net = detector(name)
    ref = detector_state_dict_shapes()[name]
    assert [[k, list(t.shape)] for k, t in net.state_dict().items()] == ref
    fresh = mr.Resnet18_8s_detector() if name == "Resnet18_8s_detector" else \
        mr.Resnet18_8s_detector_v2(mr.Resnet18_8s_detector())
    sd = seeded_state_dict(fresh, seed=4)
    assert fresh.load_state_dict(sd, strict=True)
    head = "resnet18_8s.fc" if name == "Resnet18_8s_detector" else "out_conv"
    assert torch.equal(fresh.state_dict()[head + ".weight"], sd[head + ".weight"])


def test_v2_shares_the_base_parameters():
    base = mr.Resnet18_8s_detector()
    v2 = mr.Resnet18_8s_detector_v2(base)
    assert v2.base_detector is base
    assert v2.state_dict()["base_detector.resnet18_8s.conv1.weight"].data_ptr() == \
        base.resnet18_8s.conv1.weight.data_ptr()
    assert tuple(v2.out_conv.weight.shape) == (1, 128, 3, 3) and tuple(base.resnet18_8s.fc.weight.shape) == (1, 512, 3, 3)


def test_heads_keep_conv2d_default_init():
    """The trunk's init loop (N(0, sqrt(2/n))) runs before fc / out_conv exist, so they keep nn.Conv2d's default
    uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)) initialisation, as in the reference."""
    torch.manual_seed(0)
    v2 = mr.Resnet18_8s_detector_v2(mr.Resnet18_8s_detector())
    for conv, fan in ((v2.base_detector.resnet18_8s.fc, 512 * 9), (v2.out_conv, 128 * 9)):
        bound = fan ** -0.5
        assert conv.weight.abs().max() <= bound and conv.bias.abs().max() <= bound
        assert conv.weight.std() < 0.7 * bound           # uniform: std = bound / sqrt(3); N(0, sqrt(2/9)) is far wider


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_torch_graph_reproduces_reference_outputs(name):
    x, gold = detector_golden(name)
    net = detector(name).eval()
    with torch.no_grad():
        out = net._forward_torch(torch.from_numpy(x)).numpy()
    assert out.shape == gold.shape == (2, 1, 7, 10)
    np.testing.assert_allclose(out, gold, rtol=1e-5, atol=1e-5 * np.abs(gold).max())


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_slots_cover_every_convolution_in_execution_order(name):
    """Every Conv2d the graph runs is a slot, once; per block the downsample comes just before the conv whose
    epilogue adds it, and the head is last."""
    net = detector(name).eval()
    ran = []
    names = {m: n for n, m in net.named_modules()}
    hooks = [m.register_forward_hook(lambda m, i, o: ran.append(names[m]))
             for m in net.modules() if isinstance(m, nn.Conv2d)]
    with torch.no_grad():
        net._forward_torch(torch.randn(1, 3, 32, 32))
    for h in hooks:
        h.remove()
    slots = [c for c, _ in net._slots()]
    assert sorted(slots) == sorted(ran) and len(set(slots)) == len(slots)
    expect = []
    for n in ran:                                        # BasicBlock.forward runs the downsample after conv2
        if n.endswith("downsample.0"):
            expect.insert(len(expect) - 1, n)
        else:
            expect.append(n)
    assert slots == expect
    assert slots[-1] == net._score_slot and net._slots()[-1][1] is None
    rc, handle = _create(last_stage=net._last_stage)
    assert rc == 0
    try:
        assert _native.lib().pvnet_backbone_handle_num_convs(handle) == len(slots) == (21 if net._last_stage == 4 else 11)
        conv_stages = [s for s in _stage_names(handle) if s.split(" ")[0].endswith(("conv1", "conv2", "downsample"))
                       or s.startswith("stem")]
        assert len(conv_stages) == len(slots) - 1
        for s, (c, _) in zip(conv_stages[1:], net._slots()[1:-1]):
            assert c.removesuffix(".0").endswith(s.split(" ")[0]), (s, c)
    finally:
        _native.lib().pvnet_backbone_destroy(handle)


@pytest.mark.parametrize("last_stage", [4, 2])
def test_creator_reports_the_plan(last_stage):
    L = _native.lib()
    rc, handle = _create(last_stage=last_stage)
    assert rc == 0
    try:
        names = _stage_names(handle)
        assert names[:3] == ["image: space-to-depth packing", "stem conv1+bn1+relu", "maxpool 3x3/2"]
        assert names[-1] == ("fc 3x3 -> 1 score head (fp32)" if last_stage == 4 else "out_conv 3x3 -> 1 score head (fp32)")
        assert not any(n.startswith(("fc.0", "conv8s", "conv4s", "conv2s", "convraw", "upsample")) for n in names)
        assert len(names) == 3 + (20 if last_stage == 4 else 10)
        assert L.pvnet_backbone_output_scale(handle) == 8
        for b, h, w in ((2, 56, 80), (16, 480, 640)):
            n = ctypes.c_size_t()
            assert L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)) == 0
            assert n.value == buffer_offsets(detector_buffers(last_stage), b, h, w)[1] + 256
        assert L.pvnet_backbone_forward(handle, None, 1, 64, 64, None, None, 0, None, 0, None) == -1
    finally:
        L.pvnet_backbone_destroy(handle)


def test_creator_rejects_bad_descriptions():
    L = _native.lib()
    for kw, msg in ((dict(last_stage=3), b"last_stage"), (dict(last_stage=0), b"last_stage"),
                    (dict(kind=2), b"block kind"), (dict(blocks=None), b"null block"),
                    (dict(blocks=(2, 0, 2, 2)), b"blocks"), (dict(kind=1, blocks=(3, 4, 6, 3)), b"512 channels")):
        rc, _ = _create(**kw)
        assert rc == -1 and msg in L.pvnet_last_error(), kw
    assert L.pvnet_backbone_create_detector(0, (ctypes.c_int * 4)(2, 2, 2, 2), 4, None) == -1
    rc, handle = _create(kind=1, blocks=(3, 4, 6, 3), last_stage=2)    # a Bottleneck layer2 has 512 channels
    assert rc == 0
    L.pvnet_backbone_destroy(handle)


def _head3x3_order(y, w9, bias):
    """The kernel's summation order (include/pvnet_b200.h, pvnet_head3x3_nchw) for y [b,H,W,C] float32: one chain per
    output from bias, 32-channel chunks ascending, then taps, then channels; fmaf emulated as an exact fp64 product
    plus the fp32 accumulator, rounded to fp32."""
    b, H, W, C = y.shape
    pad = np.zeros((b, H + 2, W + 2, C), np.float32)
    pad[:, 1:-1, 1:-1] = y
    inside = np.zeros((b, H + 2, W + 2), bool)
    inside[:, 1:-1, 1:-1] = True
    acc = np.full((b, H, W), bias[0], np.float32)
    for c0 in range(0, C, 32):
        for t in range(9):
            ky, kx = divmod(t, 3)
            src = pad[:, ky:ky + H, kx:kx + W]
            ok = inside[:, ky:ky + H, kx:kx + W]
            for c in range(c0, c0 + 32):
                nxt = (np.float64(w9[t, c]) * src[..., c].astype(np.float64) + acc.astype(np.float64)).astype(np.float32)
                acc = np.where(ok, nxt, acc)
    return acc


def test_head_summation_order_restated():
    rng = np.random.default_rng(0)
    y = rng.standard_normal((2, 5, 7, 64)).astype(np.float32)
    w = torch.from_numpy(rng.standard_normal((1, 64, 3, 3)).astype(np.float32))
    bias = torch.tensor([0.25])
    w9 = pc.pack_head3x3(w).numpy()
    assert w9.shape == (9, 64) and w9[4, 3] == w[0, 3, 1, 1] and w9[2, 7] == w[0, 7, 0, 2]
    got = _head3x3_order(y, w9, bias.numpy())
    ref, R = head3x3_fp64(torch.from_numpy(y).permute(0, 3, 1, 2), w, bias)
    err = (torch.from_numpy(got).double() - ref[:, 0]).abs() / R[:, 0]
    assert err.max() <= (9 * 64 + 1) * 2.0 ** -24
    assert err.max() > 0                                   # the fp32 chain really rounds


@pytest.mark.parametrize("name", DETECTOR_CLASSES)
def test_eval_refuses_cpu_and_train_mode_runs_torch(name):
    net = detector(name)
    x = torch.randn(1, 3, 32, 48)
    out = net.train()(x)
    assert out.shape == (1, 1, 4, 6)
    torch.manual_seed(0)
    a = detector(name).train()
    b = detector(name).train()
    assert torch.equal(a(x), b._forward_torch(x))
    with pytest.raises(RuntimeError, match="CUDA"):
        net.eval()(x)
    with pytest.raises(RuntimeError, match="CUDA"):
        net.forward_train(x)
    for kw in (dict(with_mask=True), dict(pixel_major=True)):
        with pytest.raises(ValueError, match="score map"):
            net.forward_native(x, **kw)


def test_shim_exports_the_detectors():
    import lib.networks.model_repository as shim
    assert shim.Resnet18_8s_detector is mr.Resnet18_8s_detector
    assert shim.Resnet18_8s_detector_v2 is mr.Resnet18_8s_detector_v2
    assert "Resnet18_8s_detector" not in shim.__all__
