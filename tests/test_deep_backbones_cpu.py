"""CPU: Resnet34_8s and Resnet50_8s are the reference's graphs -- the same state-dict keys and shapes in the same
order (tests/golden/resnet_8s_ref_state_dicts.json), the same eval outputs (tests/golden/resnet{34,50}_8s_ref.npz, both
made by tests/golden/make_golden_backbones.py from the reference classes) -- and the trunk-description ABI
(pvnet_backbone_create_trunk) plans them, and Resnet18_8s, as the modules describe them."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from pvnet_b200 import _native
from pvnet_b200 import model_repository as mr
from tests.deep_backbones import DEEP_BACKBONE_CLASSES, deep_backbone_golden
from tests.helpers import GOLDEN, seeded_state_dict

REF_KEYS = json.load(open(os.path.join(GOLDEN, "resnet_8s_ref_state_dicts.json")))
SLOTS = {"Resnet34_8s": 42, "Resnet50_8s": 59}


def _create_trunk(kind, blocks, ver=18, seg=2, dims=(384, 256, 128, 64, 64)):
    L = _native.lib()
    handle = ctypes.c_void_p()
    rc = L.pvnet_backbone_create_trunk(kind, None if blocks is None else (ctypes.c_int * 4)(*blocks), ver, seg, *dims,
                                       ctypes.byref(handle))
    return rc, handle


def _stage_names(handle):
    L = _native.lib()
    return [L.pvnet_backbone_handle_stage_name(handle, i).decode() for i in range(L.pvnet_backbone_handle_num_stages(handle))]


def test_shim_exports_the_three_networks():
    ns = {}
    exec("from lib.networks.model_repository import *", ns)
    assert {"Resnet18_8s", "Resnet34_8s", "Resnet50_8s"} <= set(ns)
    assert "Resnet50_8s_2o" not in ns and "Resnet18_8s_detector" not in ns


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_state_dict_matches_reference(name):
    net = getattr(mr, name)(18, 2)
    assert [[k, list(t.shape)] for k, t in net.state_dict().items()] == REF_KEYS[name]
    assert all(k.startswith(("resnet50_8s.", "conv8s.", "conv4s.", "conv2s.", "convraw.")) for k in net.state_dict())
    # a reference-format checkpoint (its keys, its shapes) loads strictly
    ref_sd = {k: torch.zeros(s) for k, s in REF_KEYS[name]}
    ref_sd.update(seeded_state_dict(net, seed=4))
    assert net.load_state_dict(ref_sd, strict=True)
    assert torch.equal(net.state_dict()["convraw.3.weight"], ref_sd["convraw.3.weight"])


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_torch_graph_reproduces_reference_outputs(name):
    x, gseg, gver = deep_backbone_golden(name)
    net = getattr(mr, name)(18, 2)
    net.load_state_dict(seeded_state_dict(net, seed=1))
    net.eval()
    with torch.no_grad():
        seg, ver = net._forward_torch(torch.from_numpy(x))
    # the same fp32 graph on the same CPU library: only summation-order noise
    for got, ref in ((seg, gseg), (ver, gver)):
        assert np.abs(got.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_slots_cover_every_conv_in_execution_order(name):
    net = getattr(mr, name)(18, 2)
    slots = net._slots()
    convs = [n for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)]
    assert len(slots) == SLOTS[name] and sorted(c for c, _ in slots) == sorted(convs)
    mods = dict(net.named_modules())
    for conv, bn in slots:
        if bn is not None:
            assert mods[bn].num_features == mods[conv].out_channels
    # execution order: a block's convs in sequence, its downsample just before the conv that adds it
    order = {c: i for i, (c, _) in enumerate(slots)}
    t = net.resnet50_8s
    for li in range(1, 5):
        for bi, blk in enumerate(getattr(t, f"layer{li}")):
            p = f"resnet50_8s.layer{li}.{bi}."
            last = "conv3" if isinstance(blk, mr.Bottleneck) else "conv2"
            assert order[p + "conv1"] < order[p + last]
            if blk.downsample is not None:
                assert order[p + "downsample.0"] == order[p + last] - 1
    assert [c for c, _ in slots[-5:]] == ["conv8s.0", "conv4s.0", "conv2s.0", "convraw.0", "convraw.3"]
    # the library's stage list runs the slots in this order
    h = ctypes.c_void_p()
    net._create_handle(h)
    try:
        conv_stages = [s for s in _stage_names(h) if s.startswith(("stem", "layer", "fc.", "conv8s", "conv4s", "conv2s",
                                                                   "convraw.0"))]
        assert len(conv_stages) == len(slots) - 1
        for s, (conv, _) in zip(conv_stages[1:], slots[1:]):
            assert conv.replace("resnet50_8s.", "").startswith(s.split(" ")[0].replace("downsample", "downsample.0"))
    finally:
        _native.lib().pvnet_backbone_destroy(h)


@pytest.mark.parametrize("kind,blocks,slots", [(0, (3, 4, 6, 3), 42), (1, (3, 4, 6, 3), 59)])
def test_new_trunk_handles_report_their_plan(kind, blocks, slots):
    L = _native.lib()
    rc, h = _create_trunk(kind, blocks)
    assert rc == 0
    try:
        assert L.pvnet_backbone_handle_num_convs(h) == slots
        names = _stage_names(h)
        # pack, pool, 3 upsamplings and the head besides one stage per conv slot but the head
        assert len(names) == slots - 1 + 6 and len(set(names)) == len(names)
        assert names[0].startswith("image") and names[-1].startswith("convraw.3")
    finally:
        L.pvnet_backbone_destroy(h)
    # the handle-less queries keep describing Resnet18_8s
    assert L.pvnet_backbone_num_convs() == 26 and L.pvnet_backbone_num_stages() == 31


def test_resnet18_restated_through_the_trunk_creator():
    L = _native.lib()
    rc, h = _create_trunk(0, (2, 2, 2, 2), dims=(256, 128, 64, 32, 32))
    assert rc == 0
    try:
        assert L.pvnet_backbone_handle_num_convs(h) == L.pvnet_backbone_num_convs() == 26
        assert _stage_names(h) == [L.pvnet_backbone_stage_name(i).decode() for i in range(L.pvnet_backbone_num_stages())]
        for b, hh, ww in [(1, 16, 16), (16, 480, 640)]:
            n = ctypes.c_size_t()
            _native.check(L.pvnet_backbone_workspace_bytes(h, b, hh, ww, ctypes.byref(n)), "workspace")
            h2 = ctypes.c_void_p()
            _native.check(L.pvnet_backbone_create(18, 2, 256, 128, 64, 32, 32, ctypes.byref(h2)), "create")
            n2 = ctypes.c_size_t()
            _native.check(L.pvnet_backbone_workspace_bytes(h2, b, hh, ww, ctypes.byref(n2)), "workspace")
            L.pvnet_backbone_destroy(h2)
            assert n.value == n2.value
    finally:
        L.pvnet_backbone_destroy(h)


@pytest.mark.parametrize("kind,blocks,dims,what", [
    (2, (3, 4, 6, 3), (384, 256, 128, 64, 64), "block kind"),
    (-1, (3, 4, 6, 3), (384, 256, 128, 64, 64), "block kind"),
    (1, None, (384, 256, 128, 64, 64), "null block counts"),
    (1, (3, 0, 6, 3), (384, 256, 128, 64, 64), "blocks"),
    (0, (3, 4, 65, 3), (384, 256, 128, 64, 64), "blocks"),
    (1, (3, 4, 6, 3), (384, 256, 128, 64, 48), "raw_dim"),
    (1, (3, 4, 6, 3), (384, 256, 128, 64, 128), "raw_dim"),
    (1, (3, 4, 6, 3), (384, 250, 128, 64, 64), "multiples of 32"),
    (0, (3, 4, 6, 3), (1024, 256, 128, 64, 64), "above 512"),
])
def test_trunk_creator_rejects_bad_descriptions(kind, blocks, dims, what):
    rc, h = _create_trunk(kind, blocks, dims=dims)
    assert rc != 0 and not h.value
    assert what in _native.lib().pvnet_last_error().decode()


def test_trunk_creator_rejects_bad_head_width():
    rc, h = _create_trunk(0, (3, 4, 6, 3), ver=70, seg=2)
    assert rc != 0 and not h.value


def test_handle_queries_on_null():
    L = _native.lib()
    assert L.pvnet_backbone_handle_num_convs(None) == -1 and L.pvnet_backbone_handle_num_stages(None) == -1
    assert L.pvnet_backbone_handle_stage_name(None, 0) == b""


@pytest.mark.parametrize("name", DEEP_BACKBONE_CLASSES)
def test_eval_mode_refuses_cpu_and_train_mode_runs_torch(name):
    net = getattr(mr, name)(18, 2).eval()
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.zeros(1, 3, 32, 32))
    net.train()
    seg, ver = net(torch.randn(2, 3, 32, 48))
    assert seg.shape == (2, 2, 32, 48) and ver.shape == (2, 18, 32, 48) and seg.requires_grad
