"""CPU: the workspace layout and stage table of tests/backbone_stages.py agree with the built library, so the
stage-by-stage GPU test (test_gpu_backbone_stages.py) opens the buffers the forward really uses."""
import ctypes

import pytest

from pvnet_b200 import _native
from tests import backbone_stages as bs

WIDTHS = [bs.DEFAULT_DIMS, (128, 64, 32, 64, 32), (256, 128, 64, 256, 32), (512, 512, 512, 512, 32),
          (32, 32, 32, 32, 32)]
SHAPES = [(1, 16, 16), (3, 16, 16), (2, 64, 96), (1, 72, 104), (1, 256, 264), (16, 480, 640)]
# trunks of pvnet_backbone_create_trunk: both block kinds at 1-1-1-1, 3-4-6-3 and an irregular count whose layer1 /
# layer2 need the E buffer (more than two blocks), at the deep networks' decoder widths (raw_dim 64)
TRUNKS = [bs.Trunk(k, blocks, bs.DEEP_DIMS, "t.") for k in (False, True)
          for blocks in ((1, 1, 1, 1), (3, 4, 6, 3), (3, 1, 2, 5))]


def _trunk_id(t):
    return ("bottleneck-" if t.bottleneck else "basic-") + "-".join(map(str, t.blocks))


def _create(trunk, ver=18, seg=2):
    """A library handle for `trunk`: pvnet_backbone_create for Resnet18's, pvnet_backbone_create_trunk otherwise."""
    L = _native.lib()
    handle = ctypes.c_void_p()
    if trunk.blocks == (2, 2, 2, 2) and not trunk.bottleneck and trunk.dims[4] == 32:
        _native.check(L.pvnet_backbone_create(ver, seg, *trunk.dims, ctypes.byref(handle)), "pvnet_backbone_create")
    else:
        blocks = (ctypes.c_int * 4)(*trunk.blocks)
        _native.check(L.pvnet_backbone_create_trunk(int(trunk.bottleneck), blocks, ver, seg, *trunk.dims,
                                                    ctypes.byref(handle)), "pvnet_backbone_create_trunk")
    return handle


def _workspace_bytes(trunk, b, h, w):
    L = _native.lib()
    handle = _create(trunk)
    try:
        n = ctypes.c_size_t()
        _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)), "pvnet_backbone_workspace_bytes")
        return n.value
    finally:
        L.pvnet_backbone_destroy(handle)


def _check_layout(trunk, shape):
    at, total = bs.layout(trunk, *shape)
    assert total + 256 == _workspace_bytes(trunk, *shape)
    assert all(v % bs.ALIGN == 0 for v in at.values())
    assert list(at) == bs.buffers(trunk) and sorted(at.values()) == list(at.values())


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("dims", WIDTHS, ids=str)
def test_layout_matches_library(dims, shape):
    _check_layout(bs.RESNET18._replace(dims=dims), shape)


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("trunk", TRUNKS, ids=_trunk_id)
def test_trunk_layout_matches_library(trunk, shape):
    _check_layout(trunk, shape)
    if max(trunk.blocks[:2]) > 2:
        assert {"E1", "E2"} & set(bs.buffers(trunk))


@pytest.mark.parametrize("seg,ver", [(2, 18), (2, 34), (3, 18)])
def test_stage_table_matches_library(seg, ver):
    L = _native.lib()
    table = bs.stages(bs.RESNET18, seg, ver, 2, 64, 96)
    assert len(table) == L.pvnet_backbone_num_stages()
    assert [s.name for s in table] == [L.pvnet_backbone_stage_name(i).decode() for i in range(len(table))]
    # exactly one stage, the head when convraw.0 carries it, launches nothing
    idle = [s.name for s in table if not s.writes]
    assert idle == ([table[-1].name] if seg + ver <= 32 else [])


@pytest.mark.parametrize("trunk", TRUNKS + [bs.RESNET18, bs.RESNET34, bs.RESNET50], ids=_trunk_id)
def test_trunk_stage_table_matches_library(trunk):
    L = _native.lib()
    handle = _create(trunk)
    try:
        n = L.pvnet_backbone_handle_num_stages(handle)
        names = [L.pvnet_backbone_handle_stage_name(handle, i).decode() for i in range(n)]
    finally:
        L.pvnet_backbone_destroy(handle)
    table = bs.stages(trunk, 2, 18, 2, 64, 96)
    assert [s.name for s in table] == names
    # raw_dim 64: the head is never fused, every stage launches something
    assert all(s.writes for s in table) == (trunk.dims[4] == 64)


def test_deep_tables_name_the_networks_modules():
    from pvnet_b200.model_repository import Resnet34_8s, Resnet50_8s, Resnet18_8s
    for cls, trunk in ((Resnet18_8s, bs.RESNET18), (Resnet34_8s, bs.RESNET34), (Resnet50_8s, bs.RESNET50)):
        net = cls(18, 2)
        mods = dict(net.named_modules())
        table = bs.stages(trunk, 2, 18, 2, 64, 96)
        convs = [(s.conv, s.bn) for s in table if s.kind in ("stem", "conv")]
        # the stage order of the convs is the native slot order the host layer packs weights in
        assert convs == net._slots()[:-1], cls.__name__
        for st in table:
            if st.kind != "conv":
                continue
            conv = mods[st.conv]
            cin = sum(r.cc for r in st.reads)
            assert conv.in_channels == cin - (5 if st.conv == "convraw.0" else 0), st.name
            assert conv.out_channels == st.writes[0].cc or st.writes[0].buf == "out", st.name
            assert (st.res is not None) == (".conv" in st.conv and st.conv.endswith(
                ".conv3" if trunk.bottleneck else ".conv2")), st.name
            if st.res is not None:
                assert st.res.cc == conv.out_channels and st.res.grid == st.writes[0].grid, st.name
            n, h, w = st.reads[0].grid
            ho, wo = st.writes[0].grid[1:]
            assert (h // conv.stride[0], w // conv.stride[0]) == (ho, wo), st.name


def test_stage_regions_lie_inside_their_buffers():
    trunks = [bs.RESNET18._replace(dims=d) for d in WIDTHS] + TRUNKS + [bs.RESNET34, bs.RESNET50]
    for trunk in trunks:
        b, h, w = 2, 72, 104
        sizes = bs.buffer_floats(trunk, b, h, w)
        for st in bs.stages(trunk, 2, 18, b, h, w):
            for r in st.reads + st.writes + ((st.res,) if st.res else ()):
                if r.buf in sizes:
                    n, hh, ww = r.grid
                    assert r.off + n * hh * ww * r.cs <= sizes[r.buf], (st.name, r)
                    assert 0 <= r.co and r.co + r.cc <= r.cs, (st.name, r)
