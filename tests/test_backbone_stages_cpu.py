"""CPU: the workspace layout and stage table of tests/backbone_stages.py agree with the built library, so the
stage-by-stage GPU test (test_gpu_backbone_stages.py) opens the buffers the forward really uses."""
import ctypes

import pytest

from pvnet_b200 import _native
from tests import backbone_stages as bs

WIDTHS = [bs.DEFAULT_DIMS, (128, 64, 32, 64, 32), (256, 128, 64, 256, 32), (512, 512, 512, 512, 32),
          (32, 32, 32, 32, 32)]
SHAPES = [(1, 16, 16), (3, 16, 16), (2, 64, 96), (1, 72, 104), (1, 256, 264), (16, 480, 640)]


def _workspace_bytes(dims, b, h, w, ver=18, seg=2):
    L = _native.lib()
    handle = ctypes.c_void_p()
    _native.check(L.pvnet_backbone_create(ver, seg, *dims, ctypes.byref(handle)), "pvnet_backbone_create")
    try:
        n = ctypes.c_size_t()
        _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)), "pvnet_backbone_workspace_bytes")
        return n.value
    finally:
        L.pvnet_backbone_destroy(handle)


@pytest.mark.parametrize("shape", SHAPES, ids=str)
@pytest.mark.parametrize("dims", WIDTHS, ids=str)
def test_layout_matches_library(dims, shape):
    at, total = bs.layout(dims, *shape)
    assert total + 256 == _workspace_bytes(dims, *shape)
    assert all(v % bs.ALIGN == 0 for v in at.values())
    assert list(at) == list(bs.BUFFERS) and sorted(at.values()) == list(at.values())


@pytest.mark.parametrize("seg,ver", [(2, 18), (2, 34), (3, 18)])
def test_stage_table_matches_library(seg, ver):
    L = _native.lib()
    table = bs.stages(bs.DEFAULT_DIMS, seg, ver, 2, 64, 96)
    assert len(table) == L.pvnet_backbone_num_stages()
    assert [s.name for s in table] == [L.pvnet_backbone_stage_name(i).decode() for i in range(len(table))]
    # exactly one stage, the head when convraw.0 carries it, launches nothing
    idle = [s.name for s in table if not s.writes]
    assert idle == ([table[-1].name] if seg + ver <= 32 else [])


def test_stage_regions_lie_inside_their_buffers():
    for dims in WIDTHS:
        b, h, w = 2, 72, 104
        sizes = bs.buffer_floats(dims, b, h, w)
        for st in bs.stages(dims, 2, 18, b, h, w):
            for r in st.reads + st.writes + ((st.res,) if st.res else ()):
                if r.buf in sizes:
                    n, hh, ww = r.grid
                    assert r.off + n * hh * ww * r.cs <= sizes[r.buf], (st.name, r)
                    assert 0 <= r.co and r.co + r.cc <= r.cs, (st.name, r)
