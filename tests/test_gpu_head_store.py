"""GPU: convraw.0's fused head stages each tile's output in shared memory and warps that issue no MMAs copy it out.
Only where the bytes are stored from changed, so every output and mask must be byte-identical to the digests
recorded before that change (tests/golden/make_golden_head_store.py), in both layouts, with both mask dtypes and at
shapes with partial tiles."""
import json
import os

import pytest

from tests.golden import make_golden_head_store as mg

pytestmark = pytest.mark.gpu

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "head_store.json")) as _f:
    GOLDEN = {(tuple(c["shape"]), c["pixel_major"], c["mask_dtype"]): (c["out_sha256"], c["mask_sha256"])
              for c in json.load(_f)["cases"]}


@pytest.fixture(scope="module")
def net():
    return mg.make_net()


@pytest.mark.parametrize("shape,pixel_major,mask_dtype", list(mg.cases()),
                         ids=lambda v: str(v) if not isinstance(v, bool) else ("pixel-major" if v else "nchw"))
def test_head_store_bytes_unchanged(net, shape, pixel_major, mask_dtype):
    got = mg.digests(net, mg.make_input(shape), pixel_major, mask_dtype)
    out_sha, mask_sha = GOLDEN[(tuple(shape), pixel_major, mask_dtype)]
    assert got[0] == out_sha, "head output bytes differ from the recorded digest"
    assert got[1] == mask_sha, "mask bytes differ from the recorded digest"
