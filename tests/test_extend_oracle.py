"""CPU: the farthest-point-sampling / rasterisation oracle (oracle/extend_oracle.c) against the reference's own
compiled code, as recorded in tests/golden/ref_extend.npz (tests/golden/make_golden_ref_extend.py), and the
`lib.utils.extend_utils.extend_utils` shim: the reference's import lines, its eight public names and signatures
(tests/golden/ref_extend_utils_signatures.json), no cv2 or plyfile at import, and the two stubs."""
import inspect
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import extend_oracle as eo
from tests import extend_cases as ec
from tests.helpers import GOLDEN, same_as_stored

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_extend.npz")))


@pytest.mark.parametrize("name", ec.FPS_CASES)
def test_fps_oracle_equals_reference(golden, name):
    pts = ec.fps_cloud(name)
    pn = len(pts)
    for mode in ec.FPS_MODES:
        for sn in ec.fps_sample_counts(pn):
            got = eo.farthest_point_sampling(pts, sn, None if mode == "center" else ec.fps_start(pn))
            assert same_as_stored(got, golden[f"fps/{name}/{mode}/{sn}"]), (name, mode, sn)


@pytest.mark.parametrize("name", ec.RASTER_CASES)
def test_raster_oracle_equals_reference(golden, name):
    t, h, w = ec.raster_case(name)
    got = eo.mesh_binary_rasterization(t, h, w)
    assert got.dtype == np.uint8 and got.shape == (h, w) and set(np.unique(got)) <= {0, 1}
    assert same_as_stored(got, golden[f"raster/{name}"]), name


def test_golden_covers_every_case(golden):
    want = ec.golden_entries(lambda p, sn, s: np.zeros(sn, np.int32), lambda t, h, w: np.zeros((h, w), np.uint8))
    assert sorted(golden) == sorted(want)


def test_fps_oracle_known_answers():
    # a unit segment with its midpoint: the centre is the midpoint, so the first pick is the lowest farthest end;
    # the midpoint starts at min_dist 0 and is never picked, and once no min_dist is above 0 the answer is index 0
    pts = np.array([[0, 0, 0], [1, 0, 0], [0.5, 0, 0], [1, 0, 0]], np.float32)
    assert eo.farthest_point_sampling(pts, 4).tolist() == [0, 1, 0, 0]
    assert eo.farthest_point_sampling(pts, 3, start=2).tolist() == [2, 0, 1]
    assert eo.farthest_point_sampling(pts, 2, start=6).tolist() == [2, 0]   # start is taken modulo pn


def test_raster_oracle_known_answers():
    # a right triangle with its legs on the mask's axes covers the lattice points with x + y <= 4
    m = eo.mesh_binary_rasterization(np.array([[[0, 0], [4, 0], [0, 4]]], np.float32), 8, 9)
    yy, xx = np.mgrid[0:8, 0:9]
    assert np.array_equal(m, ((xx + yy) <= 4).astype(np.uint8))
    # the box stops at w - 2 and h - 2 before the +1: the last row and column are reachable, nothing beyond
    m = eo.mesh_binary_rasterization(np.array([[[-10, -10], [100, -10], [-10, 100]]], np.float32), 6, 7)
    assert m.all()


def test_reference_import_lines_without_cv2_or_plyfile():
    code = "\n".join([
        "import sys",
        "from lib.utils.extend_utils.extend_utils import farthest_point_sampling",            # data_utils.py:18
        "from lib.utils.extend_utils.extend_utils import uncertainty_pnp, find_nearest_point_idx, uncertainty_pnp_v2",
        "from lib.utils.extend_utils.extend_utils import mesh_binary_rasterization, post_refinement, "
        "render_mesh_depth, render_mesh_rgb",
        "print(sorted(m for m in ('cv2', 'plyfile') if m in sys.modules))",
    ])
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "[]", out.stdout


def _signature(fn):
    parts = []
    for p in inspect.signature(fn).parameters.values():
        if p.kind is not inspect.Parameter.POSITIONAL_OR_KEYWORD:
            continue                      # keyword-only extras (start=, return_indices=) are ours
        parts.append(p.name if p.default is inspect.Parameter.empty else f"{p.name}={p.default!r}")
    return ", ".join(parts)


def test_all_public_names_with_reference_signatures():
    import lib.utils.extend_utils.extend_utils as ex
    with open(os.path.join(GOLDEN, "ref_extend_utils_signatures.json")) as f:
        expected = json.load(f)
    assert len(expected) == 8
    for name, want in expected.items():
        assert _signature(getattr(ex, name)) == want, name


def test_stubs():
    import lib.utils.extend_utils.extend_utils as ex
    assert ex.post_refinement(np.zeros((4, 4)), np.eye(3, 4), np.eye(3), np.zeros((5, 3))) is None
    with pytest.raises(NotImplementedError, match="commented out"):
        ex.render_mesh_depth(np.eye(3, 4), np.eye(3), np.zeros((3, 3)), np.zeros((1, 3)), 4, 4, True)
    with pytest.raises(NotImplementedError, match="commented out"):
        ex.render_mesh_rgb(np.eye(3, 4), np.eye(3), np.zeros((3, 3)), np.zeros((3, 3)), np.zeros((1, 3)), 4, 4, True)
