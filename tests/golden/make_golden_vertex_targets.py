"""Regenerates tests/golden/ref_vertex_targets.npz by running the REFERENCE'S OWN compute_vertex_hcoords
(lib/datasets/linemod_dataset.py:68-81) and tools/demo.py's compute_vertex (:58-71) on the CPU.

    PVNET_REFERENCE=<path> python tests/golden/make_golden_vertex_targets.py

Their modules import cv2, torchvision and the project config at module level, so the two function definitions are
taken out of the source files with `ast` and executed with numpy alone.  The inputs are rebuilt from seeds by
tests/vertex_target_cases.py, so the file holds only outputs: per case the field [b,2K,h,w] (the loader's [h,w,2K]
per image after permute(2,0,1), NaNs made canonical) as a sha256 digest and a small slice of it; and the same for the
demo fixture (tests/helpers.demo_fixture) through compute_vertex.
"""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.helpers import _pack, demo_fixture, reference_root  # noqa: E402
from tests.vertex_target_cases import CASES, canon_nan, case_inputs  # noqa: E402


def load_function(relpath, name):
    """The function `name` defined at the top level of the reference's `relpath`, executed with only numpy bound."""
    path = os.path.join(reference_root(), relpath)
    tree = ast.parse(open(path).read(), filename=path)
    defs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == name]
    if len(defs) != 1:
        raise SystemExit(f"{relpath}: expected one top-level `def {name}`, found {len(defs)}")
    scope = {"np": np}
    exec(compile(ast.Module(body=defs, type_ignores=[]), path, "exec"), scope)
    return scope[name]


def slice_of(field):
    """Image 0, every channel, the first 8 pixels of the middle row."""
    return np.ascontiguousarray(canon_nan(field[0, :, field.shape[2] // 2, :8]))


def main():
    hcoords_fn = load_function(os.path.join("lib", "datasets", "linemod_dataset.py"), "compute_vertex_hcoords")
    demo_fn = load_function(os.path.join("tools", "demo.py"), "compute_vertex")
    out = {}
    for name in CASES:
        mask, hc, motion = case_inputs(name)
        with np.errstate(all="ignore"):
            field = np.stack([hcoords_fn(mask[i], hc[i], motion).transpose(2, 0, 1) for i in range(len(mask))])
        out[f"{name}/field"] = _pack(canon_nan(field))
        out[f"{name}/slice"] = slice_of(field)
        print(name, field.shape, int(np.isnan(field).sum()), "NaN")
    mask, _, pts = demo_fixture()
    field = demo_fn(mask, pts).transpose(2, 0, 1)[None]
    out["demo/field"] = _pack(canon_nan(field))
    out["demo/slice"] = slice_of(field)
    np.savez_compressed(os.path.join(HERE, "ref_vertex_targets.npz"), **out)
    print("wrote ref_vertex_targets.npz", len(out), "arrays")


if __name__ == "__main__":
    main()
