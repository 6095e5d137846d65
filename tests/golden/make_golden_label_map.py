"""Regenerates tests/golden/ref_label_map.npz from the reference's
`OcclusionLineModDB.get_mask_of_all_objects` (lib/utils/data_utils.py).

The method is read with `ast` and run as it stands on a stub `self`: its `read_blender_pose` returns an empty array
for the missing poses of tests/label_map_cases.py's `golden_depth_maps(case)` and its `opengl_renderer.render`
returns that recipe's depth maps, so the reference's own compositing (argwhere, lexsort, unique) produces the label
maps.  Only those uint8 maps are stored (compressed); tests/test_label_map_cpu.py composites the same depth maps
with oracle/label_map_oracle.py and compares.
    PVNET_REFERENCE=<path> python tests/golden/make_golden_label_map.py
"""
import ast
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SOURCE = "lib/utils/data_utils.py"


def reference_method(path, cls, name):
    tree = ast.parse(open(path).read())
    node = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls)
    fn = next(n for n in node.body if isinstance(n, ast.FunctionDef) and n.name == name)
    namespace = {"np": np}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), namespace)
    return namespace[name]


class Stub:
    def __init__(self, case, class_type_to_number):
        from tests import label_map_cases as lc
        self.maps = dict(lc.golden_depth_maps(case))
        self.class_type_to_number = class_type_to_number
        self.class_type = None
        self.opengl_renderer = self

    def read_blender_pose(self, index):
        return np.array([]) if self.maps[self.class_type] is None else np.zeros((3, 4))

    def render(self, class_type, pose, camera_type=None):
        assert camera_type == "linemod" and class_type == self.class_type and pose.shape == (3, 4)
        return self.maps[class_type].copy()


def main():
    sys.path.insert(0, ROOT)
    from tests import label_map_cases as lc
    from tests.helpers import GOLDEN, reference_root
    path = os.path.join(reference_root(), SOURCE)
    fn = reference_method(path, "OcclusionLineModDB", "get_mask_of_all_objects")
    out = {}
    for case in range(lc.GOLDEN_CASES):
        out[f"case{case}"] = fn(Stub(case, dict(lc.OCCLUSION_CLASSES)), case)
        assert out[f"case{case}"].dtype == np.uint8 and out[f"case{case}"].shape == (lc.H, lc.W)
    np.savez_compressed(os.path.join(GOLDEN, "ref_label_map.npz"), **out)
    print("wrote", lc.GOLDEN_CASES, "cases")


if __name__ == "__main__":
    main()
