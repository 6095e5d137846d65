"""Regenerates tests/golden/ref_eval_signatures.json: the positional parameters (names and default expressions) of
the reference's evaluation entry points, read from its source with `ast`:
    lib/utils/evaluation_utils.py            pnp, find_nearest_point_distance, Evaluator.<methods>
    lib/utils/extend_utils/extend_utils.py   find_nearest_point_idx, uncertainty_pnp, uncertainty_pnp_v2
tests/test_dropin_eval_imports.py compares the shims' signatures with this file.
    PVNET_REFERENCE=<path> python tests/golden/make_golden_eval_signatures.py
"""
import ast
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WANTED = {
    "lib/utils/evaluation_utils.py": ["pnp", "find_nearest_point_distance", "Evaluator"],
    "lib/utils/extend_utils/extend_utils.py": ["find_nearest_point_idx", "uncertainty_pnp", "uncertainty_pnp_v2"],
}


def signature(fn):
    args = fn.args.args
    defaults = [None] * (len(args) - len(fn.args.defaults)) + list(fn.args.defaults)
    return ", ".join(a.arg if d is None else f"{a.arg}={ast.unparse(d)}" for a, d in zip(args, defaults))


def main():
    sys.path.insert(0, ROOT)
    from tests.helpers import GOLDEN, reference_root
    ref = reference_root()
    out = {}
    for rel, names in WANTED.items():
        tree = ast.parse(open(os.path.join(ref, rel)).read())
        for node in tree.body:
            if isinstance(node, ast.FunctionDef) and node.name in names:
                out[node.name] = signature(node)
            elif isinstance(node, ast.ClassDef) and node.name in names:
                for f in node.body:
                    if isinstance(f, ast.FunctionDef):
                        out[f"{node.name}.{f.name}"] = signature(f)
    with open(os.path.join(GOLDEN, "ref_eval_signatures.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "signatures")


if __name__ == "__main__":
    main()
