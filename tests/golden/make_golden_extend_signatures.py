"""Regenerates tests/golden/ref_extend_utils_signatures.json: the positional parameters (names and default
expressions) of every public function of the reference's lib/utils/extend_utils/extend_utils.py, read from its
source with `ast`.  tests/test_extend_oracle.py compares the shim's signatures with this file.
    PVNET_REFERENCE=<path> python tests/golden/make_golden_extend_signatures.py
"""
import ast
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SOURCE = "lib/utils/extend_utils/extend_utils.py"


def signature(fn):
    args = fn.args.args
    defaults = [None] * (len(args) - len(fn.args.defaults)) + list(fn.args.defaults)
    return ", ".join(a.arg if d is None else f"{a.arg}={ast.unparse(d)}" for a, d in zip(args, defaults))


def main():
    sys.path.insert(0, ROOT)
    from tests.helpers import GOLDEN, reference_root
    tree = ast.parse(open(os.path.join(reference_root(), SOURCE)).read())
    out = {node.name: signature(node) for node in tree.body
           if isinstance(node, ast.FunctionDef) and not node.name.startswith("_")}
    with open(os.path.join(GOLDEN, "ref_extend_utils_signatures.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "signatures")


if __name__ == "__main__":
    main()
