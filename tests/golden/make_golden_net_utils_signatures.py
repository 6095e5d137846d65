"""Regenerates tests/golden/ref_net_utils_signatures.json: the positional parameters (names and default expressions)
of the eight names tools/demo.py:6 and tools/train_linemod.py:19 import from the reference's lib/utils/net_utils.py,
and of the methods of its AverageMeter and Recorder classes, read from its source with `ast`.
tests/test_net_utils_cpu.py compares the shim's signatures with this file.
    PVNET_REFERENCE=<path> python tests/golden/make_golden_net_utils_signatures.py
"""
import ast
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WANTED = ["AverageMeter", "Recorder", "smooth_l1_loss", "load_model", "save_model", "adjust_learning_rate",
          "compute_precision_recall", "set_learning_rate"]


def signature(fn):
    args = fn.args.args
    defaults = [None] * (len(args) - len(fn.args.defaults)) + list(fn.args.defaults)
    return ", ".join(a.arg if d is None else f"{a.arg}={ast.unparse(d)}" for a, d in zip(args, defaults))


def main():
    sys.path.insert(0, ROOT)
    from tests.helpers import GOLDEN, reference_root
    tree = ast.parse(open(os.path.join(reference_root(), "lib", "utils", "net_utils.py")).read())
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in WANTED:
            out[node.name] = signature(node)
        elif isinstance(node, ast.ClassDef) and node.name in WANTED:
            for f in node.body:
                if isinstance(f, ast.FunctionDef):
                    out[f"{node.name}.{f.name}"] = signature(f)
    with open(os.path.join(GOLDEN, "ref_net_utils_signatures.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", len(out), "signatures")


if __name__ == "__main__":
    main()
