"""CPU: the reference's evaluation import lines resolve against the shims under lib/ without loading cv2 or plyfile,
and the public signatures equal the reference's, as recorded from its source in tests/golden/ref_eval_signatures.json
(tests/golden/make_golden_eval_signatures.py)."""
import inspect
import json
import os
import subprocess
import sys

from tests.helpers import GOLDEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the value of the reference's default expression where the shim spells it differently
SAME_DEFAULT = {"cv2.SOLVEPNP_ITERATIVE": "0"}


def test_reference_import_lines_without_cv2_or_plyfile():
    code = "\n".join([
        "import sys",
        "from lib.utils.evaluation_utils import pnp",                                      # tools/demo.py:9
        "from lib.utils.evaluation_utils import Evaluator",                                # tools/train_linemod.py:18
        "from lib.utils.extend_utils.extend_utils import uncertainty_pnp, find_nearest_point_idx, uncertainty_pnp_v2",
        "print(sorted(m for m in ('cv2', 'plyfile') if m in sys.modules))",               # evaluation_utils.py:16
    ])
    out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == "[]", out.stdout


def _signature(fn):
    parts = []
    for p in inspect.signature(fn).parameters.values():
        if p.kind is not inspect.Parameter.POSITIONAL_OR_KEYWORD:
            continue                      # keyword-only extras (model_db=, projector=) are ours
        parts.append(p.name if p.default is inspect.Parameter.empty else f"{p.name}={p.default!r}")
    return ", ".join(parts)


def test_signatures_equal_reference():
    import lib.utils.evaluation_utils as ev
    import lib.utils.extend_utils.extend_utils as ex
    with open(os.path.join(GOLDEN, "ref_eval_signatures.json")) as f:
        expected = json.load(f)
    assert len(expected) == 15
    for name, want in expected.items():
        for ref_expr, ours in SAME_DEFAULT.items():
            want = want.replace(ref_expr, ours)
        if "." in name:
            cls, meth = name.split(".")
            fn = getattr(getattr(ev, cls), meth)
        else:
            fn = getattr(ev, name, None) or getattr(ex, name)
        assert _signature(fn) == want, name
    for name in ("find_nearest_point_idx", "uncertainty_pnp", "uncertainty_pnp_v2"):
        assert _signature(getattr(ex, name)) == expected[name]
