"""Regenerates tests/golden/ref_nn.npz: the indices the reference's own nearest-point kernel
(lib/utils/extend_utils/src/nearest_neighborhood.cu, compiled verbatim into oracle/_ref/libpvnet_refnn.so by
oracle/eval.mk) returns for the inputs of the search test in tests/test_gpu_eval.py.  Needs a GPU and that library,
which __graft_entry__.build() compiles when PVNET_REFERENCE names a checkout of the reference project:
    PVNET_REFERENCE=<path> python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_golden_ref_nn.py
Runs that test once in recording mode: the reference kernel's indices are computed live, the test's assertions run
against them, and the file is written when the module finishes.  Arrays above 4 KB are stored as sha256 digests.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import eval_oracle
    if not eval_oracle.ref_nn_available():
        sys.exit("oracle/_ref/libpvnet_refnn.so is missing: run build() with PVNET_REFERENCE set first")
    env = dict(os.environ, PVNET_RECORD_REF_GOLDEN="1")
    sys.exit(subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider",
                              os.path.join(ROOT, "tests", "test_gpu_eval.py") + "::test_nearest_point_idx_bit_exact"],
                             cwd=ROOT, env=env))
