"""Regenerates tests/golden/ref_layer.npz and tests/golden/ref_vp.npz: the outputs of the reference's own CUDA
voting kernels that tests/test_gpu_reference_layer.py and the vanishing-point test of
tests/test_gpu_variants.py compare the oracle and the product against.  Needs a GPU and
oracle/_ref/libpvnet_refcuda.so, which __graft_entry__.build() compiles when PVNET_REFERENCE names a
checkout of the reference project:
    PVNET_REFERENCE=<path> python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_golden_ref.py
Runs those tests once in recording mode: every reference-side value is computed live, the tests'
assertions run against it, and each file is written when its module finishes.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import ref_cuda
    if not ref_cuda.available():
        sys.exit("oracle/_ref/libpvnet_refcuda.so is missing: run build() with PVNET_REFERENCE set first")
    env = dict(os.environ, PVNET_RECORD_REF_GOLDEN="1")
    sys.exit(subprocess.call([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider",
                              os.path.join(ROOT, "tests", "test_gpu_reference_layer.py"),
                              os.path.join(ROOT, "tests", "test_gpu_variants.py")
                              + "::test_vanishing_point_pair_bit_exact_vs_oracle_and_reference_kernels"],
                             cwd=ROOT, env=env))
