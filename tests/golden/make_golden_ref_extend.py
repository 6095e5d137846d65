"""Regenerates tests/golden/ref_extend.npz: the indices and masks the reference's own farthest_point_sampling.cpp and
mesh_rasterization.cpp return for the cases of tests/extend_cases.py.  The two files are compiled verbatim with the
reference's flags into oracle/_ref/libpvnet_refextend.so by oracle/extend.mk (its random start made an input by
oracle/ref_rand_shim.c); __graft_entry__.build() does that when PVNET_REFERENCE names a checkout:
    PVNET_REFERENCE=<path> python -c "import __graft_entry__ as g; g.build()"
    python tests/golden/make_golden_ref_extend.py
Runs on the CPU.  Arrays above 4 KB are stored as sha256 digests (tests/helpers.py _pack); the file is written with
fixed timestamps, so regenerating it reproduces it byte for byte.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from oracle import extend_oracle as eo
    from tests import extend_cases as ec
    from tests.helpers import GOLDEN
    if not eo.ref_available():
        sys.exit("oracle/_ref/libpvnet_refextend.so is missing: run build() with PVNET_REFERENCE set first")
    entries = ec.golden_entries(eo.ref_farthest_point_sampling, eo.ref_mesh_binary_rasterization)
    ec.write_npz(os.path.join(GOLDEN, "ref_extend.npz"), entries)
    print("wrote", len(entries), "entries")
