"""Regenerates tests/golden/ref_variants.npz by running the REFERENCE'S OWN Python functions.

Needs PVNET_REFERENCE = a checkout of the reference project:  python tests/golden/make_golden_variants.py

lib/ransac_voting_gpu_layer/ransac_voting_gpu.py is imported unmodified from the reference project
with its compiled extension `ransac_voting` replaced by a stub whose two functions call the
oracle's C kernels (oracle/pvnet_oracle.c -- pinned bit-exactly against the reference's CUDA
kernels by tests/test_gpu_reference_layer.py) on CPU tensors.  The stub also records every
`idxs` tensor the reference draws, so the same samples can be injected into the oracle and
into the CUDA path.  Functions that still run under torch 2.11 on the CPU:

  ransac_voting_layer (v1, :10)            bool masks  -> runs
  ransac_voting_layer_v2 (:99)             bool masks, pinverse refit -> runs (uint8 indexing still accepted)
  ransac_voting_hypothesis (:218)          bool masks  -> runs
  estimate_voting_distribution (:263)      bool masks  -> runs
  ransac_motion_voting (:960)              indexes with a uint8 mask -> runs only if torch still
                                           accepts it; otherwise the fixture omits it
  v3/v4/v5 use masked_select with a uint8 mask (rejected by torch >= 1.2) and torch.gesv: they
  are pinned through oracle/ref_cuda.py instead.

Inputs are small (64 x 80 image, K = 5) so that the fixture stays a few KB; they are rebuilt
in the tests from the stored seeds.
"""
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.helpers import reference_root  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import pvnet_oracle as po  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import VARIANT_HWK, variant_inputs as make_inputs  # noqa: E402

H, W, K = VARIANT_HWK


def import_reference():
    recorded = []
    stub = types.ModuleType("lib.ransac_voting_gpu_layer.ransac_voting")

    def generate_hypothesis(direct, coords, idxs):
        recorded.append(idxs.numpy().copy())
        return torch.from_numpy(po.generate_hypothesis_kernel(direct.numpy(), coords.numpy(), idxs.numpy()))

    def voting_for_hypothesis(direct, coords, hyp, inlier, thresh):
        inlier.copy_(torch.from_numpy(po.voting_for_hypothesis_kernel(direct.numpy(), coords.numpy(), hyp.numpy(),
                                                                      np.float32(thresh))))

    stub.generate_hypothesis = generate_hypothesis
    stub.voting_for_hypothesis = voting_for_hypothesis
    for name in ("lib", "lib.ransac_voting_gpu_layer"):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(reference_root(), *name.split("."))]
        sys.modules[name] = m
    sys.modules["lib.ransac_voting_gpu_layer.ransac_voting"] = stub
    sys.modules["lib.ransac_voting_gpu_layer"].ransac_voting = stub
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "lib.ransac_voting_gpu_layer.ransac_voting_gpu",
        os.path.join(reference_root(), "lib", "ransac_voting_gpu_layer", "ransac_voting_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, recorded


def main():
    ref, rec = import_reference()
    out = {"hwk": np.array([H, W, K])}

    # ---- v1: two object classes
    mask, vertex, _ = make_inputs(11, n_fg=1200, classes=2)
    torch.manual_seed(1)
    del rec[:]
    r = ref.ransac_voting_layer(torch.from_numpy(mask), torch.from_numpy(vertex), 3, 32, inlier_thresh=0.99)
    # idxs is drawn once per (image, class); later rounds re-use it, so keep the first of each run
    uniq = []
    for a in rec:
        if not uniq or not np.array_equal(uniq[-1], a):
            uniq.append(a)
    assert len(uniq) == 2, len(uniq)
    out["v1_seed"] = np.array([11, 1200, 2])
    out["v1_idxs"] = np.stack(uniq)                       # [class, hn, K, 2]
    out["v1_out"] = r.numpy()
    print("v1", r.shape, r[0, :, 0].tolist())

    # ---- v2: two classes, two refinement rounds (pinverse refit, :178-204)
    mask, vertex, _ = make_inputs(15, n_fg=1000, classes=2)
    torch.manual_seed(5)
    del rec[:]
    try:
        r2 = ref.ransac_voting_layer_v2(torch.from_numpy(mask), torch.from_numpy(vertex), 3, 32, inlier_thresh=0.99,
                                        refine_iter_num=2)
        uniq = []
        for a in rec:
            if not uniq or not np.array_equal(uniq[-1], a):
                uniq.append(a)
        assert len(uniq) == 2, len(uniq)
        out["v2_seed"] = np.array([15, 1000, 2])
        out["v2_idxs"] = np.stack(uniq)
        out["v2_out"] = r2.numpy()
        print("v2", r2.shape, r2[0, :, 0].tolist())
    except Exception as e:
        print("ransac_voting_layer_v2 does not run under this torch:", type(e).__name__, str(e)[:120])

    # ---- ransac_voting_hypothesis
    mask, vertex, _ = make_inputs(12, n_fg=700)
    torch.manual_seed(2)
    del rec[:]
    hyp, cnt = ref.ransac_voting_hypothesis(torch.from_numpy(mask), torch.from_numpy(vertex), 48, inlier_thresh=0.99)
    out["hyp_seed"] = np.array([12, 700, 1])
    out["hyp_idxs"] = rec[0]
    out["hyp_out"] = hyp.numpy()
    out["hyp_counts"] = cnt.numpy()
    print("hypothesis", hyp.shape, cnt.dtype, int(cnt.max()))

    # ---- estimate_voting_distribution: 3 rounds of 32, top 24
    mask, vertex, _ = make_inputs(13, n_fg=800)
    torch.manual_seed(3)
    del rec[:]
    mean, cov = ref.estimate_voting_distribution(torch.from_numpy(mask), torch.from_numpy(vertex), round_hyp_num=32,
                                                 min_hyp_num=96, topk=24, inlier_thresh=0.99)
    out["dist_seed"] = np.array([13, 800, 1])
    out["dist_idxs"] = np.stack(rec)                      # [rounds, hn, K, 2]
    out["dist_mean"] = mean.numpy()
    out["dist_cov"] = cov.numpy()
    print("distribution", mean[0, 0].tolist(), cov[0, 0].tolist())

    # ---- ransac_motion_voting
    mask, vertex, _ = make_inputs(14, n_fg=500)
    try:
        pts = ref.ransac_motion_voting(torch.from_numpy(mask), torch.from_numpy(vertex))
        out["motion_seed"] = np.array([14, 500, 1])
        out["motion_out"] = pts.numpy()
        print("motion", pts[0, :2].tolist())
    except Exception as e:        # uint8 mask indexing removed from torch
        print("ransac_motion_voting does not run under this torch:", type(e).__name__, str(e)[:80])

    np.savez_compressed(os.path.join(HERE, "ref_variants.npz"), **out)
    print("wrote ref_variants.npz", sorted(out))


if __name__ == "__main__":
    main()
