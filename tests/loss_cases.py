"""Seeded inputs of the validation-loss cases, shared by tests/golden/make_golden_net_utils.py (which feeds them to the
reference's own smooth_l1_loss / compute_precision_recall) and the tests that compare against its record,
tests/golden/ref_net_utils.npz."""
import numpy as np

# name -> (b, h, w, K, C, sigma, weights, special values in the predictions)
CASES = {
    "k9_s1_binary": (3, 48, 64, 9, 2, 1.0, "binary", False),
    "k9_s3_fractional": (3, 48, 64, 9, 2, 3.0, "fractional", False),
    "k9_s05_nan_inf": (3, 48, 64, 9, 2, 0.5, "binary", True),
    "k17_s1_c3_nan_inf": (2, 37, 53, 17, 3, 1.0, "fractional", True),
    "k17_s05_c3": (2, 37, 53, 17, 3, 0.5, "binary", False),
}


def case_inputs(name):
    """seg float32 [b,C,h,w], mask int64 [b,h,w], vertex_pred / vertex float32 [b,2K,h,w], weights float32
    [b,1,h,w], sigma.  Logits sit on a 0.25 grid so that argmax ties occur; vertex differences span both branches
    of the smooth-L1 for every sigma."""
    b, h, w, k, c, sigma, wkind, special = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    seg = (np.round(rng.normal(0, 1.5, (b, c, h, w)) * 4) / 4).astype(np.float32)
    mask = rng.integers(0, c, (b, h, w)).astype(np.int64)
    pred = rng.normal(0, 1.2, (b, 2 * k, h, w)).astype(np.float32)
    vertex = rng.normal(0, 1.0, (b, 2 * k, h, w)).astype(np.float32)
    fg = (mask > 0).astype(np.float32)[:, None]
    weights = fg if wkind == "binary" else (fg * rng.uniform(0, 1, fg.shape)).astype(np.float32)
    if special:
        for arr, vals in ((pred, (np.nan, np.inf, -np.inf)), (seg, (np.nan, np.inf, -np.inf))):
            flat = arr.reshape(-1)
            idx = rng.choice(flat.size, 60, replace=False)
            flat[idx] = np.array(vals, np.float32)[np.arange(60) % 3]
    return seg, mask, pred, vertex, weights, sigma


def canon_nan(a):
    """a as float32 numpy with every NaN replaced by one canonical NaN: the elementwise records compare values bit
    for bit and NaN positions only (the sign and payload of a NaN differ between CPU and GPU arithmetic)."""
    a = np.asarray(a.detach().cpu().numpy() if hasattr(a, "detach") else a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a)
