"""Seeded inputs of the vertex-target cases, shared by tests/golden/make_golden_vertex_targets.py (which feeds them to
the reference's own compute_vertex_hcoords) and the tests that compare against its record,
tests/golden/ref_vertex_targets.npz."""
import numpy as np

# name -> (b, h, w, K, mask dtype, hcoords dtype, hw kind, special keypoints, use_motion)
#   hw kind: "one" (hw = 1, tools/demo.py's case), "zero" (vanishing points, VotingType.VanPts), "other" (a
#   perspective-like hw in [0.5, 2)), "mixed" (each keypoint one of the three)
CASES = {
    "k1_i64_f64": (2, 37, 53, 1, "int64", "float64", "one", False, False),
    "k8_i32_f32": (2, 48, 64, 8, "int32", "float32", "other", False, False),
    "k9_u8_f64": (3, 37, 53, 9, "uint8", "float64", "one", False, False),
    "k9_i64_f32_motion": (2, 37, 53, 9, "int64", "float32", "other", False, True),
    "k17_bool_f64_hw0": (2, 41, 60, 17, "bool", "float64", "zero", False, False),
    "k17_i64_f64_mixed": (2, 40, 67, 17, "int64", "float64", "mixed", False, False),
    "k21_i64_f64_special": (2, 37, 53, 21, "int64", "float64", "one", True, False),
    "k21_i32_f32_special": (2, 37, 53, 21, "int32", "float32", "mixed", True, False),
    "k21_u8_f64_special_motion": (1, 37, 53, 21, "uint8", "float64", "mixed", True, True),
    "k9_b16_480x640": (16, 480, 640, 9, "int64", "float64", "other", False, False),
}

MASK_DTYPES = {"int64": np.int64, "int32": np.int32, "uint8": np.uint8, "bool": np.bool_}


def _special(rng, mask, hc, hw_kind):
    """Keypoints the plain draw would never give: exactly on a foreground pixel centre, within 1e-3 of one, at +-1e6,
    and NaN / +-inf in each coordinate."""
    ys, xs = np.nonzero(mask == 1)
    K = hc.shape[0]
    for k in range(K):
        kind = k % 7
        i = rng.integers(len(ys))
        x, y = float(xs[i]), float(ys[i])
        hw = 1.0 if hw_kind == "one" or kind < 2 else hc[k, 2]
        if kind == 0:                                       # on a pixel centre: 0 / 1e-3 = 0
            hc[k] = (x, y, 1.0)
        elif kind == 1:                                     # within 1e-3 of a pixel centre
            hc[k] = (x + rng.uniform(-6e-4, 6e-4), y + rng.uniform(-6e-4, 6e-4), 1.0)
        elif kind == 2:
            hc[k, :2] = rng.choice([-1e6, 1e6], 2) * max(hw, 1.0)
        elif kind == 3:
            hc[k, rng.integers(3)] = np.nan
        elif kind == 4:
            hc[k, rng.integers(3)] = np.inf
        elif kind == 5:
            hc[k, rng.integers(3)] = -np.inf
    return hc


def case_inputs(name):
    """mask [b,h,w] of the case's dtype with values in {0, 1, 2} ({0, 1} for bool; only 1 is foreground),
    hcoords [b,K,3] of the case's dtype, use_motion."""
    b, h, w, K, mdt, hdt, hw_kind, special, motion = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    if mdt == "bool":
        mask = rng.random((b, h, w)) < 0.5
    else:
        mask = rng.choice(np.array([0, 1, 2], MASK_DTYPES[mdt]), (b, h, w), p=[0.4, 0.45, 0.15])
    hc = np.empty((b, K, 3), np.float64)
    for i in range(b):
        kinds = [hw_kind] * K if hw_kind != "mixed" else list(rng.choice(["one", "zero", "other"], K))
        for k, kind in enumerate(kinds):
            X, Y = rng.uniform(-0.2 * w, 1.2 * w), rng.uniform(-0.2 * h, 1.2 * h)
            if kind == "one":
                hc[i, k] = (X, Y, 1.0)
            elif kind == "zero":
                hc[i, k] = (rng.normal(), rng.normal(), 0.0)
            else:
                hw = rng.uniform(0.5, 2.0)
                hc[i, k] = (X * hw, Y * hw, hw)
        if special:
            hc[i] = _special(rng, mask[i], hc[i], hw_kind)
    return mask, hc.astype(np.float32 if hdt == "float32" else np.float64), motion


def canon_nan(a):
    """a as float32 numpy with every NaN replaced by one canonical NaN (the sign and payload of a NaN differ between
    CPU and GPU arithmetic; the records compare values bit for bit and NaN positions only)."""
    a = np.asarray(a.detach().cpu().numpy() if hasattr(a, "detach") else a, np.float32)
    return np.where(np.isnan(a), np.float32(np.nan), a)
