"""GPU: the product and the oracle against the outputs of the reference's OWN CUDA kernels
(ransac_voting_kernel.cu compiled verbatim by oracle/Makefile into oracle/_ref, run through the
reference layer's own torch orchestration in oracle/ref_cuda.py).  Those outputs are stored in
tests/golden/ref_layer.npz (tests/golden/make_golden_ref.py records them on a GPU where
oracle/_ref is built), so every run compares against them without the reference.  This is what pins
the oracle (SURVEY.md §8c) and what measures "within 1e-4 of the reference CUDA layer"."""
import numpy as np
import pytest
import torch

from oracle import pvnet_oracle as po
from pvnet_b200 import ransac_voting_gpu as rv
from pvnet_b200 import synthetic as syn
from tests.helpers import RefGolden, cfg1_inputs, demo_fixture, reference_kernels, same_as_stored

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
_gold = RefGolden("ref_layer.npz")


@pytest.fixture(scope="module", autouse=True)
def _write_golden():
    yield
    _gold.save()


def _dev_inputs(mask_np, field_np):
    mask = torch.from_numpy(np.ascontiguousarray(mask_np)).to(DEV)
    ver = torch.from_numpy(np.ascontiguousarray(field_np)).to(DEV)
    b, c2, h, w = ver.shape
    return mask, ver.permute(0, 2, 3, 1).view(b, h, w, c2 // 2, 2)


@pytest.mark.parametrize("kind", ["random", "planted"])
def test_reference_kernels_pin_the_oracle(kind):
    mask, field, idxs = cfg1_inputs(kind)
    coords, direct = po.compact(mask.astype(np.uint8), syn.as_reference_view(field[None])[0])
    d, c, i = (torch.from_numpy(a).to(DEV) for a in (direct, coords, idxs))

    def reference():
        rc = reference_kernels()
        hyp = rc.generate_hypothesis(d, c, i)
        inl = torch.zeros([128, 9, 10000], dtype=torch.uint8, device=DEV)
        rc.voting_for_hypothesis(d, c, hyp, inl, 0.99)
        return {"hyp": hyp, "counts": inl.sum(2).to(torch.int32), "inl8": inl[:8]}
    ref = _gold.get(f"pin_{kind}", reference, exact=("hyp", "counts", "inl8"))
    ohyp = po.generate_hypothesis_kernel(direct, coords, idxs)
    assert same_as_stored(ohyp, ref["hyp"])
    assert same_as_stored(po.vote_counts(direct, coords, ohyp, 0.99).astype(np.int32), ref["counts"])
    assert same_as_stored(po.voting_for_hypothesis_kernel(direct, coords, ohyp[:8], 0.99).astype(np.uint8), ref["inl8"])


def test_reference_kernels_pin_the_oracle_on_edge_values():
    rng = np.random.default_rng(0)
    tn, vn, hn = 4096, 3, 64
    direct = rng.standard_normal((tn, vn, 2)).astype(np.float32)
    direct[:200] *= 1e-6            # around the 1e-6 norm test
    direct[200:300] = 0
    direct[300:400, :, 1] = direct[300:400, :, 0]          # near-parallel families
    coords = np.stack([rng.integers(0, 640, tn), rng.integers(0, 480, tn)], 1).astype(np.float32)
    idxs = rng.integers(0, tn, (hn, vn, 2), dtype=np.int32)
    d, c, i = (torch.from_numpy(a).to(DEV) for a in (direct, coords, idxs))
    ohyp = po.generate_hypothesis_kernel(direct, coords, idxs)
    # also hypotheses ON pixels (norm2 == 0) and far away
    extra = np.concatenate([coords[:32, None, :].repeat(vn, 1), np.full((8, vn, 2), 3e7, np.float32)]).astype(np.float32)
    cases = [(thresh, j, hp) for thresh in (0.99, 0.5, -0.25) for j, hp in enumerate((ohyp, extra))]

    def reference():
        rc = reference_kernels()
        out = {"hyp": rc.generate_hypothesis(d, c, i)}
        for thresh, j, hp in cases:
            inl = torch.zeros([hp.shape[0], vn, tn], dtype=torch.uint8, device=DEV)
            rc.voting_for_hypothesis(d, c, torch.from_numpy(hp).to(DEV), inl, thresh)
            out[f"inl_{thresh}_{j}"] = inl
        return out
    ref = _gold.get("edge", reference, exact=["hyp"] + [f"inl_{t}_{j}" for t, j, _ in cases])
    assert same_as_stored(ohyp, ref["hyp"])
    for thresh, j, hp in cases:
        assert same_as_stored(po.voting_for_hypothesis_kernel(direct, coords, hp, thresh).astype(np.uint8), ref[f"inl_{thresh}_{j}"])


def _product_vs_reference_layer(mask_np, field_np, hn, thresh, max_num=30000, label=""):
    """Runs the reference layer (its own kernels + its torch ops, fp32 refit), the same
    with the refit ops in fp64, and the product, all from torch.manual_seed(0).
    Asserts fixed-seed parity of samples / hypotheses / counts, and that the product is
    within 1e-4 of the reference layer once the reference's fp32 refit rounding is taken
    out (fp64 run).  Returns the gaps."""
    mask, vertex = _dev_inputs(mask_np, field_np)

    def reference():
        rc = reference_kernels()
        rec = []
        torch.manual_seed(0)
        out = {"kp": rc.layer_v3(mask, vertex, hn, inlier_thresh=thresh, max_num=max_num, record=rec)}
        torch.manual_seed(0)
        out["kp64"] = rc.layer_v3(mask, vertex, hn, inlier_thresh=thresh, max_num=max_num, refit_dtype=torch.float64)
        for bi, r in enumerate(rec):
            out[f"rec{bi}"] = np.array(r is not None)
            if r is not None:
                out.update({f"idxs{bi}": r["idxs"], f"tn{bi}": np.array(r["tn"]), f"counts{bi}": r["counts"],
                            f"hyp{bi}": r["hyp"]})
        return out
    ref = _gold.get(label, reference, exact=[f"{n}{bi}" for n in ("idxs", "counts", "hyp") for bi in range(mask.shape[0])])
    torch.manual_seed(0)
    kp, dbg = rv.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, max_num=max_num, return_debug=True)
    for bi in range(mask.shape[0]):
        if not ref.get(f"rec{bi}", False):
            continue
        # fixed-seed parity: same samples drawn, same counts, same winner
        assert same_as_stored(dbg["idxs"][bi], ref[f"idxs{bi}"]), "RNG stream differs from the reference's"
        assert int(dbg["tn"][bi]) == int(ref[f"tn{bi}"])
        assert same_as_stored(dbg["counts"][bi].long(), ref[f"counts{bi}"]), "inlier counts differ from the reference layer"
        assert same_as_stored(dbg["hyp"][bi], ref[f"hyp{bi}"])
    ref_kp, ref_kp64 = ref["kp"], ref["kp64"]
    kp = kp.cpu().numpy()
    gap32 = np.abs(kp - ref_kp).max()
    gap64 = np.abs(kp - ref_kp64).max()
    noise = np.abs(ref_kp - ref_kp64).max()
    print(f"\n[reference-layer gap] {label}: |ours - ref(fp32 refit)| = {gap32:.3e}; "
          f"|ours - ref(fp64 refit)| = {gap64:.3e}; reference's own fp32 noise |ref32 - ref64| = {noise:.3e}")
    assert gap64 <= 1e-4, "product differs from the reference layer beyond its fp32 refit rounding"
    # and the distance to the STOCK fp32 reference is explained by that rounding noise, not hidden behind it
    assert gap32 <= 1.5 * noise + 1e-5, (gap32, noise)
    return gap32, gap64, noise


def test_fixed_seed_parity_with_reference_layer_config1():
    mask, field, _ = cfg1_inputs("planted")
    _product_vs_reference_layer(np.stack([mask, mask]), np.stack([field, field]), 128, 0.99,
                                label="config1 planted, tn=10000, K=9 (odd keypoints 260 px outside the mask)")


def test_fixed_seed_parity_with_reference_layer_demo():
    """The reference's own demo fixture (well conditioned: keypoints inside the object)."""
    mask, field, pts = demo_fixture()
    gap32, _, _ = _product_vs_reference_layer(mask[None], field[None], 512, 0.99, label="demo fixture, tn=2289")
    assert gap32 <= 1e-3


def test_fixed_seed_parity_near_keypoints():
    """Keypoints inside the mask (R=20 px): the best-conditioned case."""
    mask = syn.disc_mask(3000)
    rng = np.random.default_rng(5)
    kps = np.stack([320 + 20 * np.cos(np.arange(9)), 240 + 20 * np.sin(np.arange(9))], 1)
    ys, xs = np.mgrid[0:480, 0:640].astype(np.float64)
    field = np.zeros((18, 480, 640), np.float32)
    for j in range(9):
        dx, dy = kps[j, 0] - xs, kps[j, 1] - ys
        n = np.sqrt(dx * dx + dy * dy) + 1e-3
        eps = rng.normal(0, 0.03, size=dx.shape)
        field[2 * j] = (np.cos(eps) * dx / n - np.sin(eps) * dy / n) * (mask != 0)
        field[2 * j + 1] = (np.sin(eps) * dx / n + np.cos(eps) * dy / n) * (mask != 0)
    gap32, _, _ = _product_vs_reference_layer(mask[None], field[None], 256, 0.99, label="near keypoints, tn=3000")
    assert gap32 <= 1e-3


def test_fixed_seed_parity_with_subsampling():
    masks = np.stack([syn.disc_mask(40000), syn.disc_mask(3), syn.disc_mask(9000)])
    fields = np.stack([syn.planted_field(masks[i], 9, 40 + i)[0] for i in range(3)])
    _product_vs_reference_layer(masks, fields, 256, 0.99, max_num=30000, label="subsampled 40000->~30000")


def test_covariance_fixed_seed_parity():
    masks = np.stack([syn.disc_mask(7000), syn.disc_mask(12000)])
    fields = np.stack([syn.planted_field(masks[i], 9, 60 + i, sigma=0.05)[0] for i in range(2)])
    mask, vertex = _dev_inputs(masks, fields)
    torch.manual_seed(1)
    mean = rv.ransac_voting_layer_v3(mask, vertex, 256, inlier_thresh=0.99)
    ref = _ref_cov("cov_parity", mask, vertex, mean, dict(round_hyp_num=128, min_hyp_num=512, inlier_thresh=0.99), 2)
    torch.manual_seed(2)
    _, cov, dbg = rv.estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=128, min_hyp_num=512,
                                                            inlier_thresh=0.99, return_debug=True)
    for bi in range(mask.shape[0]):
        if f"idxs{bi}" not in ref:
            continue
        assert same_as_stored(dbg["idxs"][bi], ref[f"idxs{bi}"])
        assert same_as_stored(dbg["counts"][bi].long(), ref[f"counts{bi}"])
    ref_cov = torch.from_numpy(ref["cov"]).to(DEV)
    gap = (cov - ref_cov).abs()
    print(f"\n[reference-layer gap] covariance: max abs {gap.max().item():.3e}, "
          f"max rel {(gap / ref_cov.abs().clamp_min(1e-6)).max().item():.3e}, |cov| max {ref_cov.abs().max().item():.3e}")
    assert torch.allclose(cov, ref_cov, atol=1e-4, rtol=1e-4)


def _ref_cov(key, mask, vertex, mean, kw, seed):
    """reference layer estimate_voting_distribution_with_mean under torch.manual_seed(seed): covariances and,
    per image, the recorded samples and counts"""
    def reference():
        rec = []
        torch.manual_seed(seed)
        _, cov = reference_kernels().layer_cov_with_mean(mask, vertex, mean, record=rec, **kw)
        out = {"cov": cov}
        for bi, r in enumerate(rec):
            out.update({f"idxs{bi}": r["idxs"], f"counts{bi}": r["counts"]})
        return out
    return _gold.get(key, reference, exact=[f"{n}{bi}" for n in ("idxs", "counts") for bi in range(mask.shape[0])])


def _cov_vs_reference_layer(masks, fields, hn, min_hyp, thresh, max_num, seed):
    mask, vertex = _dev_inputs(masks, fields)
    torch.manual_seed(seed)
    mean = rv.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=thresh, max_num=max_num)
    ref = _ref_cov(f"cov_{seed}", mask, vertex, mean,
                   dict(round_hyp_num=hn, min_hyp_num=min_hyp, inlier_thresh=thresh, max_num=max_num), seed + 1)
    torch.manual_seed(seed + 1)
    _, cov, dbg = rv.estimate_voting_distribution_with_mean(mask, vertex, mean, round_hyp_num=hn, min_hyp_num=min_hyp,
                                                            inlier_thresh=thresh, max_num=max_num, return_debug=True)
    for bi in range(mask.shape[0]):
        if f"idxs{bi}" not in ref:
            continue
        assert same_as_stored(dbg["idxs"][bi], ref[f"idxs{bi}"]), "RNG stream differs from the reference's"
        assert same_as_stored(dbg["counts"][bi].long(), ref[f"counts{bi}"]), "inlier counts differ from the reference layer"
    ref_cov = torch.from_numpy(ref["cov"]).to(DEV)
    assert torch.allclose(cov, ref_cov, atol=1e-4, rtol=1e-4), (cov - ref_cov).abs().max().item()


def test_config4_shape_fixed_seed_vs_reference_layer():
    """BASELINE config 4 per image (K=9, 20000 px, v3(256) + with_mean(256, 4096), thresh 0.99) against the reference's
    own kernels + torch ops under the same torch seed: samples, counts, keypoints, covariances."""
    masks = np.stack([syn.disc_mask(20000)])
    fields = np.stack([syn.planted_field(masks[0], 9, 4400, sigma=0.05)[0]])
    _product_vs_reference_layer(masks, fields, 256, 0.99, label="config 4 shape, tn=20000, K=9, 256 hyp")
    _cov_vs_reference_layer(masks, fields, 256, 4096, 0.99, 30000, seed=44)


def test_config5_shape_fixed_seed_vs_reference_layer():
    """BASELINE config 5 per image (K=17, 92160 px subsampled to ~30000 by the reference's own uniform_ draw,
    v3(1024) + with_mean(1024, 1024))."""
    masks = np.stack([syn.disc_mask(92160)])
    fields = np.stack([syn.planted_field(masks[0], 17, 5500, sigma=0.05)[0]])
    _product_vs_reference_layer(masks, fields, 1024, 0.99, max_num=30000, label="config 5 shape, 92160 px -> ~30000, K=17, 1024 hyp")
    _cov_vs_reference_layer(masks, fields, 1024, 1024, 0.99, 30000, seed=55)
