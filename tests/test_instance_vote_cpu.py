"""CPU: the centre search and instance split of `ransac_voting_center` (DESIGN.md section 29) as
oracle/instance_vote_oracle.py restates it -- accuracy on seeded scenes, its first round against the reference's
loop body, the exact fmaf and cosine, the device sampler's stream and the public signature."""
import inspect

import numpy as np
import pytest

from oracle import instance_vote_oracle as iv
from oracle import philox_oracle as px
from oracle import pvnet_oracle as po
from tests.instance_vote_cases import draw_center_idxs, instance_scene, match_ids

THRESH, MIN_NUM, I, HN = 0.99, 100, 8, 256

# (instances, seed, touching, sigma, least label agreement, largest centre error in px): the bounds are the
# oracle's own results on these seeds, rounded outwards.  A winner's inliers include the pixels of other
# instances whose direction passes within the inlier cone of its centre, and the refit over them moves the
# centre, so several instances are not split exactly even on noise-free fields.
SCENES = [
    (1, 11, False, 0.0, 1.0, 1e-3),
    (2, 1, True, 0.0, 0.9999, 0.1),
    (3, 2, False, 0.0, 0.997, 0.3),
    (5, 3, False, 0.0, 0.975, 1.7),
    (4, 4, True, 0.0, 0.985, 1.4),
    (3, 5, False, 0.03, 0.98, 0.35),
    (5, 6, True, 0.03, 0.955, 1.0),
]


@pytest.mark.parametrize("n,seed,touching,sigma,agree_min,err_max", SCENES)
def test_scene_accuracy(n, seed, touching, sigma, agree_min, err_max):
    sc = instance_scene(n, seed, sigma=sigma, touching=touching)
    r = iv.center_search(sc["mask"], sc["field"][:, :, -1], draw_center_idxs(1, I, HN, seed)[0], THRESH, MIN_NUM)
    assert r["num"] == n
    cen = r["centers"][:n]
    err = [np.min(np.hypot(*(sc["centers"] - c[None]).T)) for c in cen]
    assert max(err) <= err_max
    assert sorted({int(np.argmin(np.hypot(*(sc["centers"] - c[None]).T))) for c in cen}) == list(range(n))
    lab = match_ids(r["labels"], sc["gt"], cen, sc["centers"])
    fg = sc["mask"] > 0
    assert (lab[fg] == sc["gt"][fg]).mean() >= agree_min
    assert np.all(r["labels"][~fg] == 0)
    assert np.all(r["centers"][n:] == 0)


def _reference_round(mask_img, field_img, idxs_round, thresh):
    """The reference's loop body (ransac_voting_gpu.py:624-665) for one round, restated with the v3 kernels'
    oracle: compaction, hypotheses, the [hn,1,tn] inlier tensor, torch.max, the ratio update and the final
    vote for the best point."""
    cur_mask = po._byte_mask(mask_img)
    coords, direct = po.compact(cur_mask, np.asarray(field_img, np.float32)[:, :, None, :])
    tn = coords.shape[0]
    idxs = (idxs_round.view(np.uint32) % np.uint32(tn)).astype(np.int32)[:, None, :]
    hyp = po.generate_hypothesis_kernel(direct, coords, idxs)
    inl = po.voting_for_hypothesis_kernel(direct, coords, hyp, thresh)         # [hn,1,tn]
    counts = inl.astype(np.int64).sum(2)                                      # [hn,1]
    win = int(counts[:, 0].argmax())                                          # first max
    all_win_ratio, all_win_pts = np.float32(0), np.zeros((1, 2), np.float32)
    ratio = np.float32(counts[win, 0]) / np.float32(tn)
    if all_win_ratio < ratio:
        all_win_pts = hyp[win]
    all_inlier = po.voting_for_hypothesis_kernel(direct, coords, all_win_pts[None], thresh)[0, 0]
    return counts[:, 0], win, np.nonzero(all_inlier)[0]


@pytest.mark.parametrize("seed", [2, 6])
def test_first_round_equals_reference_loop_body(seed):
    sc = instance_scene(3, seed, sigma=0.03)
    idxs = draw_center_idxs(1, I, HN, seed)[0]
    r = iv.center_search(sc["mask"], sc["field"][:, :, -1], idxs, THRESH, MIN_NUM)
    counts, win, inliers = _reference_round(sc["mask"], sc["field"][:, :, -1], idxs[0], THRESH)
    np.testing.assert_array_equal(r["counts"][0], counts)
    assert r["win_idx"][0] == win
    np.testing.assert_array_equal(r["inliers"][0], inliers)


def test_stops():
    sc = instance_scene(2, 1)
    idxs = draw_center_idxs(1, I, HN, 1)[0]
    fg = int(sc["mask"].sum())
    r = iv.center_search(sc["mask"], sc["field"][:, :, -1], idxs, THRESH, fg + 1)       # fg < min_num
    assert r["num"] == 0 and r["tn"][0] == fg and np.all(r["labels"] == 0) and np.all(r["counts"] == 0)
    r = iv.center_search(sc["mask"], sc["field"][:, :, -1], idxs[:1], THRESH, MIN_NUM)  # more objects than I
    assert r["num"] == 1 and set(np.unique(r["labels"])) == {0, 1}
    empty = np.zeros_like(sc["mask"])
    r = iv.center_search(empty, sc["field"][:, :, -1], idxs, THRESH, MIN_NUM)
    assert r["num"] == 0 and np.all(r["tn"] == 0)
    # the second instance's pixels all remain, so a min_num above the first winner's count stops in round 0
    r = iv.center_search(sc["mask"], sc["field"][:, :, -1], idxs, THRESH, MIN_NUM)
    r2 = iv.center_search(sc["mask"], sc["field"][:, :, -1], idxs, THRESH, int(r["win_counts"][0]) + 1)
    assert r2["num"] == 0 and r2["win_counts"][0] == r["win_counts"][0]


def test_fmaf_is_single_rounding():
    rng = np.random.default_rng(0)
    a = rng.standard_normal(200000).astype(np.float32)
    b = rng.standard_normal(200000).astype(np.float32)
    c = rng.standard_normal(200000).astype(np.float32)
    got = iv.fmaf(a, b, c)
    from fractions import Fraction
    for i in range(0, 200000, 997):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        f = np.float32(float(exact))
        lo, hi = np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))
        best = min((lo, f, hi), key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.uint32)) & 1))
        assert got[i] == best
    # a sum that lies exactly half-way between two floats in fp64 but not exactly
    x = np.float32(1.0) + np.float32(2.0 ** -23)
    assert iv.fmaf(x, x, np.float32(-1.0)) == np.float32((float(x) * float(x) - 1.0))


def test_cosine_matches_inlier_predicate():
    sc = instance_scene(2, 1, sigma=0.03)
    coords, direct = po.compact(sc["mask"], sc["field"][:, :, -1:, :])
    hyp = np.array([[[200.3, 150.7]], [[401.1, 300.2]]], np.float32)
    inl = po.voting_for_hypothesis_kernel(direct, coords, hyp, THRESH)[:, 0]
    for h in range(2):
        valid, ang = iv.exact_cosine(direct[:, 0, 0], direct[:, 0, 1], coords[:, 0], coords[:, 1], *hyp[h, 0])
        np.testing.assert_array_equal(valid & (ang > np.float32(THRESH)), inl[h] != 0)


def test_device_stream_restatement():
    words = iv.device_center_idxs(1234, 7, 3, 4, 64)
    assert words.shape == (3, 4, 64, 2)
    r = px.draw(1234, 7, 2, iv.STREAM_CENTER, [3 * 64 + 5])[0]
    assert words[2, 3, 5, 0] == np.int32(np.uint32(r[0]).view(np.int32))
    assert words[2, 3, 5, 1] == np.int32(np.uint32(r[1]).view(np.int32))
    assert iv.STREAM_CENTER not in (px.STREAM_SELECTION, px.STREAM_V3, px.STREAM_COV)


def test_positional_signature_is_the_reference():
    # ransac_voting_gpu.py:600 of the reference, transcribed
    expected = ("mask, vertex, round_hyp_num, inlier_thresh=0.99, confidence=0.999, max_iter=20, min_num=100")
    import lib.ransac_voting_gpu_layer.ransac_voting_gpu as shim
    parts = []
    for p in inspect.signature(shim.ransac_voting_center).parameters.values():
        if p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD:
            parts.append(p.name if p.default is inspect.Parameter.empty else f"{p.name}={p.default!r}")
    assert ", ".join(parts) == expected
