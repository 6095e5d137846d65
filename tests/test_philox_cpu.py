"""CPU tests of oracle/philox_oracle.py, the restatement of the voting layer's device-side sampler
(`rng="device"`) that tests/test_gpu_device_sampler.py holds the kernels to: Random123's published
Philox4x32-10 known answers, the vectorised form against a scalar loop, the counter and key layout, and
`device_samples` at its edges (nothing drawn below min_num, nothing left after subsampling, fg == max_num)."""
import numpy as np
import pytest

from oracle import philox_oracle as px
from oracle import pvnet_oracle as po
from pvnet_b200 import synthetic as syn

M32 = 0xFFFFFFFF


def _philox_scalar(ctr, key):
    """Philox4x32-10 one counter at a time in Python integers."""
    c, k = [int(v) for v in ctr], [int(v) for v in key]
    for r in range(10):
        if r:
            k = [(k[0] + 0x9E3779B9) & M32, (k[1] + 0xBB67AE85) & M32]
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & M32, (p0 >> 32) ^ c[3] ^ k[1], p0 & M32]
    return c


# Random123 1.09, kat_vectors: philox4x32 10
KAT = [
    ([0, 0, 0, 0], [0, 0], [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]),
    ([M32] * 4, [M32] * 2, [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]),
    ([0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344], [0xA4093822, 0x299F31D0],
     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]),
]


@pytest.mark.parametrize("ctr,key,expect", KAT, ids=["zeros", "ones", "pi"])
def test_known_answer_vectors(ctr, key, expect):
    assert px.philox4x32_10(ctr, key).tolist() == expect
    assert _philox_scalar(ctr, key) == expect


def test_vectorised_equals_scalar_loop():
    rng = np.random.default_rng(0)
    ctr = rng.integers(0, 2 ** 32, (300, 4), dtype=np.uint64)
    key = rng.integers(0, 2 ** 32, (300, 2), dtype=np.uint64)
    ctr[:10] = M32 - np.arange(10)[:, None]          # words near 2^32: the 32x32-bit products at their largest
    got = px.philox4x32_10(ctr, key)
    assert got.dtype == np.uint32 and got.shape == (300, 4)
    for i in range(300):
        assert got[i].tolist() == _philox_scalar(ctr[i], key[i]), i
    # one key broadcast over many counters
    got = px.philox4x32_10(ctr, key[7])
    assert all(got[i].tolist() == _philox_scalar(ctr[i], key[7]) for i in range(300))


def test_counter_and_key_layout():
    """counter (item, image | stream << 28, offset low, offset high), key (seed low, seed high)."""
    seed, offset = (0x1234 << 32) | 0x89ABCDEF, (5 << 32) | 0xFFFFFFF0
    for image, stream, item in [(0, 0, 0), (3, 1, 77), (1023, 2, 12345)]:
        want = _philox_scalar([item, image | stream << 28, offset & M32, offset >> 32], [seed & M32, seed >> 32])
        assert px.draw(seed, offset, image, stream, [item])[0].tolist() == want
    # every word of the seed and the offset reaches the draw, and the three streams are distinct
    items = np.arange(64)
    base = px.draw(seed, offset, 3, 1, items)
    for s, o, im, st in [(seed ^ (1 << 40), offset, 3, 1), (seed, offset ^ (1 << 33), 3, 1),
                         (seed, offset, 3, 2), (seed, offset, 3, 0), (seed, offset, 4, 1)]:
        assert not np.array_equal(px.draw(s, o, im, st, items), base)


def test_selection_values_are_24_bit_fractions():
    seed, offset = 99, 3
    x = px.draw(seed, offset, 2, px.STREAM_SELECTION, np.arange(4096))[:, 0]
    sel = px.selection_values(seed, offset, 2, 4096)
    assert sel.dtype == np.float32
    assert np.array_equal((sel * np.float32(2 ** 24)).astype(np.uint32), x & 0xFFFFFF)
    assert sel.min() >= 0 and sel.max() < 1


def _masks(ns, h=24, w=32):
    return np.stack([syn.disc_mask(n, h, w, center=(w // 2, h // 2)) for n in ns])


def test_device_samples_layout_and_subsampling():
    ns = [0, 3, 200, 700]
    masks = _masks(ns)
    seed, offset, hn, vn, hnt = 2 ** 40 + 5, 2 ** 32 + 7, 16, 3, 32
    ds = px.device_samples(masks, "nonzero", seed, offset, hn, vn, hnt, 5, 500)
    assert ds["idxs"].shape == (4, hn, vn, 2) and ds["idxs"].dtype == np.int32
    assert ds["cov_idxs"].shape == (4, hnt, vn, 2) and ds["selection"].shape == (4, 24, 32)
    # images 0 and 1 are below min_num: nothing drawn
    assert ds["tn"][0] == 0 and ds["tn"][1] == 0
    assert not ds["idxs"][:2].any() and not ds["cov_idxs"][:2].any()
    assert ds["tn"][2] == 200                                   # fg <= max_num: every pixel kept
    p = po.subsample_probability(500, 700)
    kept = (masks[3] != 0) & (ds["selection"][3] < p)
    assert ds["tn"][3] == kept.sum() and 0 < ds["tn"][3] < 700
    # item h*vn + k of stream 1 (v3) / stream 2 (covariance), words x and y, as int32 bit patterns
    for bi in (2, 3):
        for h, k in [(0, 0), (5, 2), (hn - 1, vn - 1)]:
            w = _philox_scalar([h * vn + k, bi | 1 << 28, offset & M32, offset >> 32], [seed & M32, seed >> 32])
            assert ds["idxs"][bi, h, k].view(np.uint32).tolist() == w[:2]
        w = _philox_scalar([(hnt - 1) * vn + 1, bi | 2 << 28, offset & M32, offset >> 32], [seed & M32, seed >> 32])
        assert ds["cov_idxs"][bi, hnt - 1, 1].view(np.uint32).tolist() == w[:2]
        sel = _philox_scalar([37, bi, offset & M32, offset >> 32], [seed & M32, seed >> 32])[0] & 0xFFFFFF
        assert ds["selection"][bi].ravel()[37] == np.float32(sel * 2.0 ** -24)
    red = px.reduce(ds["idxs"], ds["tn"])
    assert red[0] is None and red[1] is None
    assert red[3].min() >= 0 and red[3].max() < ds["tn"][3]
    assert np.array_equal(red[3], (ds["idxs"][3].view(np.uint32) % ds["tn"][3]).astype(np.int32))
    assert px.device_samples(masks, "nonzero", seed, offset, hn, vn, 0, 5, 500)["cov_idxs"] is None
    # min_num is tested before max_num: an image below min_num is skipped even when it is above max_num
    assert px.device_samples(masks[3:], "nonzero", seed, offset, hn, vn, 0, 800, 500)["tn"][0] == 0


def test_device_samples_tn_zero_after_subsampling():
    """fg > max_num and every foreground pixel dropped: tn == 0 and nothing is drawn."""
    masks = _masks([2])
    offs = [o for o in range(64)
            if px.device_samples(masks, "nonzero", 11, o, 4, 1, 8, 1, 1)["tn"][0] == 0]
    assert offs, "no offset in [0, 64) drops both pixels at p = 0.5"
    ds = px.device_samples(masks, "nonzero", 11, offs[0], 4, 1, 8, 1, 1)
    assert (ds["selection"][0][masks[0] != 0] >= np.float32(0.5)).all()
    assert not ds["idxs"].any() and not ds["cov_idxs"].any()


def test_device_samples_fg_equal_max_num_is_not_subsampled():
    masks = _masks([9])
    p = po.subsample_probability(8, 9)
    for off in range(32):
        at = px.device_samples(masks, "nonzero", 5, off, 4, 1, 0, 5, 9)
        assert at["tn"][0] == 9                                  # fg == max_num keeps every pixel
        above = px.device_samples(masks, "nonzero", 5, off, 4, 1, 0, 5, 8)
        fg_sel = at["selection"][0][masks[0] != 0]
        assert above["tn"][0] == (fg_sel < p).sum()
    assert any(px.device_samples(masks, "nonzero", 5, o, 4, 1, 0, 5, 8)["tn"][0] < 9 for o in range(32))


def test_device_samples_mask_modes():
    """"nonzero" reads `.byte()` (2 counts, 256 does not); "equals_one" reads value == 1."""
    m = _masks([300])
    ys, xs = np.nonzero(m[0])
    m[0, ys[:100], xs[:100]] = 2
    m[0, ys[100:120], xs[100:120]] = 256
    a = px.device_samples(m, "nonzero", 1, 0, 4, 1, 0, 5, 10 ** 6)
    b = px.device_samples(m, "equals_one", 1, 0, 4, 1, 0, 5, 10 ** 6)
    assert a["tn"][0] == 280 and b["tn"][0] == 180
    assert np.array_equal(a["idxs"], b["idxs"])                  # the draw depends on {seed, offset, image} only
    with pytest.raises(ValueError):
        px.device_samples(m, "nonzero-byte", 1, 0, 4, 1, 0, 5, 10)


def test_selection_tie_state():
    """The {seed, offset} tests/test_gpu_device_sampler.py uses for the tie `sel == p`: with 65536 foreground
    pixels and max_num 32768, p is exactly 0.5, and pixel 45589 of image 0 draws exactly 2^23 * 2^-24."""
    mask = syn.disc_mask(65536, 256, 320, center=(160, 128))
    assert po.subsample_probability(32768, 65536) == np.float32(0.5)
    sel = px.selection_values(7, 201, 0, 256 * 320)
    assert mask.ravel()[45589] == 1 and sel[45589] == np.float32(0.5)
    ds = px.device_samples(mask[None], "nonzero", 7, 201, 4, 1, 0, 5, 32768)
    fg_sel = sel[mask.ravel() != 0]
    assert ds["tn"][0] == (fg_sel < 0.5).sum() == (fg_sel <= 0.5).sum() - 1      # the tie pixel is dropped
