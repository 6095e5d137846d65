"""GPU tests of the voting layer's device-side sampler (`rng="device"`: Philox4x32-10 inside the compaction and
hypothesis kernels) against its restatement in oracle/philox_oracle.py, bit for bit.

Each call reads the sampler's {seed, offset} from its state tensor first, then checks
  (a) the device-drawn hyp, counts, tn, cov_hyp and cov_counts (and keypoints and covariances) equal those of
      the same call with the restated samples injected;
  (b) where the CPU oracle can afford it, hypotheses, counts and tn are bit-exact to the oracle run on those
      samples, keypoints within 1e-4 and covariances within tests/test_gpu_pipeline.py's tolerance;
  (c) the state afterwards is {seed, offset + 1}.
"""
import math

import numpy as np
import pytest
import torch

from oracle import philox_oracle as px
from oracle import pvnet_oracle as po
from pvnet_b200 import ransac_voting_gpu as rv
from pvnet_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KP_TOL = 1e-4
H, W = 192, 256
RAGGED = [0, 3, 1500, 9000]          # empty, below min_num, small, above max_num
BASE = dict(round_hyp_num=128, inlier_thresh=0.99, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=256,
            cov_inlier_thresh=0.99, min_num=5, max_num=4000, mask_mode="nonzero")


@pytest.fixture(autouse=True)
def _restore_torch_rng():
    """The tests re-seed torch; the next device call after them re-seeds the sampler from the restored seed."""
    with torch.random.fork_rng(devices=[torch.device(DEV).index]):
        yield


def _state_tensor():
    return rv._rng_state(torch.device(DEV))


def _state():
    """{seed, offset} the next call draws with (re-made first when torch.manual_seed changed, as a call does)."""
    seed, off = _state_tensor().tolist()
    return seed, off


def _set_state(seed, offset):
    torch.manual_seed(seed)
    rv.reset_device_rng(DEV)
    _state_tensor().copy_(torch.tensor([seed, offset], dtype=torch.int64))
    assert _state() == (seed, offset)


def _inputs(ns, vn, seed, h=H, w=W):
    masks = np.stack([syn.disc_mask(n, h, w, center=(w // 2, h // 2)) for n in ns])
    fields = np.stack([syn.planted_field(masks[i], vn, seed + i, sigma=0.05)[0] for i in range(len(ns))])
    return masks, fields


def _dev(masks, fields, mask_dtype=torch.int64):
    mask = torch.from_numpy(np.ascontiguousarray(masks)).to(DEV).to(mask_dtype)
    ver = torch.from_numpy(np.ascontiguousarray(fields)).to(DEV)
    b, c2, h, w = ver.shape
    return mask, ver.permute(0, 2, 3, 1).view(b, h, w, c2 // 2, 2)


def _hnt(cfg):
    if not cfg["with_covariance"]:
        return 0
    return cfg["cov_round_hyp_num"] * math.ceil(cfg["cov_min_hyp_num"] / cfg["cov_round_hyp_num"])


def _call(mask, vertex, cfg, **kw):
    """ransac_voting_pipeline -> (keypoints, covariances or None, debug dict)."""
    r = rv.ransac_voting_pipeline(mask, vertex, return_debug=True, **cfg, **kw)
    return (r[0], r[1], r[2]) if cfg["with_covariance"] else (r[0], None, r[1])


def _restate(masks, vn, cfg, seed, offset):
    return px.device_samples(masks, cfg["mask_mode"], seed, offset, cfg["round_hyp_num"], vn, _hnt(cfg),
                             cfg["min_num"], cfg["max_num"])


def _injected(mask, vertex, cfg, idxs, cov_idxs, selection):
    kw = dict(idxs=torch.from_numpy(idxs), selection=torch.from_numpy(selection))
    if cfg["with_covariance"]:
        kw["cov_idxs"] = torch.from_numpy(cov_idxs)
    return _call(mask, vertex, cfg, rng="none", **kw)


def _bits(t):
    return t.view(torch.int32)         # NaN keypoints of the same computation compare equal bit for bit


def _assert_same_run(got, want, tag=""):
    (kp, cov, d), (kp2, cov2, d2) = got, want
    for k in ("hyp", "counts", "tn", "cov_hyp", "cov_counts"):
        if k in d:
            assert torch.equal(d[k], d2[k]), f"{tag}{k}: the device draw differs from the restated samples"
    assert torch.equal(_bits(kp), _bits(kp2)), f"{tag}keypoints differ"
    if cov is not None:
        assert torch.equal(_bits(cov), _bits(cov2)), f"{tag}covariances differ"


def _assert_oracle(masks, fields, cfg, ds, run, images=None):
    """(b): the CPU oracle on the restated samples, on `images` (default: all) of the batch."""
    kp, cov, d = run
    images = np.arange(masks.shape[0]) if images is None else np.asarray(images)
    vn = fields.shape[1] // 2
    m, view, tn = masks[images], syn.as_reference_view(fields[images]), ds["tn"][images]
    sels = list(ds["selection"][images])
    v3_mask = m if cfg["mask_mode"] == "nonzero" else (m == 1).astype(np.int64)
    okp, odbg = po.ransac_voting_layer_v3(v3_mask, view, cfg["round_hyp_num"], inlier_thresh=cfg["inlier_thresh"],
                                          min_num=cfg["min_num"], max_num=cfg["max_num"],
                                          idxs=px.reduce(ds["idxs"][images], tn), selection=sels, return_debug=True)
    if cfg["with_covariance"]:
        hn = cfg["cov_round_hyp_num"]
        cidx = [None if c is None else c.reshape(-1, hn, vn, 2) for c in px.reduce(ds["cov_idxs"][images], tn)]
        _, ocov, ocdbg = po.estimate_voting_distribution_with_mean(
            m, view, okp, hn, cfg["cov_min_hyp_num"], inlier_thresh=cfg["cov_inlier_thresh"], min_num=cfg["min_num"],
            max_num=cfg["max_num"], idxs=cidx, selection=sels, return_debug=True)
    kp_n = kp.cpu().numpy()[images]
    got = {k: v.cpu().numpy()[images] for k, v in d.items() if k in ("hyp", "counts", "tn", "cov_hyp", "cov_counts")}
    for j in range(len(images)):
        if odbg[j] is None:
            assert got["tn"][j] == 0 and not kp_n[j].any()
            continue
        assert got["tn"][j] == odbg[j]["tn"] == tn[j]
        assert np.array_equal(got["hyp"][j].view(np.uint32), odbg[j]["hyp"].view(np.uint32)), "v3 hypotheses"
        assert np.array_equal(got["counts"][j], odbg[j]["counts"]), "v3 counts"
        if cfg["with_covariance"]:
            assert ocdbg[j]["tn"] == tn[j]
            assert np.array_equal(got["cov_hyp"][j].view(np.uint32), ocdbg[j]["hyp"].view(np.uint32)), "cov hypotheses"
            assert np.array_equal(got["cov_counts"][j], ocdbg[j]["counts"]), "cov counts"
        both_nan = np.isnan(kp_n[j]) & np.isnan(okp[j])
        assert np.all(both_nan | (np.abs(kp_n[j] - okp[j]) <= KP_TOL)), (kp_n[j], okp[j])
    if cfg["with_covariance"]:
        c = cov.cpu().numpy()[images]
        assert np.allclose(c, ocov, atol=1e-4 + 2e-4 * np.abs(ocov).max() ** 0.5, rtol=1e-4), np.abs(c - ocov).max()


def _check_call(masks, fields, cfg, mask, vertex, oracle=True, images=None):
    """One rng="device" call checked for (a), (b) and (c); returns the restated samples."""
    vn = fields.shape[1] // 2
    seed, off = _state()
    run = _call(mask, vertex, cfg)
    assert _state() == (seed, off + 1), "the call must advance the offset by exactly one"
    ds = _restate(masks, vn, cfg, seed, off)
    assert np.array_equal(run[2]["tn"].cpu().numpy(), ds["tn"]), "kept-pixel counts differ from the restatement"
    _assert_same_run(run, _injected(mask, vertex, cfg, ds["idxs"], ds["cov_idxs"], ds["selection"]),
                     f"{{seed {seed}, offset {off}}} ")
    if oracle:
        _assert_oracle(masks, fields, cfg, ds, run, images)
    return ds


# ------------------------------------------------------------------------------------------ ragged batch
RAGGED_CASES = {
    "cov_same_threshold": dict(BASE),
    "cov_different_thresholds": dict(BASE, inlier_thresh=0.999),
    "no_cov": dict(BASE, with_covariance=False),
    "equals_one": dict(BASE, mask_mode="equals_one"),
}


@pytest.mark.parametrize("case", list(RAGGED_CASES))
def test_ragged_batch(case):
    cfg = RAGGED_CASES[case]
    masks, fields = _inputs(RAGGED, 5, 40)
    if case == "equals_one":                 # label 2: foreground to `nonzero`, background to `== 1`
        for bi in (2, 3):
            ys, xs = np.nonzero(masks[bi])
            masks[bi, ys[::7], xs[::7]] = 2
    mask, vertex = _dev(masks, fields)
    torch.manual_seed(1000 + list(RAGGED_CASES).index(case))
    rv.reset_device_rng(DEV)
    for _ in range(2):                       # offsets 0 and 1
        ds = _check_call(masks, fields, cfg, mask, vertex)
        fg3 = int(px.foreground(masks[3], cfg["mask_mode"]).sum())
        assert fg3 > cfg["max_num"] and 0 < ds["tn"][3] < fg3        # image 3 was subsampled, tn exact
        assert ds["tn"][2] == px.foreground(masks[2], cfg["mask_mode"]).sum()


def test_image_below_min_num_is_skipped_even_above_max_num():
    """min_num 50 > max_num 20: the 30-pixel image is skipped, as the reference tests min_num before it
    subsamples (ransac_voting_gpu.py:531-540); the compaction used to subsample it and vote."""
    masks, fields = _inputs([30, 60, 10], 3, 200, 32, 32)
    mask, vertex = _dev(masks, fields)
    cfg = dict(BASE, round_hyp_num=16, cov_round_hyp_num=16, cov_min_hyp_num=32, min_num=50, max_num=20)
    torch.manual_seed(9)
    rv.reset_device_rng(DEV)
    ds = _check_call(masks, fields, cfg, mask, vertex)
    assert ds["tn"][0] == 0 and ds["tn"][2] == 0 and 0 < ds["tn"][1] < 60


def test_v3_entry_point_routes_through_the_sampler():
    masks, fields = _inputs(RAGGED, 5, 60)
    mask, vertex = _dev(masks, fields)
    cfg = dict(BASE, with_covariance=False, inlier_thresh=0.999)
    torch.manual_seed(2024)
    rv.reset_device_rng(DEV)
    seed, off = _state()
    kp, d = rv.ransac_voting_layer_v3(mask, vertex, 128, inlier_thresh=0.999, max_num=4000, rng="device",
                                      return_debug=True)
    assert _state() == (seed, off + 1)
    ds = _restate(masks, 5, cfg, seed, off)
    kp2, d2 = rv.ransac_voting_layer_v3(mask, vertex, 128, inlier_thresh=0.999, max_num=4000,
                                        idxs=torch.from_numpy(ds["idxs"]), selection=ds["selection"],
                                        return_debug=True)
    _assert_same_run((kp, None, d), (kp2, None, d2))
    _assert_oracle(masks, fields, cfg, ds, (kp, None, d))


# ------------------------------------------------------------------------------------------ mixed injection
@pytest.mark.parametrize("given", ["idxs+cov_idxs", "idxs+selection", "cov_idxs", "all"])
def test_mixed_injection(given):
    """Injected sample sets are used as given; the others come from the sampler at the call's {seed, offset}.
    The offset advances iff some set was left to the device."""
    masks, fields = _inputs(RAGGED, 5, 80)
    mask, vertex = _dev(masks, fields)
    cfg = BASE
    rng = np.random.default_rng(7)
    mine = dict(idxs=rng.integers(0, 2 ** 31 - 1, (4, 128, 5, 2), dtype=np.int32),
                cov_idxs=rng.integers(0, 2 ** 31 - 1, (4, _hnt(cfg), 5, 2), dtype=np.int32),
                selection=rng.random((4, H, W), dtype=np.float32))
    names = given.split("+") if given != "all" else list(mine)
    kw = {k: torch.from_numpy(mine[k]) for k in names}
    torch.manual_seed(31)
    rv.reset_device_rng(DEV)
    _call(mask, vertex, cfg)                 # offset 1: the draw is not the offset-0 one by accident
    seed, off = _state()
    run = _call(mask, vertex, cfg, rng="device", **kw)
    ds = _restate(masks, 5, cfg, seed, off)
    want = {k: (mine[k] if k in names else ds[k]) for k in mine}
    _assert_same_run(run, _injected(mask, vertex, cfg, **want), f"{given} ")
    assert _state() == (seed, off if given == "all" else off + 1)


# ------------------------------------------------------------------------------------------ seed and offset
def test_seed_high_word_reaches_the_key():
    masks, fields = _inputs(RAGGED, 5, 100)
    mask, vertex = _dev(masks, fields)
    torch.manual_seed(2 ** 40 + 5)
    rv.reset_device_rng(DEV)
    assert _state() == (2 ** 40 + 5, 0)
    _check_call(masks, fields, BASE, mask, vertex)


def test_offset_high_word_carries():
    masks, fields = _inputs(RAGGED, 5, 120)
    mask, vertex = _dev(masks, fields)
    _set_state(77, 2 ** 32 - 1)
    _check_call(masks, fields, BASE, mask, vertex)              # offset 0x00000000_ffffffff
    _check_call(masks, fields, BASE, mask, vertex)              # offset 0x00000001_00000000
    assert _state() == (77, 2 ** 32 + 1)


def test_manual_seed_resets_the_state_in_place():
    masks, fields = _inputs(RAGGED, 5, 140)
    mask, vertex = _dev(masks, fields)
    torch.manual_seed(5)
    rv.reset_device_rng(DEV)
    st = _state_tensor()
    ptr = st.data_ptr()
    _check_call(masks, fields, BASE, mask, vertex)
    _check_call(masks, fields, BASE, mask, vertex)
    assert st.tolist() == [5, 2]
    torch.manual_seed(6)                     # no reset_device_rng: the next call re-seeds {6, 0}
    run = _call(mask, vertex, BASE)
    assert st.tolist() == [6, 1] and _state_tensor().data_ptr() == ptr
    ds = _restate(masks, 5, BASE, 6, 0)
    _assert_same_run(run, _injected(mask, vertex, BASE, ds["idxs"], ds["cov_idxs"], ds["selection"]))


# ------------------------------------------------------------------------------------------ selection tie
def test_selection_tie_drops_the_pixel():
    """fg = 65536, max_num = 32768: p is exactly 0.5.  At {seed 7, offset 201} (found by searching offsets with
    the restatement; tests/test_philox_cpu.py checks it) pixel 45589 of image 0 draws sel == 0.5 == p, and
    `sel < p` must drop it."""
    mask_np = syn.disc_mask(65536, 256, 320, center=(160, 128))
    masks = mask_np[None]
    fields = syn.planted_field(mask_np, 2, 160, sigma=0.05)[0][None]
    mask, vertex = _dev(masks, fields)
    cfg = dict(BASE, round_hyp_num=32, with_covariance=False, max_num=32768)
    _set_state(7, 201)
    ds = _check_call(masks, fields, cfg, mask, vertex)
    sel = ds["selection"][0].ravel()
    assert sel[45589] == np.float32(0.5) and mask_np.ravel()[45589] == 1
    fg_sel = sel[mask_np.ravel() != 0]
    assert ds["tn"][0] == (fg_sel <= 0.5).sum() - 1


# ------------------------------------------------------------------------------------------ largest batch
def test_largest_batch():
    """b = 1024 (the most one call takes) 16x16 images: every image index enters the counter.  The whole batch
    is compared with the injected run; the CPU oracle checks images at both ends and the middle."""
    b = 1024
    ns = [(i * 97) % 257 for i in range(b)]                      # 0..256 foreground pixels, max_num 100
    masks = np.stack([syn.disc_mask(n, 16, 16, center=(8, 8)) for n in ns])
    fields = np.stack([syn.random_field(masks[i], 2, 5000 + i) for i in range(b)])
    mask, vertex = _dev(masks, fields, torch.uint8)
    cfg = dict(BASE, round_hyp_num=16, cov_round_hyp_num=16, cov_min_hyp_num=32, max_num=100)
    torch.manual_seed(4242)
    rv.reset_device_rng(DEV)
    images = [0, 1, 2, 3, 510, 511, 512, 513, 1020, 1021, 1022, 1023]
    assert any(ns[i] > 100 for i in images) and any(5 <= ns[i] <= 100 for i in images)
    ds = _check_call(masks, fields, cfg, mask, vertex, images=images)
    assert (ds["tn"][np.array(ns) > 100] < np.array(ns)[np.array(ns) > 100]).any()


# ------------------------------------------------------------------------------------------ graph replay
def test_graph_replays_draw_at_successive_offsets():
    masks, fields = _inputs(RAGGED, 5, 180)
    mask, vertex = _dev(masks, fields, torch.uint8)
    torch.manual_seed(77)
    rv.reset_device_rng(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):           # eager once on the capture stream: workspace and state exist
        _call(mask, vertex, BASE)
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        static = _call(mask, vertex, BASE)
    seed, off0 = _state()
    for i in range(3):
        g.replay()
        torch.cuda.synchronize()
        got = tuple(x.clone() for x in static[:2]) + ({k: v.clone() for k, v in static[2].items()
                                                       if torch.is_tensor(v)},)
        ds = _restate(masks, 5, BASE, seed, off0 + i)
        _assert_same_run(got, _injected(mask, vertex, BASE, ds["idxs"], ds["cov_idxs"], ds["selection"]),
                         f"replay {i} ")
    assert _state() == (seed, off0 + 3)


def test_pose_pipeline_graph_and_eager_draw_the_restated_samples():
    from pvnet_b200.model_repository import Resnet18_8s
    from pvnet_b200.pipeline import IMAGENET_MEAN, IMAGENET_STD, PoseKeypointPipeline
    from tests.helpers import seeded_state_dict
    net = Resnet18_8s(18, 2)
    net.load_state_dict(seeded_state_dict(net, 3))
    net = net.to(DEV).eval()
    kw = dict(round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=128, max_num=3000)
    cfg = dict(BASE, round_hyp_num=64, cov_round_hyp_num=64, cov_min_hyp_num=128, max_num=3000)
    host = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)).pin_memory()
    x = host.to(DEV)
    with torch.no_grad():
        out, mask = net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, mean=IMAGENET_MEAN, std=IMAGENET_STD,
                                       pixel_major=True)
    vertex = out[..., 2:].unflatten(3, (9, 2))
    masks = mask.cpu().numpy()

    def expect(seed, off):
        ds = _restate(masks, 9, cfg, seed, off)
        kp, cov, _ = _injected(mask, vertex, cfg, ds["idxs"], ds["cov_idxs"], ds["selection"])
        return kp, cov

    torch.manual_seed(17)
    rv.reset_device_rng(DEV)
    seed, off = _state()
    with torch.no_grad():
        kp, cov = PoseKeypointPipeline(net, **kw).step(x)
    assert _state() == (seed, off + 1)
    for a, b in zip((kp, cov), expect(seed, off)):
        assert torch.equal(_bits(a), _bits(b)), "eager pipeline"
    graph = PoseKeypointPipeline(net, graph=True, **kw)
    for i in range(2):                       # first run: eager warm-up at off+1, capture, replay at off+2
        res = graph.run([host])
        torch.cuda.synchronize()
        for a, b in zip(res, expect(seed, off + 2 + i)):
            assert torch.equal(_bits(a), _bits(b)), f"graph run {i}"
    assert _state() == (seed, off + 4)
