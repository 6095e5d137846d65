"""The native launch sequence of every host entry point of the voting layer, counted with
`_native.launch_count()`.  Samples are injected (or drawn on the device), so no foreground-count
launches are mixed in; only the native kernels of the one call are counted.

v3's sequence is k_chunk_count, k_compact_write, k_gather, k_gen_hyp, k_vote3, k_refit and
k_refit_final; an image that may be subsampled adds k_chunk_kept, debug outputs add k_export.
"""
import pytest
import torch

from pvnet_b200 import _native
from pvnet_b200 import ransac_voting_gpu as rv

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, H, W, VN, HN = 2, 60, 80, 3, 256       # 4800 pixels per image, about half of them foreground


def _inputs(seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    mask = (torch.rand([B, H, W], generator=g, device=DEV) < 0.5).to(torch.uint8)
    vertex = torch.randn([B, H, W, VN, 2], generator=g, device=DEV)
    return mask, vertex


def _idxs(hn):
    return torch.randint(0, 2 ** 31 - 1, [B, hn, VN, 2], dtype=torch.int32, device=DEV)


def _selection():
    return torch.rand([B, H, W], device=DEV)


def _launches(fn):
    torch.cuda.synchronize()
    _native.launch_count_reset()
    fn()
    n = _native.launch_count()
    torch.cuda.synchronize()
    return n


@pytest.mark.parametrize("subsample", [False, True])
@pytest.mark.parametrize("debug", [False, True])
def test_v3(subsample, debug):
    mask, vertex = _inputs()
    idxs = _idxs(HN)
    sel = _selection() if subsample else None
    n = _launches(lambda: rv.ransac_voting_layer_v3(mask, vertex, HN, max_num=1000, idxs=idxs, selection=sel,
                                                    return_debug=debug))
    assert n == 7 + subsample + debug


def test_v3_selection_without_subsampling():
    """A selection field with max_num >= h*w: no image can be subsampled, so no k_chunk_kept."""
    mask, vertex = _inputs()
    n = _launches(lambda: rv.ransac_voting_layer_v3(mask, vertex, HN, max_num=H * W, idxs=_idxs(HN),
                                                    selection=_selection()))
    assert n == 7


def test_v3_device_rng():
    """rng="device" hands v3 to the pipeline: v3's sequence and k_rng_bump."""
    mask, vertex = _inputs()
    assert _launches(lambda: rv.ransac_voting_layer_v3(mask, vertex, HN, rng="device")) == 8


def test_v4_v5():
    mask, vertex = _inputs()
    idxs = _idxs(HN)
    assert _launches(lambda: rv.ransac_voting_layer_v4(mask, vertex, HN, idxs=idxs)) == 7 + 2   # k_resid_sum, _final
    assert _launches(lambda: rv.ransac_voting_layer_v5(mask, vertex, HN, idxs=idxs)) == 7 + 2    # k_conf_count, _final


@pytest.mark.parametrize("debug", [False, True])
def test_with_mean(debug):
    """k_chunk_count, k_compact_write, k_gather, k_gen_hyp, k_vote3, k_cov (+ k_export)."""
    mask, vertex = _inputs()
    mean = torch.rand([B, VN, 2], device=DEV) * W
    n = _launches(lambda: rv.estimate_voting_distribution_with_mean(mask, vertex, mean, 128, 512, idxs=_idxs(512),
                                                                    return_debug=debug))
    assert n == 6 + debug


@pytest.mark.parametrize("with_cov,cov_thresh,debug,expected", [
    (False, 0.99, False, 7),      # v3's sequence
    (False, 0.99, True, 8),       # + k_export
    (True, 0.99, False, 9),       # + a second k_gen_hyp, one k_vote3 for both sets, k_cov
    (True, 0.999, False, 10),     # different thresholds: one k_vote3 per set
    (True, 0.99, True, 11),       # + k_export of both sets
])
def test_pipeline_injected(with_cov, cov_thresh, debug, expected):
    mask, vertex = _inputs()
    cov_idxs = _idxs(512) if with_cov else None
    n = _launches(lambda: rv.ransac_voting_pipeline(mask, vertex, HN, 0.99, with_cov, 256, 512, cov_thresh,
                                                    idxs=_idxs(HN), cov_idxs=cov_idxs, rng="none",
                                                    return_debug=debug))
    assert n == expected


@pytest.mark.parametrize("with_cov,max_num,expected", [
    (False, 30000, 8),            # v3's sequence + k_rng_bump
    (True, 30000, 10),            # + k_gen_hyp, k_cov
    (True, 1000, 11),             # + k_chunk_kept: the device RNG may subsample
])
def test_pipeline_device_rng(with_cov, max_num, expected):
    mask, vertex = _inputs()
    n = _launches(lambda: rv.ransac_voting_pipeline(mask, vertex, HN, 0.99, with_cov, 256, 512, 0.99,
                                                    max_num=max_num, rng="device"))
    assert n == expected
