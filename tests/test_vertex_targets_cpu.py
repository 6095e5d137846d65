"""CPU: the keypoint vertex targets' numpy restatement (oracle/vertex_target_oracle.py) bit for bit against the
reference's own compute_vertex_hcoords and tools/demo.py's compute_vertex, as recorded in
tests/golden/ref_vertex_targets.npz (tests/golden/make_golden_vertex_targets.py); the shim's two new names; the
argument checks of the host layer and of the C ABI."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import vertex_target_oracle as vo
from pvnet_b200 import _native
from pvnet_b200 import net_utils as nu
from tests.helpers import GOLDEN, demo_fixture, same_as_stored
from tests.vertex_target_cases import CASES, canon_nan, case_inputs


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_vertex_targets.npz")))


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_equals_reference(golden, name):
    mask, hc, motion = case_inputs(name)
    got = vo.vertex_targets(mask, hc, motion)
    assert same_as_stored(canon_nan(got), golden[f"{name}/field"])
    assert canon_nan(got[0, :, got.shape[2] // 2, :8]).tobytes() == golden[f"{name}/slice"].tobytes()


def test_oracle_equals_reference_demo(golden):
    mask, field, pts = demo_fixture()
    hc = np.concatenate([pts, np.ones((len(pts), 1))], 1)[None]
    got = vo.vertex_targets(mask[None], hc)
    assert same_as_stored(canon_nan(got), golden["demo/field"])
    assert got[0].tobytes() == field.tobytes()


def test_float32_keypoints_are_widened_exactly():
    mask, hc, _ = case_inputs("k9_u8_f64")
    hc32 = hc.astype(np.float32)
    assert vo.vertex_targets(mask, hc32).tobytes() == vo.vertex_targets(mask, hc32.astype(np.float64)).tobytes()


def test_shim_exports_the_keypoint_functions():
    import lib.utils.net_utils as shim
    assert shim.vertex_targets is nu.vertex_targets
    assert shim.seg_vertex_losses_from_keypoints is nu.seg_vertex_losses_from_keypoints
    assert {"vertex_targets", "seg_vertex_losses_from_keypoints"} <= set(shim.__all__)


def _inputs(b=2, h=8, w=12, K=3, C=2):
    seg = torch.zeros(b, C, h, w)
    pred = torch.zeros(b, 2 * K, h, w)
    mask = torch.zeros(b, h, w, dtype=torch.int64)
    hc = torch.zeros(b, K, 3, dtype=torch.float64)
    wgt = torch.zeros(b, 1, h, w)
    return seg, pred, mask, hc, wgt


def test_host_layer_validation():
    seg, pred, mask, hc, wgt = _inputs()
    bad = [
        (dict(hc=hc[:, :, :2]), "hcoords must be"), (dict(hc=hc[:1]), "hcoords must be"),
        (dict(hc=hc.float().half()), "float32 or float64"), (dict(mask=mask.float()), "mask dtype"),
        (dict(hc=torch.zeros(2, 4, 3)), "ver_dim"), (dict(wgt=wgt[:, :, :4]), "vertex_weights"),
        (dict(pred=pred.double()), "float32"), (dict(seg=seg[:1]), "mask must be"),
    ]
    for kw, text in bad:
        a = {**dict(seg=seg, pred=pred, mask=mask, hc=hc, wgt=wgt), **kw}
        with pytest.raises(ValueError, match=text):
            nu.seg_vertex_losses_from_keypoints(a["seg"], a["pred"], a["mask"], a["hc"], a["wgt"])
    with pytest.raises(ValueError, match="hcoords must be"):
        nu.vertex_targets(mask, hc[:, :, :2])
    with pytest.raises(ValueError, match="hcoords must be"):
        nu.vertex_targets(mask, torch.zeros(2, 0, 3))
    with pytest.raises(ValueError, match="mask must be"):
        nu.vertex_targets(mask[0], hc)
    with pytest.raises(ValueError, match="mask dtype"):
        nu.vertex_targets(mask.to(torch.int16), hc)


def test_cpu_tensors_raise():
    seg, pred, mask, hc, wgt = _inputs()
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.vertex_targets(mask, hc)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_losses_from_keypoints(seg, pred, mask, hc, wgt)
    with pytest.raises(RuntimeError, match="CUDA"):                 # grad mode materialises the field on the device
        nu.seg_vertex_losses_from_keypoints(seg, pred.requires_grad_(), mask, hc, wgt)


def test_abi_argument_validation():
    L = _native.lib()
    s4 = (ctypes.c_int64 * 4)(20 * 64, 64, 8, 1)
    s3 = (ctypes.c_int64 * 3)(64, 8, 1)
    bad3 = (ctypes.c_int64 * 3)(64, 8, 2)
    bad4 = (ctypes.c_int64 * 4)(20 * 64, 64, 8, 2)
    p = ctypes.c_void_p(256)                                       # never dereferenced: every call below is refused
    out = ctypes.c_void_p(512)

    def targets(mask=p, msz=8, masks=s3, hc=p, b=2, h=8, w=8, K=9, vout=out):
        return L.pvnet_vertex_targets(mask, msz, masks, hc, 1, b, h, w, K, 0, vout, None)

    def losses(seg=p, segs=s4, mask=p, msz=8, masks=s3, pred=p, preds=s4, hc=p, wgt=p, wgts=s4, b=2, h=8, w=8, C=2,
               vd=18, sigma=1.0, ls=out, lv=out, pr=out, rc=out, ws=p, wsb=1 << 20):
        return L.pvnet_seg_vertex_losses_keypoints(seg, segs, mask, msz, masks, pred, preds, hc, 1, 0, wgt, wgts, b, h,
                                                   w, C, vd, sigma, 1, ls, lv, pr, rc, ws, wsb, None)

    cases = [
        (targets, dict(b=0), b"dimension"), (targets, dict(K=0), b"dimension"), (targets, dict(mask=None), b"null"),
        (targets, dict(hc=None), b"null"), (targets, dict(vout=None), b"null"), (targets, dict(msz=2), b"mask_elem"),
        (targets, dict(masks=bad3), b"unit stride"),
        (losses, dict(b=0), b"dimension"), (losses, dict(vd=17), b"ver_dim"), (losses, dict(hc=None), b"null"),
        (losses, dict(mask=None), b"null"), (losses, dict(mask=None, ls=None, pr=None, rc=None), b"null"),
        (losses, dict(pred=None), b"null"), (losses, dict(wgt=None), b"null"), (losses, dict(ws=None), b"null"),
        (losses, dict(preds=bad4), b"unit stride"), (losses, dict(masks=bad3), b"unit stride"),
        (losses, dict(msz=2), b"mask_elem_size"), (losses, dict(wsb=8), b"workspace"),
        (losses, dict(sigma=0.0), b"sigma"), (losses, dict(ls=None, lv=None, pr=None, rc=None), b"no output"),
    ]
    for fn, kw, text in cases:
        assert fn(**kw) == -1, kw
        assert text in L.pvnet_last_error(), (kw, L.pvnet_last_error())
