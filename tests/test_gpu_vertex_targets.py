"""GPU: the keypoint vertex targets (pvnet_b200.net_utils.vertex_targets, seg_vertex_losses_from_keypoints;
csrc/losses.cu):
  - the field bit for bit against the reference's compute_vertex_hcoords (tests/golden/ref_vertex_targets.npz): K in
    {1, 8, 9, 17, 21}, 37x53 and other ragged shapes, 480x640 at b = 16, every mask dtype with values {0, 1, 2},
    strided and non-contiguous masks, float32 and float64 keypoints, hw in {1, 0, other}, keypoints on and near pixel
    centres, at +-1e6 and NaN / +-inf, use_motion on and off; and against tools/demo.py's field (the demo fixture);
  - the keypoint loss bit for bit against seg_vertex_losses on the materialised field, on channel slices of one
    network-shaped tensor, for every output and for the partial and elementwise forms;
  - grad mode, determinism, CUDA-graph capture, a canary after the output, and the documented errors."""
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

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TORCH_MASK = {np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32, np.dtype(np.uint8): torch.uint8,
              np.dtype(np.bool_): torch.bool}


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_vertex_targets.npz")))


def _gpu(name):
    mask, hc, motion = case_inputs(name)
    return torch.from_numpy(mask).to(DEV), torch.from_numpy(hc).to(DEV), motion


def _stored(golden, name, got):
    return (same_as_stored(canon_nan(got), golden[f"{name}/field"]) and
            canon_nan(got[0, :, got.shape[2] // 2, :8]).tobytes() == golden[f"{name}/slice"].tobytes())


@pytest.mark.parametrize("name", list(CASES))
def test_field_bit_exact(golden, name):
    mask, hc, motion = _gpu(name)
    got = nu.vertex_targets(mask, hc, use_motion=motion)
    assert got.dtype == torch.float32 and got.is_contiguous()
    assert got.shape == (mask.shape[0], 2 * hc.shape[1], *mask.shape[1:])
    assert _stored(golden, name, got)
    bg = (mask != 1)[:, None].expand_as(got)
    assert (got[bg].view(torch.int32) == 0).all()                          # background is +0.0f


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
@pytest.mark.parametrize("name", ["k17_i64_f64_mixed", "k21_i64_f64_special"])
def test_mask_dtypes_and_layouts(golden, name, dtype):
    mask, hc, motion = _gpu(name)
    m = mask.to(dtype)
    b, h, w = m.shape
    if dtype == torch.bool:                               # 2 becomes True: compare with the oracle on that mask
        want = torch.from_numpy(vo.vertex_targets(m.cpu().numpy(), hc.cpu().numpy(), motion)).to(DEV)
        check = lambda got: canon_nan(got).tobytes() == canon_nan(want).tobytes()    # noqa: E731
    else:
        check = lambda got: _stored(golden, name, got)                                # noqa: E731
    assert check(nu.vertex_targets(m, hc, motion))
    big = torch.full((b + 1, h + 5, w + 7), 1, dtype=dtype, device=DEV)
    view = big[1:, 3:3 + h, 5:5 + w]                     # non-contiguous, unaligned rows: the scalar mask path
    view.copy_(m)
    assert not view.is_contiguous()
    assert check(nu.vertex_targets(view, hc, motion))
    t = m.transpose(1, 2).contiguous().transpose(1, 2)   # stride along w is not 1: the host layer copies
    assert check(nu.vertex_targets(t, hc, motion))


def test_float32_keypoints_equal_their_float64_widening():
    mask, hc, _ = _gpu("k9_u8_f64")
    hc32 = hc.float()
    assert torch.equal(nu.vertex_targets(mask, hc32), nu.vertex_targets(mask, hc32.double()))


def test_demo_field(golden):
    mask, field, pts = demo_fixture()
    hc = torch.from_numpy(np.concatenate([pts, np.ones((len(pts), 1))], 1)[None]).to(DEV)
    got = nu.vertex_targets(torch.from_numpy(mask[None]).to(DEV), hc)
    assert got[0].cpu().numpy().tobytes() == field.tobytes()
    assert same_as_stored(canon_nan(got), golden["demo/field"])


def _network_output(name, C=2, seed=0):
    """seg_pred / vertex_pred as channel slices of one [b, C + 2K, h, w] tensor, and the case's mask and weights."""
    mask, hc, motion = _gpu(name)
    b, h, w = mask.shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = torch.randn(b, C + 2 * hc.shape[1], h, w, device=DEV, generator=g)
    weights = (mask == 1).float()[:, None] * torch.rand(b, 1, h, w, device=DEV, generator=g).round()
    return out[:, :C], out[:, C:], mask, hc, weights, motion


LOSS_CASES = ["k9_u8_f64", "k9_i64_f32_motion", "k17_bool_f64_hw0", "k21_i32_f32_special", "k21_i64_f64_special",
              "k9_b16_480x640"]


def _bits(x):
    return canon_nan(x).tobytes()


@pytest.mark.parametrize("name", LOSS_CASES)
def test_keypoint_loss_equals_loss_on_field(name):
    seg, ver, mask, hc, weights, motion = _network_output(name)
    assert not seg.is_contiguous() and not ver.is_contiguous()
    with torch.no_grad():
        field = nu.vertex_targets(mask, hc, motion)
        want = nu.seg_vertex_losses(seg, ver, mask, field, weights)
        got = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights, use_motion=motion)
        assert all(_bits(a) == _bits(b) for a, b in zip(got, want))
        # the vertex loss alone (the mask read for the foreground only), and the elementwise form
        alone = nu._native_losses(pred=ver, mask=mask, wgt=weights, hcoords=hc, use_motion=motion, want=("ver",))
        assert _bits(alone["ver"]) == _bits(want[1])
        el = nu._native_losses(pred=ver, mask=mask, wgt=weights, hcoords=hc, use_motion=motion, normalize=False,
                               want=("ver",))["ver"]
        assert _bits(el) == _bits(nu.smooth_l1_loss(ver, field, weights, normalize=False))


@pytest.mark.parametrize("dtype", [torch.int32, torch.uint8])
def test_keypoint_loss_mask_dtypes_and_views(dtype):
    seg, ver, mask, hc, weights, motion = _network_output("k9_u8_f64")
    m = mask.to(dtype)
    b, h, w = m.shape
    view = torch.zeros((b, h + 2, w + 3), dtype=dtype, device=DEV)[:, 1:1 + h, 2:2 + w]
    view.copy_(m)
    with torch.no_grad():
        want = nu.seg_vertex_losses(seg, ver, m, nu.vertex_targets(m, hc, motion), weights)
        for mm in (m, view):
            got = nu.seg_vertex_losses_from_keypoints(seg, ver, mm, hc, weights, motion)
            assert all(_bits(a) == _bits(b) for a, b in zip(got, want))


def _torch_smooth_l1(pred, tgt, w):
    """The reference's expression (net_utils.py:64-74, sigma = 1) restated with torch ops."""
    diff = w * (pred - tgt)
    ad = torch.abs(diff)
    sign = (ad < 1.).detach().float()
    in_loss = torch.pow(diff, 2) * 0.5 * sign + (ad - 0.5) * (1. - sign)
    b, vd = pred.shape[:2]
    return torch.sum(in_loss.view(b, -1), 1) / (vd * torch.sum(w.view(b, -1), 1) + 1e-3)


def test_grad_mode():
    seg, ver, mask, hc, weights, motion = _network_output("k9_u8_f64")
    mask = mask.clamp(max=1)                              # two classes: a target of 2 would make loss_seg NaN
    seg, ver = seg.clone().requires_grad_(), ver.clone().requires_grad_()
    out = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights)
    assert out[1].requires_grad and out[0].requires_grad
    (out[0].sum() + out[1].sum()).backward()
    g_seg, g_ver = seg.grad.clone(), ver.grad.clone()
    seg.grad = ver.grad = None
    field = nu.vertex_targets(mask, hc)
    want = nu.seg_vertex_losses(seg, ver, mask, field, weights)
    assert all(_bits(a) == _bits(b) for a, b in zip(out, want))
    (want[0].sum() + want[1].sum()).backward()
    assert torch.equal(g_seg, seg.grad) and torch.equal(g_ver, ver.grad)
    ver.grad = None
    _torch_smooth_l1(ver, field, weights).sum().backward()
    torch.testing.assert_close(g_ver, ver.grad, rtol=1e-6, atol=1e-9)


def test_deterministic_and_graph_capture():
    seg, ver, mask, hc, weights, motion = _network_output("k9_b16_480x640")
    with torch.no_grad():
        f1, f2 = nu.vertex_targets(mask, hc), nu.vertex_targets(mask, hc)
        a = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights)
        b = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights)
        assert torch.equal(f1, f2) and all(_bits(x) == _bits(y) for x, y in zip(a, b))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):                                      # warm-up on the capture stream
            nu.vertex_targets(mask, hc)
            nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights)
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            field = nu.vertex_targets(mask, hc)
            out = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc, weights)
        for _ in range(2):
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(field, f1) and all(_bits(x) == _bits(y) for x, y in zip(out, a))


@pytest.mark.parametrize("name,offset", [("k9_b16_480x640", 0), ("k9_u8_f64", 0), ("k9_u8_f64", 1),
                                         ("k8_i32_f32", 3)])
def test_canary_after_output(golden, name, offset):
    """The kernel writes exactly b*2K*h*w floats: a canary before (offset > 0 also makes the float4 path
    unavailable) and after the output stays untouched."""
    mask, hc, motion = _gpu(name)
    b, h, w = mask.shape
    n = b * 2 * hc.shape[1] * h * w
    buf = torch.full((offset + n + 4096,), -7.25, dtype=torch.float32, device=DEV)
    mask_c = mask.contiguous()
    s3 = (ctypes.c_int64 * 3)(*mask_c.stride())
    L = _native.lib()
    _native.check(L.pvnet_vertex_targets(mask_c.data_ptr(), mask_c.element_size(), s3, hc.data_ptr(),
                                         int(hc.dtype == torch.float64), b, h, w, hc.shape[1], int(motion),
                                         buf.data_ptr() + 4 * offset,
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  "pvnet_vertex_targets")
    torch.cuda.synchronize()
    assert (buf[:offset] == -7.25).all() and (buf[offset + n:] == -7.25).all()
    assert _stored(golden, name, buf[offset:offset + n].view(b, 2 * hc.shape[1], h, w))


def test_bad_inputs_raise():
    seg, ver, mask, hc, weights, motion = _network_output("k9_u8_f64")
    with pytest.raises(ValueError, match="ver_dim"):
        nu.seg_vertex_losses_from_keypoints(seg, ver[:, :16], mask, hc, weights)
    with pytest.raises(ValueError, match="hcoords must be"):
        nu.vertex_targets(mask, hc[:, :, :2])
    with pytest.raises(ValueError, match="float32 or float64"):
        nu.vertex_targets(mask, hc.half())
    with pytest.raises(ValueError, match="mask dtype"):
        nu.vertex_targets(mask.float(), hc)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.vertex_targets(mask.cpu(), hc)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hc.cpu(), weights)
