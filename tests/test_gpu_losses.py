"""GPU: the validation losses on the device (pvnet_b200/net_utils.py, pvnet_b200/csrc/losses.cu).
  - elementwise smooth-L1 bit for bit against the reference's record (tests/golden/ref_net_utils.npz) and a torch
    restatement of its expression on the GPU;
  - normalised smooth-L1 and cross-entropy against the oracle (oracle/loss_oracle.py) and torch;
  - precision / recall bit for bit against the record and torch: ties, NaN logits, C = 3, every mask dtype, an empty
    mask; ignore_index and invalid targets (the latter against the oracle only);
  - the channel slices of the native backbone's output read in place; determinism and a CUDA-graph replay;
  - NetWrapper in eval / no_grad and in grad mode."""
import os

import numpy as np
import pytest
import torch
from torch import nn

from oracle import loss_oracle as lo
from pvnet_b200 import net_utils as nu
from tests.helpers import GOLDEN, same_as_stored, seeded_state_dict
from tests.loss_cases import CASES, canon_nan, case_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_net_utils.npz")))


def _gpu(*arrays):
    return [torch.from_numpy(a).to(DEV) for a in arrays]


def _torch_smooth_l1(pred, tgt, w, sigma, normalize):
    """The reference's expression (net_utils.py:64-74) restated with torch ops."""
    s2 = sigma ** 2
    diff = w * (pred - tgt)
    ad = torch.abs(diff)
    sign = (ad < 1. / s2).detach().float()
    in_loss = torch.pow(diff, 2) * (s2 / 2.) * sign + (ad - (0.5 / s2)) * (1. - sign)
    if normalize:
        b, vd = pred.shape[:2]
        in_loss = torch.sum(in_loss.view(b, -1), 1) / (vd * torch.sum(w.view(b, -1), 1) + 1e-3)
    return in_loss


def _torch_precision_recall(scores, target):
    b = scores.shape[0]
    p = torch.argmax(scores, 1).float()
    t = target.float()
    tp, fp, fn = (torch.sum(x.view(b, -1), 1) for x in (p * t, p * (1 - t), (1 - p) * t))
    return (tp + 1) / (tp + fp + 1), (tp + 1) / (tp + fn + 1)


def _torch_ce(seg, mask):
    loss = nn.CrossEntropyLoss(reduction="none")(seg, mask.long())
    return torch.mean(loss.view(loss.shape[0], -1), 1)


def _bits_equal(a, b):
    return canon_nan(a).tobytes() == canon_nan(b).tobytes()


@pytest.mark.parametrize("name", list(CASES))
def test_smooth_l1_elementwise_bit_exact(name):
    g = _golden()
    seg, mask, pred, vertex, weights, sigma = case_inputs(name)
    p, t, w = _gpu(pred, vertex, weights)
    got = nu.smooth_l1_loss(p, t, w, sigma=sigma, normalize=False)
    assert got.shape == p.shape
    assert same_as_stored(canon_nan(got), g[f"{name}/elem"])
    assert _bits_equal(got, _torch_smooth_l1(p, t, w, sigma, False))
    for s in (1.0, 3.0, 0.5):
        assert _bits_equal(nu.smooth_l1_loss(p, t, w, sigma=s, normalize=False), _torch_smooth_l1(p, t, w, s, False))


@pytest.mark.parametrize("name", list(CASES))
def test_normalized_smooth_l1_and_cross_entropy(name):
    g = _golden()
    seg, mask, pred, vertex, weights, sigma = case_inputs(name)
    p, t, w, s, m = _gpu(pred, vertex, weights, seg, mask)
    got = nu.smooth_l1_loss(p, t, w, sigma=sigma).cpu().numpy()
    np.testing.assert_allclose(got, lo.smooth_l1_normalized(pred, vertex, weights, sigma), rtol=1e-6)
    np.testing.assert_allclose(got, _torch_smooth_l1(p, t, w, sigma, True).cpu().numpy(), rtol=1e-5)
    np.testing.assert_allclose(got, g[f"{name}/norm"], rtol=1e-6)
    ce, ver, prec, rec = nu.seg_vertex_losses(s, p, m, t, w)
    np.testing.assert_allclose(ce.cpu().numpy(), lo.cross_entropy(seg, mask), rtol=1e-6)
    np.testing.assert_allclose(ce.cpu().numpy(), _torch_ce(s, m).cpu().numpy(), rtol=1e-5)
    if sigma == 1.0:
        np.testing.assert_allclose(ver.cpu().numpy(), g[f"{name}/norm"], rtol=1e-6)


@pytest.mark.parametrize("name", list(CASES))
def test_precision_recall_bit_exact(name):
    g = _golden()
    seg, mask, *_ = case_inputs(name)
    s, m = _gpu(seg, mask)
    prec, rec = nu.compute_precision_recall(s, m)
    assert prec.cpu().numpy().tobytes() == g[f"{name}/precision"].tobytes()
    assert rec.cpu().numpy().tobytes() == g[f"{name}/recall"].tobytes()
    tp, tr = _torch_precision_recall(s, m)
    assert torch.equal(prec, tp) and torch.equal(rec, tr)
    pm, rm = nu.compute_precision_recall(s, m, reduce=True)
    assert pm.dim() == 0 and torch.equal(pm, torch.mean(prec)) and torch.equal(rm, torch.mean(rec))


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
def test_mask_dtypes_and_empty_mask(dtype):
    seg, mask, pred, vertex, weights, _ = case_inputs("k9_s1_binary")
    s, p, t, w = _gpu(seg, pred, vertex, weights)
    for msk in (mask, np.zeros_like(mask)):                               # the second is an empty mask
        m64 = torch.from_numpy(msk).to(DEV)
        m = m64.to(dtype)
        want_p, want_r = _torch_precision_recall(s, m64)
        prec, rec = nu.compute_precision_recall(s, m)
        assert torch.equal(prec, want_p) and torch.equal(rec, want_r)
        ce, ver, prec2, rec2 = nu.seg_vertex_losses(s, p, m, t, w)
        assert torch.equal(prec2, want_p) and torch.equal(rec2, want_r)
        np.testing.assert_allclose(ce.cpu().numpy(), _torch_ce(s, m64).cpu().numpy(), rtol=1e-5)


def test_ignore_index_and_invalid_targets():
    seg, mask, pred, vertex, weights, _ = case_inputs("k17_s05_c3")
    mask = mask.copy()
    mask[0, :5] = -100                                                    # ignored rows in image 0
    s, m, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    ce = nu.seg_vertex_losses(s, p, m, t, w)[0].cpu().numpy()
    np.testing.assert_allclose(ce, lo.cross_entropy(seg, mask), rtol=1e-6)
    np.testing.assert_allclose(ce, _torch_ce(s, m).cpu().numpy(), rtol=1e-5)    # -100 is torch's ignore_index
    # invalid targets: NaN for that image only (torch would raise a device-side assert: never handed to it)
    bad = mask.copy()
    bad[1, 7, 11] = 3                                                     # C = 3
    bad[0, 20, 2] = -1
    got = nu.seg_vertex_losses(s, p, torch.from_numpy(bad).to(DEV), t, w)[0].cpu().numpy()
    want = lo.cross_entropy(seg, bad)
    assert np.isnan(got).all() and np.isnan(want).all()
    bad[0, 20, 2] = 0
    got = nu.seg_vertex_losses(s, p, torch.from_numpy(bad).to(DEV), t, w)[0].cpu().numpy()
    assert np.isnan(got[1]) and not np.isnan(got[0])
    np.testing.assert_allclose(got[0], lo.cross_entropy(seg, bad)[0], rtol=1e-6)


@pytest.fixture(scope="module")
def backbone_outputs():
    from pvnet_b200.model_repository import Resnet18_8s
    net = Resnet18_8s(ver_dim=18, seg_dim=2)
    net.load_state_dict(seeded_state_dict(net, seed=3))
    net = net.to(DEV).eval()
    x = torch.from_numpy(np.random.default_rng(5).standard_normal((4, 3, 480, 640), dtype=np.float32)).to(DEV)
    with torch.no_grad():
        seg, ver = net(x)
    rng = np.random.default_rng(6)
    mask = torch.from_numpy(rng.integers(0, 2, (4, 480, 640))).to(DEV)
    vertex = torch.from_numpy(rng.normal(0, 1, (4, 18, 480, 640)).astype(np.float32)).to(DEV)
    weights = (mask > 0).float()[:, None]
    return net, x, seg, ver, mask, vertex, weights


def test_strided_backbone_slices(backbone_outputs):
    _, _, seg, ver, mask, vertex, weights = backbone_outputs
    assert not seg.is_contiguous() and not ver.is_contiguous()
    with torch.no_grad():
        got = nu.seg_vertex_losses(seg, ver, mask, vertex, weights)
        contig = nu.seg_vertex_losses(seg.contiguous(), ver.contiguous(), mask, vertex, weights)
    for a, b in zip(got, contig):
        assert torch.equal(a, b)
    sn, vn, mn, tn, wn = (a.cpu().numpy() for a in (seg, ver, mask, vertex, weights))
    np.testing.assert_allclose(got[0].cpu().numpy(), lo.cross_entropy(sn, mn), rtol=1e-6)
    np.testing.assert_allclose(got[1].cpu().numpy(), lo.smooth_l1_normalized(vn, tn, wn), rtol=1e-6)
    p, r = lo.precision_recall(sn, mn)
    assert got[2].cpu().numpy().tobytes() == p.tobytes() and got[3].cpu().numpy().tobytes() == r.tobytes()
    el = nu.smooth_l1_loss(ver, vertex, weights, normalize=False)
    assert _bits_equal(el, _torch_smooth_l1(ver, vertex, weights, 1.0, False))


def test_deterministic_and_graph_capture(backbone_outputs):
    _, _, seg, ver, mask, vertex, weights = backbone_outputs
    with torch.no_grad():
        a = nu.seg_vertex_losses(seg, ver, mask, vertex, weights)
        b = nu.seg_vertex_losses(seg, ver, mask, vertex, weights)
        assert all(x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes() for x, y in zip(a, b))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            nu.seg_vertex_losses(seg, ver, mask, vertex, weights)           # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = nu.seg_vertex_losses(seg, ver, mask, vertex, weights)
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(out, a))


def test_netwrapper_eval_matches_reference_composition(backbone_outputs):
    net, x, seg, ver, mask, vertex, weights = backbone_outputs
    wrapper = nu.NetWrapper(net)
    with torch.no_grad():
        sp, vp, loss_seg, loss_vertex, precision, recall = wrapper(x, mask, vertex, weights)
        assert torch.equal(sp, seg) and torch.equal(vp, ver)
        np.testing.assert_allclose(loss_seg.cpu().numpy(), _torch_ce(sp, mask).cpu().numpy(), rtol=1e-5)
        np.testing.assert_allclose(loss_vertex.cpu().numpy(),
                                   nu.smooth_l1_loss(vp, vertex, weights, reduce=False).cpu().numpy(), rtol=1e-5)
        p, r = nu.compute_precision_recall(sp, mask)
        assert torch.equal(precision, p) and torch.equal(recall, r)


class _TinyNet(nn.Module):
    """A 1x1 convolution standing in for the network in grad mode."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 2 + 18, 1)

    def forward(self, x):
        out = self.conv(x)
        return out[:, :2], out[:, 2:]


def test_netwrapper_grad_mode_gradient():
    torch.manual_seed(0)
    net = _TinyNet().to(DEV)
    rng = np.random.default_rng(2)
    x = torch.from_numpy(rng.normal(0, 1, (2, 3, 24, 32)).astype(np.float32)).to(DEV)
    mask = torch.from_numpy(rng.integers(0, 2, (2, 24, 32))).to(DEV)
    vertex = torch.from_numpy(rng.normal(0, 1, (2, 18, 24, 32)).astype(np.float32)).to(DEV)
    weights = (mask > 0).float()[:, None]
    out = nu.NetWrapper(net)(x, mask, vertex, weights)
    out[3].sum().backward()
    got = net.conv.weight.grad.clone()
    net.conv.weight.grad = None
    seg, ver = net(x)
    _torch_smooth_l1(ver, vertex, weights, 1.0, True).sum().backward()
    torch.testing.assert_close(got, net.conv.weight.grad, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(out[2].detach().cpu().numpy(), _torch_ce(seg, mask).detach().cpu().numpy(), rtol=1e-5)


def test_cpu_tensors_without_grad_raise():
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.smooth_l1_loss(torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 4, 4), torch.zeros(1, 1, 4, 4))
