"""GPU: the training losses' backward on the device (seg_vertex_training_losses[_from_keypoints] in
pvnet_b200/net_utils.py, pvnet_seg_vertex_losses[_keypoints]_backward in pvnet_b200/csrc/losses.cu, DESIGN.md §13).
  - the vertex gradient bit for bit against torch's CUDA autograd through the reference's expression where torch's
    fp32 sum of the weights is exact, against the oracle bit for bit everywhere;
  - the seg gradient bit for bit against torch's CUDA autograd of nn.CrossEntropyLoss + mean: ignore_index, C = 3,
    NaN / inf logits, every mask dtype; invalid targets against the oracle; ATen's CUDA MeanBackward pinned;
  - the keypoint form bit-identical to the field form; the network's one output tensor; the memory of the backward;
    NULL loss gradients; bad inputs; CUDA-graph replay, determinism and nn.DataParallel."""
import numpy as np
import pytest
import torch
from torch import nn

from oracle import loss_grad_oracle as lgo
from pvnet_b200 import net_utils as nu
from tests import vertex_target_cases as vtc
from tests.helpers import seeded_state_dict
from tests.loss_cases import CASES, canon_nan, case_inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gpu(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in arrays]


def _torch_ce(seg, mask):
    """train_linemod.py:83,87-88."""
    loss = nn.CrossEntropyLoss(reduction="none")(seg, mask.long())
    return torch.mean(loss.view(loss.shape[0], -1), 1)


def _torch_smooth_l1(pred, tgt, w):
    """net_utils.py:54-80 as written (sigma = 1, normalize=True)."""
    b, ver_dim = pred.shape[:2]
    diff = w * (pred - tgt)
    abs_diff = torch.abs(diff)
    sign = (abs_diff < 1.).detach().float()
    in_loss = torch.pow(diff, 2) * (1. / 2.) * sign + (abs_diff - 0.5) * (1. - sign)
    return torch.sum(in_loss.view(b, -1), 1) / (ver_dim * torch.sum(w.view(b, -1), 1) + 1e-3)


def _loss_grads(b, seed=0):
    rng = np.random.default_rng(seed)
    return _gpu(rng.uniform(0.25, 2.0, b).astype(np.float32), rng.uniform(0.25, 2.0, b).astype(np.float32))


def _torch_grads(seg, pred, mask, vertex, w, gs, gv):
    s, p = seg.detach().clone().requires_grad_(), pred.detach().clone().requires_grad_()
    return torch.autograd.grad((_torch_ce(s, mask), _torch_smooth_l1(p, vertex, w)), (s, p), (gs, gv))


def _native_grads(seg, pred, mask, tgt, w, gs, gv, keypoints=False, use_motion=False):
    s, p = seg.detach().clone().requires_grad_(), pred.detach().clone().requires_grad_()
    if keypoints:
        out = nu.seg_vertex_training_losses_from_keypoints(s, p, mask, tgt, w, use_motion=use_motion)
    else:
        out = nu.seg_vertex_training_losses(s, p, mask, tgt, w)
    return torch.autograd.grad((out[0], out[1]), (s, p), (gs, gv))


def _bits(a):
    return canon_nan(a).tobytes()


def _exact(a):
    return a.detach().cpu().numpy().tobytes()


@pytest.mark.parametrize("name", list(CASES))
def test_vertex_gradient(name):
    seg, mask, pred, vertex, weights, _ = case_inputs(name)
    s, m, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    gs, gv = _loss_grads(s.shape[0])
    _, got = _native_grads(s, p, m, t, w, gs, gv)
    _, want = _torch_grads(s, p, m, t, w, gs, gv)
    oracle = lgo.smooth_l1_grad(pred, vertex, weights, gv.cpu().numpy())
    assert _bits(got) == _bits(oracle)
    b, vd = p.shape[:2]
    torch_den = (vd * torch.sum(w.view(b, -1), 1) + 1e-3).cpu().numpy()
    if np.array_equal(torch_den, lgo.vertex_denominator(weights, vd)):       # 0/1 weights: torch's Σw is exact
        assert CASES[name][6] == "binary"
        assert _bits(got) == _bits(want)
    else:                                                                   # only torch's fp32 Σw differs
        np.testing.assert_allclose(canon_nan(got), canon_nan(want), rtol=1e-6, atol=0)
        assert _bits(lgo.smooth_l1_grad(pred, vertex, weights, gv.cpu().numpy(), den=torch_den)) == _bits(want)


@pytest.mark.parametrize("name", list(CASES))
def test_seg_gradient(name):
    seg, mask, pred, vertex, weights, _ = case_inputs(name)
    mask = mask.copy()
    mask[0, :5] = -100                                                      # ignored rows
    s, m, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    gs, gv = _loss_grads(s.shape[0], seed=1)
    got, _ = _native_grads(s, p, m, t, w, gs, gv)
    want, _ = _torch_grads(s, p, m, t, w, gs, gv)
    assert _bits(got) == _bits(want)
    n = seg.shape[2] * seg.shape[3]
    oracle = lgo.cross_entropy_grad(seg, mask, gs.cpu().numpy())
    bound = (2.0 ** -20 * gs.cpu().numpy() / n)[:, None, None, None]
    g = canon_nan(got)
    assert np.array_equal(np.isnan(g), np.isnan(oracle))
    assert (np.abs(np.nan_to_num(g) - np.nan_to_num(oracle)) <= bound).all()
    finite = np.isfinite(seg[0, :, :5]).all(0)                               # ignored pixels: 0 in every channel
    assert (g[0, :, :5][:, finite] == 0).all()


@pytest.mark.parametrize("dtype", [torch.int64, torch.int32, torch.uint8, torch.bool])
def test_seg_gradient_mask_dtypes(dtype):
    seg, mask, pred, vertex, weights, _ = case_inputs("k9_s1_binary")
    s, m64, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    gs, gv = _loss_grads(s.shape[0], seed=2)
    want = _torch_grads(s, p, m64, t, w, gs, gv)
    got = _native_grads(s, p, m64.to(dtype), t, w, gs, gv)
    assert _bits(got[0]) == _bits(want[0]) and _bits(got[1]) == _bits(want[1])


def test_invalid_targets_nan_for_that_image_only():
    seg, mask, pred, vertex, weights, _ = case_inputs("k17_s05_c3")
    bad = mask.copy()
    bad[1, 7, 11] = 3                                                       # C = 3
    s, m, p, t, w = _gpu(seg, bad, pred, vertex, weights)
    gs, gv = _loss_grads(2, seed=3)
    got, gver = _native_grads(s, p, m, t, w, gs, gv)
    g = canon_nan(got)
    assert np.isnan(g[1]).all() and not np.isnan(g[0]).any()
    oracle = lgo.cross_entropy_grad(seg, bad, gs.cpu().numpy())
    assert np.isnan(oracle[1]).all()
    assert (np.abs(g[0] - oracle[0]) <= 2.0 ** -20 * gs[0].item() / (37 * 53)).all()
    want = _torch_grads(s[:1], p[:1], m[:1], t[:1], w[:1], gs[:1], gv[:1])     # torch asserts on image 1
    assert _bits(got[:1]) == _bits(want[0])
    assert _bits(gver[:1]) == _bits(want[1])


def test_cuda_mean_backward_is_a_reciprocal_multiply():
    """ATen divides a CUDA tensor by a CPU scalar as a * (1 / b): the seg gradient's g = gs * (1.0f / N)."""
    n = 37 * 53
    gs = torch.from_numpy(np.random.default_rng(4).uniform(0.1, 10, 4096).astype(np.float32)).to(DEV)
    x = torch.zeros(4096, n, device=DEV, requires_grad=True)
    g = torch.autograd.grad(x.view(4096, -1).mean(1), x, gs)[0][:, 0].cpu().numpy()
    gsn = gs.cpu().numpy()
    assert g.tobytes() == (gsn * (np.float32(1) / np.float32(n))).tobytes()
    assert (g != gsn / np.float32(n)).any()                                 # which differs from the division


@pytest.mark.parametrize("name", ["k8_i32_f32", "k9_u8_f64", "k9_i64_f32_motion", "k17_bool_f64_hw0",
                                  "k21_i32_f32_special", "k21_u8_f64_special_motion"])
def test_keypoint_form_equals_field_form(name):
    mask_np, hc_np, motion = vtc.case_inputs(name)
    b, h, w = mask_np.shape
    K = hc_np.shape[1]
    rng = np.random.default_rng(7)
    out = torch.from_numpy(rng.normal(0, 1, (b, 3 + 2 * K, h, w)).astype(np.float32)).to(DEV)
    mask, hc = _gpu(mask_np, hc_np)
    frac, = _gpu(rng.uniform(0.5, 1, (b, 1, h, w)).astype(np.float32))
    weights = (mask == 1).float()[:, None] * frac
    gs, gv = _loss_grads(b, seed=5)
    field = nu.vertex_targets(mask, hc, motion)
    seg, pred = out[:, :3], out[:, 3:]
    a = _native_grads(seg, pred, mask, field, weights, gs, gv)
    k = _native_grads(seg, pred, mask, hc, weights, gs, gv, keypoints=True, use_motion=motion)
    assert _exact(a[0]) == _exact(k[0]) and _exact(a[1]) == _exact(k[1])


class _TinyNet(nn.Module):
    """A 1x1 convolution whose output's channel slices stand in for the network's."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 2 + 18, 1)

    def forward(self, x):
        out = self.conv(x)
        return out[:, :2], out[:, 2:]


def _train_batch(b, h, w, seed):
    rng = np.random.default_rng(seed)
    x, mask, vertex = _gpu(rng.normal(0, 1, (b, 3, h, w)).astype(np.float32), rng.integers(0, 2, (b, h, w)),
                           rng.normal(0, 1, (b, 18, h, w)).astype(np.float32))
    return x, mask, vertex, (mask > 0).float()[:, None]


def _param_grads(net, x, mask, vertex, weights, native):
    net.zero_grad(set_to_none=True)
    seg, ver = net(x)
    fn = nu.seg_vertex_training_losses if native else nu.seg_vertex_losses
    loss_seg, loss_vertex, _, _ = fn(seg, ver, mask, vertex, weights)
    (torch.mean(loss_seg) + torch.mean(loss_vertex)).backward()
    return {k: v.grad.clone() for k, v in net.named_parameters() if v.grad is not None}, loss_seg, loss_vertex


@pytest.mark.parametrize("which", ["tiny", "resnet18_8s"])
def test_network_parameter_gradients(which):
    torch.manual_seed(0)
    if which == "tiny":
        net = _TinyNet().to(DEV)
        x, mask, vertex, weights = _train_batch(2, 24, 32, 8)
    else:
        from pvnet_b200.model_repository import Resnet18_8s
        net = Resnet18_8s(ver_dim=18, seg_dim=2)
        net.load_state_dict(seeded_state_dict(net, seed=3))
        net = net.to(DEV).train()
        x, mask, vertex, weights = _train_batch(2, 64, 80, 9)
    # fp32 convolutions: the output gradients are equal, but the bilinear upsampling's backward sums with atomics in
    # no fixed order, and TF32 convolutions would amplify those last-bit differences
    with torch.backends.cudnn.flags(enabled=True, deterministic=True, benchmark=False, allow_tf32=False):
        got, ls, lv = _param_grads(net, x, mask, vertex, weights, native=True)
        want, ls_t, lv_t = _param_grads(net, x, mask, vertex, weights, native=False)
    np.testing.assert_allclose(ls.detach().cpu().numpy(), ls_t.detach().cpu().numpy(), rtol=1e-5)
    np.testing.assert_allclose(lv.detach().cpu().numpy(), lv_t.detach().cpu().numpy(), rtol=1e-5)
    assert got.keys() == want.keys() and got
    for k in got:
        torch.testing.assert_close(got[k], want[k], rtol=1e-4, atol=1e-5 * float(want[k].abs().max()) + 1e-12,
                                   msg=k)


def _output_and_targets(b, h, w, seed=11):
    rng = np.random.default_rng(seed)
    out = torch.from_numpy(rng.normal(0, 1, (b, 20, h, w)).astype(np.float32)).to(DEV).requires_grad_()
    mask = torch.from_numpy(rng.integers(0, 2, (b, h, w))).to(DEV)
    vertex = torch.from_numpy(rng.normal(0, 1, (b, 18, h, w)).astype(np.float32)).to(DEV)
    hc = torch.from_numpy(np.concatenate([rng.uniform(0, w, (b, 9, 1)), rng.uniform(0, h, (b, 9, 1)),
                                          np.ones((b, 9, 1))], 2)).to(DEV)
    return out, mask, vertex, hc, (mask > 0).float()[:, None]


def test_one_output_tensor_equals_two_slices():
    out, mask, vertex, hc, weights = _output_and_targets(2, 37, 53)
    for tgt, fn in ((vertex, nu.seg_vertex_training_losses), (hc, nu.seg_vertex_training_losses_from_keypoints)):
        one = fn(out[:, :2], out[:, 2:], mask, tgt, weights)
        assert one[0].grad_fn.next_functions[0][0] is torch.autograd.graph.get_gradient_edge(out).node
        two = fn(out[:, :2].clone(), out[:, 2:].clone(), mask, tgt, weights)         # SliceBackward x2 + add
        g1 = torch.autograd.grad(torch.mean(one[0]) + torch.mean(one[1]), out)[0]
        g2 = torch.autograd.grad(torch.mean(two[0]) + torch.mean(two[1]), out)[0]
        assert _exact(g1) == _exact(g2)
        assert all(_exact(a) == _exact(b) for a, b in zip(one, two))


@pytest.mark.parametrize("keypoints", [False, True])
def test_backward_memory(keypoints):
    out, mask, vertex, hc, weights = _output_and_targets(4, 480, 640)
    fn = nu.seg_vertex_training_losses_from_keypoints if keypoints else nu.seg_vertex_training_losses
    loss_seg, loss_vertex, _, _ = fn(out[:, :2], out[:, 2:], mask, hc if keypoints else vertex, weights)
    loss = torch.mean(loss_seg) + torch.mean(loss_vertex)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    g = torch.autograd.grad(loss, out)[0]
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - before <= out.numel() * 4 + 2 ** 20
    assert g.shape == out.shape


def test_null_loss_gradients():
    seg, mask, pred, vertex, weights, _ = case_inputs("k9_s1_binary")
    s, m, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    gs, gv = _loss_grads(3, seed=6)
    want = _torch_grads(s, p, m, t, w, gs, gv)
    for keep in (1, 0):                                                     # only loss_vertex, then only loss_seg
        sr, pr = s.clone().requires_grad_(), p.clone().requires_grad_()
        out = nu.seg_vertex_training_losses(sr, pr, m, t, w)
        got = torch.autograd.grad(out[keep], (sr, pr), (gs, gv)[keep], allow_unused=True)
        assert got[1 - keep] is None and _bits(got[keep]) == _bits(want[keep])
        base = torch.cat([s, p], 1).requires_grad_()                        # the shared tensor: zeros in the rest
        out = nu.seg_vertex_training_losses(base[:, :2], base[:, 2:], m, t, w)
        g = torch.autograd.grad(out[keep], base, (gs, gv)[keep])[0]
        parts = (g[:, :2], g[:, 2:])
        assert _bits(parts[keep]) == _bits(want[keep])
        assert _exact(parts[1 - keep]) == _exact(torch.zeros_like(parts[1 - keep]))


def test_bad_inputs():
    seg, mask, pred, vertex, weights, _ = case_inputs("k9_s1_binary")
    s, m, p, t, w = _gpu(seg, mask, pred, vertex, weights)
    hc = torch.zeros(3, 9, 3, device=DEV)
    with pytest.raises(ValueError, match="vertex requires grad"):
        nu.seg_vertex_training_losses(s, p, m, t.clone().requires_grad_(), w)
    with pytest.raises(ValueError, match="vertex_weights requires grad"):
        nu.seg_vertex_training_losses(s, p, m, t, w.clone().requires_grad_())
    with pytest.raises(ValueError, match="hcoords requires grad"):
        nu.seg_vertex_training_losses_from_keypoints(s, p, m, hc.requires_grad_(), w)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_training_losses(s.cpu().requires_grad_(), p.cpu(), m.cpu(), t.cpu(), w.cpu())
    sr = s.clone().requires_grad_()
    gls = torch.ones(3, device=DEV, requires_grad=True)
    g = torch.autograd.grad(nu.seg_vertex_training_losses(sr, p, m, t, w)[0], sr, gls, create_graph=True)[0]
    with pytest.raises(RuntimeError, match="once_differentiable"):          # no double backward
        g.sum().backward()


def test_graph_capture_and_determinism():
    out, mask, vertex, hc, weights = _output_and_targets(2, 96, 128, seed=12)

    def step(fn, tgt):
        ls, lv, _, _ = fn(out[:, :2], out[:, 2:], mask, tgt, weights)
        return torch.autograd.grad(torch.mean(ls) + torch.mean(lv), out)[0]

    for fn, tgt in ((nu.seg_vertex_training_losses, vertex), (nu.seg_vertex_training_losses_from_keypoints, hc)):
        eager = step(fn, tgt)
        assert _exact(eager) == _exact(step(fn, tgt))
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            step(fn, tgt)                                                   # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(st)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            captured = step(fn, tgt)
        graph.replay()
        torch.cuda.synchronize()
        assert _exact(captured) == _exact(eager)


class _LossModule(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = _TinyNet()

    def forward(self, x, mask, vertex, weights):
        seg, ver = self.net(x)
        loss_seg, loss_vertex, _, _ = nu.seg_vertex_training_losses(seg, ver, mask, vertex, weights)
        return loss_seg, loss_vertex


def _dp_grads(module, m, x, mask, vertex, weights):
    module.zero_grad(set_to_none=True)
    ls, lv = m(x, mask, vertex, weights)
    (torch.mean(ls) + torch.mean(lv)).backward()
    return [p.grad.clone() for p in module.parameters()], ls.detach(), lv.detach()


def test_data_parallel_one_device():
    torch.manual_seed(1)
    module = _LossModule().to(DEV)
    batch = _train_batch(4, 24, 32, 10)
    direct = _dp_grads(module, module, *batch)
    dp = _dp_grads(module, nn.DataParallel(module, device_ids=[0]), *batch)
    assert all(_exact(a) == _exact(b) for a, b in zip(direct[0], dp[0]))
    assert _exact(direct[1]) == _exact(dp[1]) and _exact(direct[2]) == _exact(dp[2])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_data_parallel_two_devices():
    torch.manual_seed(1)
    module = _LossModule().to(DEV)
    batch = _train_batch(4, 24, 32, 10)
    direct = _dp_grads(module, module, *batch)
    two = _dp_grads(module, nn.DataParallel(module, device_ids=[0, 1]), *batch)
    assert _exact(direct[1]) == _exact(two[1]) and _exact(direct[2]) == _exact(two[2])
    for a, b in zip(direct[0], two[0]):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-7)
