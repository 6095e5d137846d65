"""CPU: the gradient oracle of the training losses (oracle/loss_grad_oracle.py) against torch's CPU autograd through the
reference's expressions, and the host layer's names and refusals (pvnet_b200/net_utils.py, the lib.utils.net_utils
shim, include/pvnet_b200.h)."""
import os
import re

import numpy as np
import pytest
import torch
from torch import nn

from oracle import loss_grad_oracle as lgo
from pvnet_b200 import _native
from pvnet_b200 import net_utils as nu
from tests.loss_cases import CASES, canon_nan, case_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("seg_vertex_training_losses", "seg_vertex_training_losses_from_keypoints")


def _torch_smooth_l1(pred, tgt, w):
    b, ver_dim = pred.shape[:2]
    diff = w * (pred - tgt)
    abs_diff = torch.abs(diff)
    sign = (abs_diff < 1.).detach().float()
    in_loss = torch.pow(diff, 2) * (1. / 2.) * sign + (abs_diff - 0.5) * (1. - sign)
    return torch.sum(in_loss.view(b, -1), 1) / (ver_dim * torch.sum(w.view(b, -1), 1) + 1e-3)


@pytest.mark.parametrize("name", list(CASES))
def test_smooth_l1_grad_oracle_equals_torch_cpu_autograd(name):
    _, _, pred, vertex, weights, _ = case_inputs(name)
    p = torch.from_numpy(pred).requires_grad_()
    t, w = torch.from_numpy(vertex), torch.from_numpy(weights)
    gv = np.random.default_rng(1).uniform(0.25, 2, pred.shape[0]).astype(np.float32)
    want = torch.autograd.grad(_torch_smooth_l1(p, t, w), p, torch.from_numpy(gv))[0]
    b, vd = pred.shape[:2]
    den = (vd * torch.sum(w.view(b, -1), 1) + 1e-3).numpy()
    # torch's own denominator: the elementwise sequence is torch's bit for bit (NaN positions compared, not payloads)
    assert canon_nan(lgo.smooth_l1_grad(pred, vertex, weights, gv, den=den)).tobytes() == canon_nan(want).tobytes()
    if CASES[name][6] == "binary":        # 0/1 weights: torch's fp32 sum is exact, so the forward's denominator too
        assert np.array_equal(den, lgo.vertex_denominator(weights, vd))
        assert canon_nan(lgo.smooth_l1_grad(pred, vertex, weights, gv)).tobytes() == canon_nan(want).tobytes()


def test_smooth_l1_grad_hand_computed():
    # w = 1, vd = 1, four pixels: diffs 0.5 (inside), -2 (outside), 0 and NaN; gi = 1 / (4 + 1e-3)
    p = np.array([0.5, -2.0, 0.0, np.nan], np.float32).reshape(1, 1, 1, 4)
    w = np.ones((1, 1, 1, 4), np.float32)
    g = lgo.smooth_l1_grad(p, np.zeros_like(p), w, np.ones(1, np.float32))[0, 0, 0]
    gi = np.float32(1) / (np.float32(4) + np.float32(1e-3))
    assert g[0] == np.float32(gi * np.float32(0.5)) * np.float32(1.0)
    assert g[1] == -gi and g[2] == 0 and np.isnan(g[3])


def test_cpu_mean_backward_divides():
    """The term that differs between the devices: torch's CPU MeanBackward divides by N, its CUDA one multiplies by
    the float reciprocal of N (pinned in tests/test_gpu_train_losses.py); the oracle restates the CUDA sequence."""
    n = 37 * 53
    gs = torch.from_numpy(np.random.default_rng(4).uniform(0.1, 10, 4096).astype(np.float32))
    x = torch.zeros(4096, n, requires_grad=True)
    g = torch.autograd.grad(x.mean(1), x, gs)[0][:, 0].numpy()
    assert g.tobytes() == (gs.numpy() / np.float32(n)).tobytes()
    assert (g != gs.numpy() * (np.float32(1) / np.float32(n))).any()


@pytest.mark.parametrize("name", list(CASES))
def test_cross_entropy_grad_oracle_against_torch_cpu(name):
    """Within 2^-20 * gs / N of torch's CPU autograd: the CPU's MeanBackward divides, and its log-softmax backward
    and exp / log are its own."""
    seg, mask, *_ = case_inputs(name)
    mask = mask.copy()
    mask[0, :5] = -100
    s = torch.from_numpy(seg).requires_grad_()
    gs = np.random.default_rng(2).uniform(0.25, 2, seg.shape[0]).astype(np.float32)
    loss = nn.CrossEntropyLoss(reduction="none")(s, torch.from_numpy(mask))
    want = canon_nan(torch.autograd.grad(loss.view(loss.shape[0], -1).mean(1), s, torch.from_numpy(gs))[0])
    got = canon_nan(lgo.cross_entropy_grad(seg, mask, gs))
    assert np.array_equal(np.isnan(got), np.isnan(want))
    bound = (2.0 ** -20 * gs / (seg.shape[2] * seg.shape[3]))[:, None, None, None]
    assert (np.abs(np.nan_to_num(got) - np.nan_to_num(want)) <= bound).all()


def test_cross_entropy_grad_invalid_targets():
    seg, mask, *_ = case_inputs("k17_s05_c3")
    bad = mask.copy()
    bad[1, 7, 11] = 3
    g = lgo.cross_entropy_grad(seg, bad, np.ones(2, np.float32))
    assert np.isnan(g[1]).all() and not np.isnan(g[0]).any()


def test_public_names_header_and_bindings():
    from lib.utils import net_utils as shim
    header = open(os.path.join(ROOT, "include", "pvnet_b200.h")).read()
    for n in NEW:
        assert n in shim.__all__ and getattr(shim, n) is getattr(nu, n)
    for sym in ("pvnet_seg_vertex_losses_backward", "pvnet_seg_vertex_losses_keypoints_backward"):
        assert re.search(r"PVNET_API\s+int\s+" + sym + r"\s*\(", header)
        assert sym in _native.SIGNATURES


def test_cpu_tensors_raise():
    s, p, t = torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 4, 4), torch.zeros(1, 2, 4, 4)
    m, w = torch.zeros(1, 4, 4, dtype=torch.int64), torch.zeros(1, 1, 4, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_training_losses(s.requires_grad_(), p, m, t, w)
    with pytest.raises(RuntimeError, match="CUDA"):
        nu.seg_vertex_training_losses_from_keypoints(s, p, m, torch.zeros(1, 1, 3), w)
