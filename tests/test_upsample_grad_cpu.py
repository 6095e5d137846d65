"""CPU: the bilinear x2 upsampling backward (k_upsample2x_backward, pvnet_b200/csrc/backbone_aux.cu) as restated in
oracle/upsample_oracle.py.  (a) The kernel's window rule -- candidates 2i-2 ... 2i+3 tested with ATen's own float index
expressions -- finds exactly the (output, slot) pairs that ATen's forward indexing sends to each input index, for
every size 1 ... 1024.  (b) The gather in the kernel's order is bit for bit a plain fp32 scatter over ATen's terms in
that order, and within fp32 rounding of the fp64 adjoint."""
import numpy as np
import pytest

from oracle import upsample_oracle as uo

F32 = np.float32


def test_window_rule_matches_aten_indexing_for_every_size():
    n_edge = 0
    for n in range(1, 1025):
        brute = uo.window_brute(n)
        table = uo.window_table(n)
        for i in range(n):
            rule = uo.window_rule(n, i, table)
            assert [(o, s) for o, s, _ in rule] == [(o, s) for o, s, _ in brute[i]], (n, i)
            assert all(a[2] == b[2] for a, b in zip(rule, brute[i])), (n, i)
        # the interior pattern: rows 2i-1, 2i through slot 1, rows 2i+1, 2i+2 through slot 0, nothing from 2i-2, 2i+3
        _, hit0, hit1, _, _ = table
        pat = (~hit0[:, 0] & ~hit1[:, 0] & hit1[:, 1] & ~hit0[:, 1] & hit1[:, 2] & ~hit0[:, 2] & hit0[:, 3] & ~hit1[:, 3]
               & hit0[:, 4] & ~hit1[:, 4] & ~hit0[:, 5] & ~hit1[:, 5])
        n_edge += int((~pat).sum())
        if n >= 3:
            assert not pat[0] and not pat[n - 1]
    assert n_edge < 4 * 1024, "the general path is for the borders only"


@pytest.mark.parametrize("n", [1, 2, 3, 60, 80, 120, 160, 240, 320])
def test_window_at_small_and_stage_sizes(n):
    """h = 1: the output pair feeds input 0 through both slots of both outputs (i0p = 0, l1 = 0); stage sizes: every
    input index gets the four outputs 2i-1 ... 2i+2 away from the borders."""
    brute = uo.window_brute(n)
    total = 0
    for i in range(n):
        rule = uo.window_rule(n, i)
        assert [(o, s) for o, s, _ in rule] == [(o, s) for o, s, _ in brute[i]]
        total += len(rule)
        if 1 < i < n - 2:
            assert [o for o, _, _ in rule] == [2 * i - 1, 2 * i, 2 * i + 1, 2 * i + 2]
    assert total == 2 * (2 * n), "every output contributes two terms along each axis"
    if n == 1:
        assert [(o, s) for o, s, _ in uo.window_rule(1, 0)] == [(0, 0), (0, 1), (1, 0), (1, 1)]


@pytest.mark.parametrize("b,h,w,C", [(1, 1, 1, 4), (2, 1, 5, 4), (1, 2, 3, 8), (2, 3, 7, 4), (1, 13, 9, 4),
                                     (1, 15, 20, 4)])
def test_gather_equals_scatter_and_adjoint(b, h, w, C):
    rng = np.random.default_rng(h * 1000 + w * 10 + C)
    dy = rng.standard_normal((b, 2 * h, 2 * w, C)).astype(F32)
    dx = uo.upsample2x_backward(dy)
    ref = uo.upsample2x_backward_scatter(dy)
    assert np.array_equal(dx.view(np.int32), ref.view(np.int32)), "gather differs from the ordered fp32 scatter"
    # fp64 adjoint: <U x, g> = <x, U^T g>, U^T g = Uh^T G Uw
    uh, uw = uo.interp_matrix(h), uo.interp_matrix(w)
    dx64 = np.einsum("yi,xj,byxc->bijc", uh, uw, dy.astype(np.float64))
    absb = np.einsum("yi,xj,byxc->bijc", np.abs(uh), np.abs(uw), np.abs(dy).astype(np.float64))
    # at most 16 terms, each with two roundings, plus 15 additions
    assert (np.abs(dx - dx64) <= 40 * np.finfo(F32).eps * absb + 1e-30).all()
    x = rng.standard_normal((b, h, w, C))
    ux = np.einsum("yi,xj,bijc->byxc", uh, uw, x)
    assert np.isclose((ux * dy).sum(), (x * dx64).sum(), rtol=1e-12, atol=1e-9)
