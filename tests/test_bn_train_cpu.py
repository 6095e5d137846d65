"""CPU: oracle/bn_train_oracle.py (the fixed-order restatement of csrc/batchnorm.cu) against exact fp64 statistics and
torch's CPU float64 autograd, and the native BatchNorm's argument checks, none of which needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import bn_train_oracle as bo
from pvnet_b200 import _native
from pvnet_b200 import conv as pc


def _ulp32(v):
    return np.spacing(np.abs(np.asarray(v, np.float32)))


@pytest.mark.parametrize("N,C,mean,sigma", [(2, 4, 0.0, 1.0), (1000, 8, 1e3, 1e-2), (70001, 12, -3e4, 0.5),
                                            (4096, 4, 5e2, 1e-3)])
def test_fixed_order_statistics_within_one_ulp_of_exact(N, C, mean, sigma):
    rng = np.random.default_rng(N + C)
    x = (mean + sigma * rng.standard_normal((N, C))).astype(np.float32)
    m, v, _ = bo.batch_stats(x, 1e-5)
    em, ev = bo.exact_stats(x)
    assert (np.abs(m.astype(np.float32).astype(np.float64) - em.astype(np.float32)) <= _ulp32(em)).all()
    assert (np.abs(v.astype(np.float32).astype(np.float64) - ev.astype(np.float32)) <= _ulp32(ev)).all()


def test_merge_order_is_lanes_then_tree():
    # 600 partials: lane t sums t, t+256, t+512; the tree halves 256 lanes
    rng = np.random.default_rng(1)
    p = rng.standard_normal((600, 1)) * 10.0 ** rng.integers(-8, 8, (600, 1))
    lane = [0.0] * 256
    for k in range(600):
        lane[k % 256] = lane[k % 256] + float(p[k, 0])
    s = 128
    while s:
        for i in range(s):
            lane[i] = lane[i] + lane[i + s]
        s //= 2
    assert bo.merge(p)[0] == lane[0]


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(2)
    a, b, c = (rng.standard_normal(200000).astype(np.float32) for _ in range(3))
    got = bo.fma32(a, b, c)
    exact = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)   # within 2^-53: rounding to fp32
    assert (np.abs(got.astype(np.float64) - exact) <= 0.5 * _ulp32(exact) * (1 + 2.0 ** -20) + 1e-45).all()
    # a constructed tie: fp64 sum exactly between two fp32 values, the exact value just above it
    one = np.float32(1.0)
    half_ulp = 2.0 ** -24
    a1, b1 = np.float32(1 + 2.0 ** -23), np.float32(1 + 2.0 ** -23)            # a*b = 1 + 2^-22 + 2^-46
    c1 = np.float32(half_ulp - 2.0 ** -22)                                     # sum = 1 + 2^-24 + 2^-46
    assert bo.fma32(a1, b1, c1) == np.nextafter(one, np.float32(2))


def _module(C, act):
    bn = torch.nn.BatchNorm2d(C).double().train()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    return bn


@pytest.mark.parametrize("form,act", [(0, bo.ACT_NONE), (0, bo.ACT_RELU), (0, bo.ACT_LEAKY), (1, bo.ACT_RELU),
                                      (2, bo.ACT_RELU)])
def test_oracle_gradients_match_torch_fp64_autograd(form, act):
    torch.manual_seed(form * 3 + act)
    b, C, H, W = 3, 8, 7, 5
    bn, bz = _module(C, act), _module(C, act)
    x = (torch.randn(b, C, H, W) * 2 + 3).float().double().requires_grad_()
    z = torch.randn(b, C, H, W).float().double().requires_grad_()
    dy = torch.randn(b, C, H, W).float().double()
    pre = bn(x)
    if form == 1:
        pre = pre + z
    elif form == 2:
        pre = pre + bz(z)
    y = {bo.ACT_NONE: lambda t: t, bo.ACT_RELU: torch.relu,
         bo.ACT_LEAKY: lambda t: torch.nn.functional.leaky_relu(t, 0.1)}[act](pre)
    params = [x, bn.weight, bn.bias] + ([z] if form else []) + ([bz.weight, bz.bias] if form == 2 else [])
    grads = torch.autograd.grad(y, params, dy)

    def nhwc(t):
        return t.detach().permute(0, 2, 3, 1).reshape(-1, C).numpy()
    xs, zs = nhwc(x).astype(np.float32), nhwc(z).astype(np.float32)
    # the mask from torch's own fp64 pre-activation (the fp32 one can differ right at zero)
    g = bo.masked_grad(nhwc(dy).astype(np.float32), nhwc(pre), act)
    N = xs.shape[0]

    def one(bnm, v):
        mean, var, invstd = bo.batch_stats(v, bnm.eps)
        Sg, Sgx = bo.backward_sums(g, v, mean)
        coef, (dg, db) = bo.backward_coef(Sg, Sgx, N, mean, invstd, bnm.weight.detach().numpy())
        return bo.backward_apply(g, v, coef), dg, db, coef

    def close(ours, ref, scale):
        ref = np.asarray(ref)
        assert np.abs(ours.astype(np.float64) - ref).max() <= 1e-5 * scale, np.abs(ours - ref).max()
    dx, dg, db, coef = one(bn, xs)
    close(dx, nhwc(grads[0]), np.abs(nhwc(grads[0])).max() + 1)
    close(dg, grads[1].numpy(), np.abs(grads[1].numpy()).max() + 1)
    close(db, grads[2].numpy(), np.abs(grads[2].numpy()).max() + 1)
    if form == 1:
        close(g, nhwc(grads[3]), 1)
    if form == 2:
        dz, dgz, dbz, _ = one(bz, zs)
        close(dz, nhwc(grads[3]), np.abs(nhwc(grads[3])).max() + 1)
        close(dgz, grads[4].numpy(), np.abs(grads[4].numpy()).max() + 1)
        close(dbz, grads[5].numpy(), np.abs(grads[5].numpy()).max() + 1)
    # the analytic fp64 backward agrees with autograd too
    edx, edg, edb = bo.exact_backward(g, xs, bn.eps, bn.weight.detach().numpy())
    close(edx, nhwc(grads[0]), np.abs(nhwc(grads[0])).max() + 1)
    close(edg, grads[1].numpy(), np.abs(grads[1].numpy()).max() + 1)


def test_frozen_backward_has_no_statistic_terms():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((300, 4)).astype(np.float32)
    g = rng.standard_normal((300, 4)).astype(np.float32)
    rm, rv = np.array([0.1, -0.2, 0.3, 0.0]), np.array([1.0, 2.0, 0.5, 1.5])
    inv = bo.invstd_of(rv.astype(np.float32), 1e-5)
    Sg, Sgx = bo.backward_sums(g, x, rm.astype(np.float32).astype(np.float64))
    (A, B, Cc), _ = bo.backward_coef(Sg, Sgx, 300, rm, inv, None, batch_stats=False)
    assert (B == 0).all() and (Cc == 0).all()
    edx, _, _ = bo.exact_backward(g, x, 1e-5, None, False, rm.astype(np.float32), rv.astype(np.float32))
    assert np.allclose(bo.backward_apply(g, x, (A, B, Cc)), edx, rtol=1e-6, atol=1e-7)


def test_running_update_rule():
    r = np.array([1.0, -2.0, 0.5], np.float32)
    s = np.array([0.25, 3.0, -1.0], np.float32)
    t = torch.from_numpy(r) * (1 - 0.1) + torch.from_numpy(s) * 0.1
    assert np.array_equal(bo.running_update(r, s, 0.1), t.numpy())
    assert bo.unbiased32(np.array([2.0]), 2)[0] == np.float32(4.0)


def test_native_argument_checks_without_gpu():
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_batchnorm_workspace_bytes(0, 32, 1000, ctypes.byref(n)) == 0 and n.value >= 2 * 32 * 4 * 8
    assert L.pvnet_batchnorm_workspace_bytes(2, 32, 1000, ctypes.byref(n)) == 0 and n.value >= 4 * 32 * 4 * 8
    assert L.pvnet_batchnorm_workspace_bytes(3, 32, 1000, ctypes.byref(n)) == -1
    assert L.pvnet_batchnorm_workspace_bytes(0, 30, 1000, ctypes.byref(n)) == -1
    assert L.pvnet_batchnorm_workspace_bytes(0, 2048, 1000, ctypes.byref(n)) == -1
    p = _native.BatchNormParams(None, None, None, None, 1, 0.1, 1e-5, 256, 256)
    fake = ctypes.c_void_p(1 << 20)
    args = lambda form, act, x, z, npix, C: (form, act, x, z, npix, C, ctypes.byref(p), None, fake, fake,  # noqa
                                             1 << 30, None)
    assert L.pvnet_batchnorm_act_forward(*args(0, 1, None, None, 100, 32)) == -1
    assert b"null" in L.pvnet_last_error()
    assert L.pvnet_batchnorm_act_forward(*args(0, 3, fake, None, 100, 32)) == -1          # bad activation
    assert L.pvnet_batchnorm_act_forward(*args(1, 2, fake, fake, 100, 32)) == -1          # tails end in ReLU
    assert L.pvnet_batchnorm_act_forward(*args(1, 1, fake, None, 100, 32)) == -1          # skip missing
    assert L.pvnet_batchnorm_act_forward(*args(2, 1, fake, fake, 100, 32)) == -1          # second BatchNorm missing
    assert L.pvnet_batchnorm_act_forward(*args(0, 1, ctypes.c_void_p((1 << 20) + 4), None, 100, 32)) == -1
    assert b"aligned" in L.pvnet_last_error()
    assert L.pvnet_batchnorm_act_forward(*args(0, 1, fake, None, 0, 32)) == -1
    assert L.pvnet_batchnorm_act_forward(*args(0, 1, fake, None, 1 << 34, 32)) == -1      # workspace too small
    assert b"workspace" in L.pvnet_last_error()
    assert L.pvnet_batchnorm_act_forward(*args(0, 1, fake, None, 1 << 50, 32)) == -1      # beyond the grid's reach
    assert b"too large" in L.pvnet_last_error()
    q = _native.BatchNormParams(None, None, None, None, 0, 0.1, 1e-5, 256, 256)           # running stats missing
    assert L.pvnet_batchnorm_act_forward(0, 1, fake, None, 100, 32, ctypes.byref(q), None, fake, fake, 1 << 30,
                                         None) == -1
    assert b"running" in L.pvnet_last_error()


def test_host_layer_checks_without_gpu():
    bn = torch.nn.BatchNorm2d(8).train()
    with pytest.raises(ValueError, match="CUDA"):
        pc.bn_act(bn, torch.zeros(2, 8, 4, 4), pc.ACT_RELU)
    assert int(bn.num_batches_tracked) == 0, "a refused call must not count a batch"
    with pytest.raises(ValueError, match="activation"):
        pc.act_of(torch.nn.LeakyReLU(0.2))
    assert pc.act_of(torch.nn.ReLU(True)) == pc.ACT_RELU and pc.act_of(torch.nn.LeakyReLU(0.1, True)) == pc.ACT_LEAKY
    with pytest.raises(ValueError):
        pc.bn_add_relu(bn, torch.zeros(2, 8, 4, 4), torch.zeros(2, 8, 4, 4))
