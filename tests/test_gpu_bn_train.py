"""Train-mode BatchNorm on the H100 (csrc/batchnorm.cu): pvnet_batchnorm_act_forward / _backward in their three forms
against oracle/bn_train_oracle.py (bit for bit: the same fixed summation order), exact fp64 and torch's own
BatchNorm2d + activation (+ add); the autograd Functions BatchNormActNHWC / BatchNormAddReluNHWC; and
Resnet18_8s.forward_train with all 25 BatchNorm layers on them."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bn_train_oracle as bo
from pvnet_b200 import conv as pc
from pvnet_b200.model_repository import Resnet18_8s

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CL = torch.channels_last
RELU, LEAKY, NONE = pc.ACT_RELU, pc.ACT_LEAKY, pc.ACT_NONE

# (form, act, b, C, H, W): every site's channel count at reduced sizes with ragged pixel counts, more than 256
# partials (the merge's lane loop), N = 2, and the large sites at their 480 x 640 batch-16 shapes
REDUCED = [(0, RELU, 2, 64, 9, 13), (1, RELU, 2, 64, 17, 11), (2, RELU, 2, 128, 9, 7), (1, RELU, 2, 128, 5, 9),
           (2, RELU, 1, 256, 6, 5), (1, RELU, 3, 256, 5, 7), (2, RELU, 2, 512, 3, 7), (1, RELU, 2, 512, 4, 3),
           (0, RELU, 2, 256, 7, 7), (0, LEAKY, 2, 128, 15, 20), (0, LEAKY, 2, 64, 13, 9), (0, LEAKY, 2, 32, 33, 40),
           (0, NONE, 3, 32, 5, 5), (0, RELU, 2, 4, 200, 170), (0, LEAKY, 1, 32, 1, 2), (1, RELU, 2, 16, 1, 1),
           (2, RELU, 1, 8, 1, 2)]
LARGE = [(0, RELU, 16, 64, 240, 320), (1, RELU, 16, 64, 120, 160), (2, RELU, 16, 128, 60, 80),
         (2, RELU, 16, 256, 60, 80), (1, RELU, 16, 512, 60, 80), (0, LEAKY, 16, 32, 240, 320),
         (0, LEAKY, 16, 32, 480, 640)]


def _module(C, seed, momentum=0.1):
    g = torch.Generator().manual_seed(seed)
    bn = torch.nn.BatchNorm2d(C, momentum=momentum).to(DEV).train()
    with torch.no_grad():
        bn.weight.copy_(torch.rand(C, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(C, generator=g) - 0.5)
        bn.running_mean.copy_(torch.randn(C, generator=g) * 0.1)
        bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    return bn


def _data(b, C, H, W, seed, mean=0.3, tied=False):
    if tied:
        # -1, 0, 1 in equal numbers per channel, 0 at pixel 0 (the kernels' shift): the fp64 sums are exact, the
        # mean is exactly 0, so with beta = 0 the pre-activation is exactly 0 wherever the value is 0
        N = b * H * W
        rng = np.random.default_rng(seed)
        v = np.stack([rng.permutation(np.arange(N) % 3 - 1) for _ in range(C)], 1).astype(np.float32)
        for c in range(C):
            k = np.flatnonzero(v[:, c] == 0)[0]
            v[[0, k], c] = v[[k, 0], c]
        return torch.from_numpy(v).reshape(b, H, W, C).permute(0, 3, 1, 2).to(DEV).contiguous(memory_format=CL)
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randn(b, C, H, W, device=DEV, generator=g) * 1.7 + mean
    return v.contiguous(memory_format=CL)


def _flat(t):
    """[b,C,H,W] -> numpy [N, C] (NHWC order)."""
    return t.detach().permute(0, 2, 3, 1).reshape(-1, t.shape[1]).cpu().numpy()


def _run(form, act, x, z, bn, bz, dy):
    """One native forward + backward through the functional layer; returns everything the checks read."""
    st = pc.BatchNormState(bn, DEV)
    sz = pc.BatchNormState(bz, DEV) if form == 2 else None
    xh, zh = pc._nhwc(x), None if z is None else pc._nhwc(z)
    y = pc.batchnorm_forward(form, act, xh, zh, st, bn.weight, bn.bias, sz, None if bz is None else bz.weight,
                             None if bz is None else bz.bias)
    dx, dz, dw, db, dwz, dbz = pc.batchnorm_backward(form, act, pc._nhwc(dy), xh, zh, st, bn.weight, sz,
                                                     None if bz is None else bz.weight)
    return dict(y=y, dx=dx, dz=dz, dw=dw, db=db, dwz=dwz, dbz=dbz, st=st, sz=sz)


def _check_stats(xs, st, bn, rm0, rv0, f):
    N = xs.shape[0]
    mean, var, invstd = bo.batch_stats(xs, bn.eps)
    saved = st.saved.cpu().numpy()
    assert np.array_equal(saved[0], mean) and np.array_equal(saved[1], var) and np.array_equal(saved[2], invstd)
    em, ev = bo.exact_stats(xs)
    ulp = lambda v: np.spacing(np.abs(np.float32(v)))  # noqa: E731
    assert (np.abs(mean.astype(np.float32).astype(np.float64) - em.astype(np.float32)) <= ulp(em)).all()
    assert (np.abs(var.astype(np.float32).astype(np.float64) - ev.astype(np.float32)) <= ulp(ev)).all()
    scale, shift = bo.scale_shift(mean, invstd, bn.weight.detach().cpu().numpy(), bn.bias.detach().cpu().numpy())
    coef = st.coef.cpu().numpy()
    assert np.array_equal(coef[0], scale) and np.array_equal(coef[1], shift)
    # the module's rule evaluated in fp32 on the native batch statistics (torch elementwise ops, no fusion)
    m32 = torch.from_numpy(mean.astype(np.float32))
    u32 = torch.from_numpy(bo.unbiased32(var, N))
    assert torch.equal(bn.running_mean.cpu(), rm0 * (1 - f) + m32 * f)
    assert torch.equal(bn.running_var.cpu(), rv0 * (1 - f) + u32 * f)
    return scale, shift, mean, invstd


def _check_case(form, act, b, C, H, W, tied=False):
    bn, bz = _module(C, 1), _module(C, 2) if form == 2 else None
    if tied:
        with torch.no_grad():
            for m in (bn, bz):
                if m is not None:
                    m.bias.zero_()
    x = _data(b, C, H, W, 3, tied=tied)
    z = None if form == 0 else _data(b, C, H, W, 4, mean=-0.2, tied=tied)
    dy = _data(b, C, H, W, 5, mean=0.0)
    rm0, rv0 = bn.running_mean.cpu().clone(), bn.running_var.cpu().clone()
    rmz0, rvz0 = (bz.running_mean.cpu().clone(), bz.running_var.cpu().clone()) if bz is not None else (None, None)
    nbt = int(bn.num_batches_tracked)
    r = _run(form, act, x, z, bn, bz, dy)
    torch.cuda.synchronize()
    assert int(bn.num_batches_tracked) == nbt + 1
    xs, dys = _flat(x), _flat(dy)
    zs = None if z is None else _flat(z)
    scale, shift, mean, invstd = _check_stats(xs, r["st"], bn, rm0, rv0, 0.1)
    sz_ = tz_ = None
    if form == 2:
        sz_, tz_, mz, invz = _check_stats(zs, r["sz"], bz, rmz0, rvz0, 0.1)
    # forward: the correctly rounded fma of the fp32 scale/shift, then the add and the activation
    pre = bo.pre_activation(xs, scale, shift, zs, sz_, tz_)
    y = _flat(r["y"])
    assert np.array_equal(y.view(np.int32), bo.act_fwd(pre, act).view(np.int32))
    # ... and within a stated bound of torch's own modules on the same input
    ref = copy.deepcopy(bn)(x)
    if form == 1:
        ref = ref + z
    elif form == 2:
        ref = ref + copy.deepcopy(bz)(z)
    ref = {NONE: lambda t: t, RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, 0.1)}[act](ref)
    # torch normalises as (x - mean) * invstd * gamma + beta with fp32 statistics: each value is off by a bounded
    # number of ulps of the terms it adds, |x*scale|, |mean*scale|, |beta| (and the same for the second operand)
    def terms(v, sc, m, beta):
        return np.abs(v * sc) + np.abs(m * sc) + np.abs(beta)
    mag = terms(xs, scale, mean, bn.bias.detach().cpu().numpy())
    if form == 1:
        mag = mag + np.abs(zs)
    elif form == 2:
        mag = mag + terms(zs, sz_, mz, bz.bias.detach().cpu().numpy())
    err = np.abs(_flat(ref).astype(np.float64) - y)
    bound = 2.0 ** -24 * 256 * mag + 1e-30
    print(f"max |native - torch| / bound = {float((err / bound).max()):.3g}")
    assert (err <= bound).all()
    # backward: bit for bit the oracle, within the stated bounds of exact fp64 for the same mask
    g = bo.masked_grad(dys, pre, act)
    Sg, Sgx = bo.backward_sums(g, xs, mean)
    coef, (dgam, dbet) = bo.backward_coef(Sg, Sgx, xs.shape[0], mean, invstd, bn.weight.detach().cpu().numpy())
    dx = _flat(r["dx"])
    assert np.array_equal(r["dw"].cpu().numpy(), dgam) and np.array_equal(r["db"].cpu().numpy(), dbet)
    assert np.array_equal(dx.view(np.int32), bo.backward_apply(g, xs, coef).view(np.int32))
    edx, edg, edb = bo.exact_backward(g, xs, bn.eps, bn.weight.detach().cpu().numpy())
    A, B, Cc = coef
    assert (np.abs(dx - edx) <= 4 * 2.0 ** -24 * (np.abs(A * g) + np.abs(B * xs) + np.abs(Cc)) + 1e-37).all()
    for ours, ex in ((dgam, edg), (dbet, edb)):
        assert (np.abs(ours.astype(np.float64) - ex) <= np.spacing(np.abs(ex.astype(np.float32)))).all()
    if form == 1:
        assert np.array_equal(_flat(r["dz"]), g)
    if form == 2:
        Sgz, Sgzz = bo.backward_sums(g, zs, mz)
        coefz, (dgz, dbz) = bo.backward_coef(Sgz, Sgzz, zs.shape[0], mz, invz, bz.weight.detach().cpu().numpy())
        assert np.array_equal(_flat(r["dz"]).view(np.int32), bo.backward_apply(g, zs, coefz).view(np.int32))
        assert np.array_equal(r["dwz"].cpu().numpy(), dgz) and np.array_equal(r["dbz"].cpu().numpy(), dbz)
    return g, pre


@pytest.mark.parametrize("form,act,b,C,H,W", REDUCED)
def test_reduced_sites_against_oracle_exact_and_torch(form, act, b, C, H, W):
    _check_case(form, act, b, C, H, W)


@pytest.mark.parametrize("form,act,b,C,H,W", LARGE)
def test_large_sites_at_full_resolution(form, act, b, C, H, W):
    _check_case(form, act, b, C, H, W)


@pytest.mark.parametrize("form,act", [(0, RELU), (0, LEAKY), (1, RELU), (2, RELU)])
def test_masks_at_exact_zeros_follow_torch(form, act):
    # tied data: pre-activations exactly 0; the oracle's rule, which _check_case holds the kernels to bit for bit,
    # is torch's (shown on the CPU against fp64 autograd)
    _, pre = _check_case(form, act, 2, 16, 12, 10, tied=True)
    assert (pre == 0).sum() > 0
    # torch's own modules on a frozen BatchNorm (running mean 0, beta 0), where both sides produce exact zeros
    bn = _module(16, 7)
    with torch.no_grad():
        bn.bias.zero_()
        bn.running_mean.zero_()
    bn.eval()
    x = _data(2, 16, 12, 10, 8, tied=True)
    skip = torch.zeros_like(x)
    dy = _data(2, 16, 12, 10, 9)
    fn = {RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, 0.1)}[act]
    xn, xt = x.clone().requires_grad_(), x.clone().requires_grad_()
    if form == 0:
        ours, ref = pc.bn_act(bn, xn, act), fn(bn(xt))
    else:
        ours, ref = pc.bn_add_relu(bn, xn, skip), F.relu(bn(xt) + skip)
    ours.backward(dy)
    ref.backward(dy)
    zero = x == 0
    assert zero.any()
    assert torch.allclose(xn.grad[zero], xt.grad[zero], rtol=1e-6, atol=0)
    if act == RELU:
        assert (xn.grad[zero] == 0).all()
    else:
        assert (xn.grad[zero] != 0).any()


@pytest.mark.parametrize("momentum", [0.1, None])
def test_module_semantics_momentum_none_and_frozen(momentum):
    bn = _module(32, 11, momentum)
    x = _data(2, 32, 8, 12, 12)
    for step in range(1, 4):
        rm0, rv0 = bn.running_mean.cpu().clone(), bn.running_var.cpu().clone()
        y = pc.bn_act(bn, x, RELU)
        f = momentum if momentum is not None else 1.0 / step
        assert int(bn.num_batches_tracked) == step
        xs = _flat(x)
        mean, var, _ = bo.batch_stats(xs, bn.eps)
        assert torch.equal(bn.running_mean.cpu(), rm0 * (1 - f) + torch.from_numpy(mean.astype(np.float32)) * f)
        assert torch.equal(bn.running_var.cpu(), rv0 * (1 - f) + torch.from_numpy(bo.unbiased32(var, xs.shape[0])) * f)
    # frozen (eval): running statistics normalise, nothing is updated, the backward has no statistic terms
    bn.eval()
    before = [t.clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]
    xg = x.clone().requires_grad_()
    y = pc.bn_act(bn, xg, RELU)
    dy = _data(2, 32, 8, 12, 13)
    y.backward(dy)
    assert all(torch.equal(a, b) for a, b in zip(before, (bn.running_mean, bn.running_var, bn.num_batches_tracked)))
    xr = x.clone().requires_grad_()
    ref = F.relu(copy.deepcopy(bn)(xr))
    ref.backward(dy)
    assert torch.allclose(y, ref, rtol=1e-5, atol=1e-6)
    assert torch.allclose(xg.grad, xr.grad, rtol=1e-5, atol=1e-6)
    # track_running_stats=False: batch statistics in both modes, no buffers
    nb = torch.nn.BatchNorm2d(32, track_running_stats=False).to(DEV).eval()
    assert torch.allclose(pc.bn_act(nb, x, RELU), F.relu(nb(x)), rtol=1e-5, atol=1e-5)


def test_autograd_functions_parameters_layouts_and_node_names():
    bn, bd = _module(64, 21), _module(64, 22)
    a = _data(2, 64, 10, 12, 23).requires_grad_()
    c = _data(2, 64, 10, 12, 24).requires_grad_()
    y = pc.bn_add_relu(bn, a, c, bd)
    assert type(y.grad_fn).__name__ == "BatchNormAddReluNHWCBackward" and y.is_contiguous(memory_format=CL)
    dy = _data(2, 64, 10, 12, 25)
    y.backward(dy)
    grads = [t.grad.clone() for t in (a, c, bn.weight, bn.bias, bd.weight, bd.bias)]
    # NCHW-contiguous inputs and gradient: the same values
    for t in (a, c, bn.weight, bn.bias, bd.weight, bd.bias):
        t.grad = None
    bn2, bd2 = _module(64, 21), _module(64, 22)
    a2, c2 = a.detach().contiguous().requires_grad_(), c.detach().contiguous().requires_grad_()
    y2 = pc.bn_add_relu(bn2, a2, c2, bd2)
    y2.backward(dy.contiguous())
    assert torch.equal(y, y2)
    for g1, g2 in zip(grads, [t.grad for t in (a2, c2, bn2.weight, bn2.bias, bd2.weight, bd2.bias)]):
        assert torch.equal(g1, g2)
    assert torch.equal(bn.running_var, bn2.running_var) and torch.equal(bd.running_mean, bd2.running_mean)


def test_run_to_run_identical_at_convraw_batch16():
    b, C, H, W = 16, 32, 480, 640
    x = _data(b, C, H, W, 31)
    dy = _data(b, C, H, W, 32)
    outs = []
    for _ in range(2):
        bn = _module(C, 33)
        r = _run(0, LEAKY, x, None, bn, None, dy)
        outs.append([r["y"], r["dx"], r["dw"], r["db"], bn.running_mean, bn.running_var])
    for u, v in zip(*outs):
        assert torch.equal(u, v)


def test_cuda_graph_capture_and_replay():
    C = 128
    bn, bd = _module(C, 41), _module(C, 42)
    x, z, dy = (_data(4, C, 20, 24, s) for s in (43, 44, 45))
    xs, zs, dys = x.clone(), z.clone(), dy.clone()

    def step():
        st, sd = pc.BatchNormState(bn, DEV), pc.BatchNormState(bd, DEV)
        y = pc.batchnorm_forward(2, RELU, pc._nhwc(xs), pc._nhwc(zs), st, bn.weight, bn.bias, sd, bd.weight, bd.bias)
        return (y,) + pc.batchnorm_backward(2, RELU, pc._nhwc(dys), pc._nhwc(xs), pc._nhwc(zs), st, bn.weight, sd,
                                            bd.weight)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    # replay on new data against an eager call with the same buffers
    for seed in (46, 47):
        xs.copy_(_data(4, C, 20, 24, seed))
        zs.copy_(_data(4, C, 20, 24, seed + 10))
        state0 = [t.clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]
        graph.replay()
        torch.cuda.synchronize()
        got = [t.clone() for t in outs if t is not None] + [bn.running_mean.clone()]
        with torch.no_grad():
            bn.running_mean.copy_(state0[0])
            bn.running_var.copy_(state0[1])
            bn.num_batches_tracked.copy_(state0[2])
        eager = [t for t in step() if t is not None] + [bn.running_mean]
        for u, v in zip(got, eager):
            assert torch.equal(u, v)


def test_bad_arguments_raise():
    bn = _module(32, 51)
    with pytest.raises(ValueError, match="channels"):
        pc.bn_act(bn, _data(1, 16, 4, 4, 52), RELU)
    with pytest.raises(ValueError):
        pc.bn_add_relu(bn, _data(1, 32, 4, 4, 53), _data(1, 32, 4, 2, 54))
    with pytest.raises(ValueError, match="float32"):
        pc.bn_act(bn, _data(1, 32, 4, 4, 55).double(), RELU)
    bn6 = torch.nn.BatchNorm2d(6).to(DEV).train()
    with pytest.raises(RuntimeError, match="multiple of 4"):
        pc.bn_act(bn6, torch.zeros(1, 6, 4, 4, device=DEV), RELU)
    with pytest.raises(RuntimeError, match="more than one value"):
        pc.bn_act(bn, _data(1, 32, 1, 1, 56), RELU)


def test_tensor_beyond_2_31_bytes():
    b, C, H, W = 56, 32, 480, 640            # 2.2 GB per tensor: element offsets past 2^31 bytes
    assert b * C * H * W * 4 > 2 ** 31
    bn = _module(C, 61)
    x = torch.empty(b, C, H, W, device=DEV, memory_format=CL)
    x.normal_(0.5, 2.0, generator=torch.Generator(device=DEV).manual_seed(62))
    st = pc.BatchNormState(bn, DEV)
    xh = pc._nhwc(x)
    y = pc.batchnorm_forward(0, LEAKY, xh, None, st, bn.weight, bn.bias)
    mean64 = x.double().mean((0, 2, 3))
    assert torch.allclose(st.saved[0], mean64, rtol=0, atol=1e-9)
    scale, shift = st.coef.cpu().numpy()
    tail = _flat(x[-1:, :, -4:])           # the last pixels, read and written through 64-bit offsets
    assert np.array_equal(_flat(y[-1:, :, -4:]), bo.act_fwd(bo.fma32(tail, scale, shift), LEAKY))
    dy = torch.ones_like(y)
    dx, _, dw, db, _, _ = pc.batchnorm_backward(0, LEAKY, pc._nhwc(dy), xh, None, st, bn.weight)
    gsum = torch.where(y > 0, 1.0, float(np.float32(0.1))).double().sum((0, 2, 3))
    assert torch.allclose(db.double(), gsum, rtol=1e-6)
    assert torch.isfinite(dx[-1, :, -1]).all() and torch.isfinite(dw).all()


def _node_names(t):
    names, seen, stack = [], set(), [t.grad_fn]
    while stack:
        n = stack.pop()
        if n is None or n in seen:
            continue
        seen.add(n)
        names.append(type(n).__name__)
        stack += [f for f, _ in n.next_functions]
    return names


def test_forward_train_graph_nodes():
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    seg, _ = net.forward_train(torch.randn(1, 3, 64, 96, device=DEV))
    names = _node_names(seg)
    for bad in ("CudnnBatchNormBackward0", "NativeBatchNormBackward0", "ReluBackward0", "LeakyReluBackward0",
                "AddBackward0"):
        assert bad not in names, bad
    assert names.count("BatchNormActNHWCBackward") == 14
    assert names.count("BatchNormAddReluNHWCBackward") == 8
    assert names.count("Upsample2xCatNHWCBackward") == 3 and names.count("CatBackward0") == 1


def test_forward_train_frozen_batchnorms_keep_their_buffers():
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    frozen = [net.resnet18_8s.layer2[0].downsample[1], net.conv4s[1]]
    for m in frozen:
        m.eval()
    before = [[t.clone() for t in m.buffers()] for m in frozen]
    seg, ver = net.forward_train(torch.randn(2, 3, 64, 96, device=DEV))
    (seg.sum() + ver.square().mean()).backward()
    for m, bufs in zip(frozen, before):
        for a, b in zip(m.buffers(), bufs):
            assert torch.equal(a, b)
        assert m.weight.grad is not None and torch.isfinite(m.weight.grad).all()
    assert int(net.conv8s[1].num_batches_tracked) == 1


def _torch_bn_act(bn, x, act=NONE):
    y = bn(x)
    return {NONE: lambda t: t, RELU: F.relu, LEAKY: lambda t: F.leaky_relu(t, 0.1)}[act](y)


def _torch_bn_add_relu(bn, a, skip, bn_skip=None):
    return F.relu(bn(a) + (skip if bn_skip is None else bn_skip(skip)))


def test_forward_train_against_torch_modules(monkeypatch):
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    mod, ref64 = copy.deepcopy(net), copy.deepcopy(net).double()
    x = torch.randn(2, 3, 128, 160, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    out_n = net.forward_train(x)
    with torch.no_grad():
        out_64 = ref64._forward_torch(x.double())
    monkeypatch.setattr(pc, "bn_act", _torch_bn_act)
    monkeypatch.setattr(pc, "bn_add_relu", _torch_bn_add_relu)
    out_t = mod.forward_train(x)
    # Both copies share the TF32 convolutions; they differ only in how BatchNorm rounds, which the TF32 rounding of
    # the next convolution's operands amplifies.  The bound per element: 3x the largest distance of the torch-module
    # copy from the fp64 graph on the same tensor (how far TF32 alone moves it), plus 1e-6 of the tensor's scale.
    rows = [("seg", out_n[0], out_t[0], out_64[0]), ("ver", out_n[1], out_t[1], out_64[1])]
    bn_, bt, b64 = dict(net.named_buffers()), dict(mod.named_buffers()), dict(ref64.named_buffers())
    rows += [(k, bn_[k], bt[k], b64[k]) for k in bn_ if "running" in k]
    for what, n, t, r in rows:
        bound = 3 * float((t.double() - r).abs().max()) + 1e-6 * float(r.abs().max())
        err = float((n.double() - t.double()).abs().max())
        print(f"{what}: max |native - torch modules| {err:.3e}, bound {bound:.3e}")
        assert err <= bound, what
    for k in bn_:
        if k.endswith("num_batches_tracked"):
            assert torch.equal(bn_[k], bt[k]), k


class _Wrapper(torch.nn.Module):
    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, x):
        seg, ver = self.net.forward_train(x)
        return seg.sum() + ver.square().mean()


def _dp_matches_direct(device_ids):
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=18, seg_dim=2).to(DEV).train()
    twin = copy.deepcopy(net)
    x = torch.randn(2 * len(device_ids), 3, 64, 96, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    torch.nn.DataParallel(_Wrapper(net), device_ids=device_ids)(x).sum().backward()
    _Wrapper(twin)(x).backward()
    return net, twin


def test_data_parallel_single_device_identical():
    net, twin = _dp_matches_direct([0])
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert torch.equal(p, q) and torch.equal(p.grad, q.grad), k
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_data_parallel_two_devices_runs_and_updates_buffers():
    net, twin = _dp_matches_direct([0, 1])
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert torch.equal(p, q), k
    for k, p in net.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
