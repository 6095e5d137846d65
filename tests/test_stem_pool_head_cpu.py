"""CPU: the restatements behind the training step's stem, max-pool and head (oracle/stem_pool_head_oracle.py) against
torch's own definitions -- the stem's space-to-depth weight-gradient fold against conv2d_weight in fp64, the max-pool
rule and gradient against torch's CPU max_pool2d, the head's fmaf chains and fixed-order sums against fp64."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_weight

from oracle import stem_pool_head_oracle as so
from pvnet_b200 import conv as pc

U32 = 2.0 ** -24


def test_stem_fold_map_is_a_bijection_onto_the_7x7_weights():
    m = so.stem_fold_map()
    assert len(m) == 147
    assert len({(c, kh, kw) for *_, c, kh, kw in m}) == 147
    assert len({(ty, tx, ch) for ty, tx, ch, *_ in m}) == 147
    idx = pc.stem_s2d_index().reshape(4, 4, 16)
    for ty, tx, ch, c, kh, kw in m:
        assert int(idx[ty, tx, ch]) == c * 49 + kh * 7 + kw
    assert int((idx == 147).sum()) == 256 - 147


def test_training_pack_equals_the_eval_pack():
    w = torch.randn(64, 3, 7, 7, generator=torch.Generator().manual_seed(0))
    assert torch.equal(pc.pack_stem_s2d_train(w), pc.pack_stem_s2d(w))


@pytest.mark.parametrize("b,H,W", [(2, 16, 22), (1, 10, 6), (3, 8, 8)])
def test_stem_weight_gradient_fold_equals_conv2d_weight(b, H, W):
    g = torch.Generator().manual_seed(H * W + b)
    x = torch.randn(b, 3, H, W, dtype=torch.float64, generator=g)
    dy = torch.randn(b, 64, H // 2, W // 2, dtype=torch.float64, generator=g)
    ref = conv2d_weight(x, (64, 3, 7, 7), dy, stride=2, padding=3)
    s = so.space_to_depth(x.numpy())
    got = so.stem_fold(so.stem_wgrad_s2d(s, dy.permute(0, 2, 3, 1).numpy()))
    np.testing.assert_allclose(got, ref.numpy(), rtol=0, atol=1e-12 * float(ref.abs().max()))
    # the forward identity the eval path relies on: conv1 == the 4x4 stride-1 conv on S with the packed weights
    w = torch.randn(64, 3, 7, 7, dtype=torch.float64, generator=g)
    w4 = torch.zeros(64, 4, 4, 16, dtype=torch.float64)
    for ty, tx, ch, c, kh, kw in so.stem_fold_map():
        w4[:, ty, tx, ch] = w[:, c, kh, kw]
    y = F.conv2d(torch.from_numpy(s).permute(0, 3, 1, 2), w4.permute(0, 3, 1, 2), padding=(2, 2))[..., :H // 2, :W // 2]
    torch.testing.assert_close(y, F.conv2d(x, w, stride=2, padding=3), rtol=0, atol=1e-12)


def _pool_cases():
    rng = np.random.default_rng(5)
    relu = np.maximum(rng.standard_normal((2, 8, 10, 8)).astype(np.float32), 0)       # many exact-zero ties
    coarse = rng.integers(-2, 3, (1, 6, 8, 4)).astype(np.float32)                        # ties of equal values
    ninf = rng.standard_normal((1, 6, 6, 4)).astype(np.float32)
    ninf[:, :3, :3] = -np.inf                                                            # all -inf windows
    nan = rng.standard_normal((1, 6, 8, 8)).astype(np.float32)
    nan[0, 1, 1, 0] = np.nan
    nan[0, 2, 3, 1:3] = np.nan
    nan[0, 3, 3, 2] = np.nan
    return {"relu": relu, "coarse": coarse, "ninf": ninf, "nan": nan}


@pytest.mark.parametrize("name", ["relu", "coarse", "ninf", "nan"])
def test_maxpool_oracle_matches_torch_cpu(name):
    x = _pool_cases()[name]
    b, H, W, C = x.shape
    out, code = so.maxpool_forward(x)
    assert code.dtype == np.uint8 and int(code.max()) <= 8
    xt = torch.from_numpy(x).permute(0, 3, 1, 2).contiguous().requires_grad_()
    ref, ind = F.max_pool2d(xt, 3, 2, 1, return_indices=True)
    refh = ref.detach().permute(0, 2, 3, 1).numpy()
    assert np.array_equal(out.view(np.int32), refh.view(np.int32))             # NaN payloads included
    oy, ox = np.mgrid[0:H // 2, 0:W // 2]
    dy, dx = np.divmod(code.astype(np.int64), 3)
    flat = (2 * oy[None, :, :, None] - 1 + dy) * W + (2 * ox[None, :, :, None] - 1 + dx)
    assert np.array_equal(flat, ind.permute(0, 2, 3, 1).numpy())
    g = np.random.default_rng(1).standard_normal(out.shape).astype(np.float32)
    (gx,) = torch.autograd.grad(ref, xt, torch.from_numpy(g).permute(0, 3, 1, 2))
    din = so.maxpool_backward(g, code, H, W)
    assert np.array_equal(din, gx.permute(0, 2, 3, 1).numpy())


@pytest.mark.parametrize("cin,cout", [(32, 20), (32, 36), (64, 3)])
def test_head_oracle_within_fp32_rounding_of_fp64(cin, cout):
    rng = np.random.default_rng(cin + cout)
    N = 2 * 37 * 61                                     # more than one HEAD_CHUNK partial, a ragged last one
    y = rng.standard_normal((N, cin)).astype(np.float32)
    w = (0.2 * rng.standard_normal((cout, cin))).astype(np.float32)
    bias = rng.standard_normal(cout).astype(np.float32)
    g = rng.standard_normal((N, cout)).astype(np.float32)
    yd = torch.from_numpy(y).double().requires_grad_()
    wd = torch.from_numpy(w).double().requires_grad_()
    bd = torch.from_numpy(bias).double().requires_grad_()
    ref = F.conv2d(yd.T[None, :, :, None], wd[:, :, None, None], bd)[0, :, :, 0].T
    rdy, rdw, rdb = torch.autograd.grad(ref, (yd, wd, bd), torch.from_numpy(g).double())
    out = so.head_forward(y, w, bias)
    R = np.abs(y).astype(np.float64) @ np.abs(w).T.astype(np.float64) + np.abs(bias)
    assert (np.abs(out - ref.detach().numpy()) <= (cin + 1) * U32 * R).all()
    dy = so.head_dy(g, w)
    Rd = np.abs(g).astype(np.float64) @ np.abs(w).astype(np.float64)
    assert (np.abs(dy - rdy.numpy()) <= (cout + 1) * U32 * Rd).all()
    dw, db = so.head_param_sums(g, y)
    for got, exact in ((dw, rdw.numpy()), (db, rdb.numpy())):
        ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
        assert (np.abs(got.astype(np.float64) - exact) <= ulp).all()
