"""The reformulations behind the native convolution backward, exact in fp64 on the CPU for every layer of
Resnet18_8s.forward_train: the flipped, transposed pack as a forward conv is conv2d_input, and zero insertion turns
the stride-2 layers' data and weight gradients into stride-1 problems."""
import pytest
import torch
from torch.nn.grad import conv2d_input, conv2d_weight

from pvnet_b200 import conv as pc
from tests import conv_grad_cases as cg

SMALL = (6, 10)      # output size of the stride-1 rows; stride-2 rows read 12 x 20


def _operands(name, cin, cout, k, stride, seed):
    g = torch.Generator().manual_seed(seed)
    ho, wo = SMALL
    cbuf = cg.buffer_channels(name, cin)
    w = torch.randn(cout, cin, k, k, generator=g).float()            # fp32 values: the pack holds them exactly
    x = torch.randn(2, cbuf, ho * stride, wo * stride, generator=g, dtype=torch.float64)
    dy = torch.randn(2, cout, ho, wo, generator=g, dtype=torch.float64)
    return w, x, dy


@pytest.mark.parametrize("row", cg.ROWS, ids=[r[0] for r in cg.ROWS])
def test_dgrad_pack_is_conv2d_input(row):
    name, cin, cout, k, stride, dil, _ = row
    w, x, dy = _operands(name, cin, cout, k, stride, 1)
    n = cg.dgrad_channels(name, cin)
    packed = pc.pack_dgrad_weight(w, n, tf32=False)
    assert packed.shape == (n, k * k, pc.cin_padded(cout))
    assert torch.all(packed[:, :, cout:] == 0)
    wbuf = torch.zeros(cout, x.shape[1], k, k, dtype=torch.float64)
    wbuf[:, :cin] = w.double()
    ref = conv2d_input(x.shape, wbuf, dy, stride=stride, padding=cg.pad_of(k, dil), dilation=dil)[:, :n]
    got = cg.dgrad_stride1_form(dy, packed.double(), n, cout, k, stride, dil)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("row", cg.ROWS, ids=[r[0] for r in cg.ROWS])
def test_wgrad_sum_is_conv2d_weight(row):
    name, cin, cout, k, stride, dil, _ = row
    w, x, dy = _operands(name, cin, cout, k, stride, 2)
    ref = conv2d_weight(x, (cout, x.shape[1], k, k), dy, stride=stride, padding=cg.pad_of(k, dil), dilation=dil)
    got = cg.wgrad_stride1_form(x, dy, k, stride, dil)
    torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


def test_pack_dgrad_flips_and_rounds():
    w = torch.randn(32, 8, 3, 3)
    p = pc.pack_dgrad_weight(w)
    assert torch.equal(p[:, :, :32], pc.round_tf32(w.flip(2, 3).permute(1, 2, 3, 0).reshape(8, 9, 32)))
    assert torch.equal(pc.pack_dgrad_weight(w, 4), p[:4])


def test_stride2_rows_are_the_two_layer2_convs():
    assert sorted(r[0] for r in cg.ROWS if r[4] == 2) == ["layer2.0.conv1", "layer2.0.downsample.0"]
    assert len(cg.ROWS) == 24


def test_rows_are_slots_1_to_24():
    from pvnet_b200.model_repository import _SLOTS
    assert [r[0] for r in cg.ROWS] == [s[0].replace("resnet18_8s.", "") for s in _SLOTS[1:25]]
