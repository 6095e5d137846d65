"""The graph table of forward_train (tests/train_stages.py) against the PyTorch graph, on the CPU.

The table is replayed call by call with the modules' own torch forward (fp64, train mode) and compared with
`_forward_torch` on a copy: the same outputs and buffers, the same module calls in the same order per module type
(convolutions, BatchNorms), each with the same input, and every parameter read by exactly one call."""
import copy

import pytest
import torch
import torch.nn.functional as F

from pvnet_b200.model_repository import Resnet18_8s
from tests import train_stages as ts

CASES = [("default", 18, 2, ts.DEFAULT_DIMS), ("narrow-seg3", 18, 3, ts.NARROW_DIMS)]
ACT = {"relu": F.relu, "leaky": lambda t: F.leaky_relu(t, 0.1), None: lambda t: t}


def _net(ver, seg, dims):
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=ver, seg_dim=seg, fcdim=dims[0], s8dim=dims[1], s4dim=dims[2], s2dim=dims[3],
                      raw_dim=dims[4]).double().train()
    with torch.no_grad():                 # BatchNorms away from their identity initialisation
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.1)
    return net


def _replay(net, x, rows):
    """The table evaluated with the modules' torch forward: {call name: output}."""
    mods = dict(net.named_modules())
    b, _, h, w = x.shape
    vals = {"image": x, "zeros": x.new_zeros(b, ts.PAD_CHANNELS, h, w)}
    for c in rows:
        vals["cat"] = torch.cat([vals[s] for s in ts.CAT], 1) if all(s in vals for s in ts.CAT) else None
        ins = [vals[s] for s in c.inputs]
        if c.kind in ("stem", "conv", "head", "maxpool"):
            m = mods[c.name]
            y = m(ins[0][:, :m.in_channels] if c.kind == "conv" else ins[0])
        elif c.kind == "bn_act":
            y = ACT[c.act](mods[c.name](ins[0]))
        elif c.kind == "bn_add_relu":
            y = mods[c.name](ins[0])
            y = F.relu(y + (ins[1] if c.bn_skip is None else mods[c.bn_skip](ins[1])))
        else:
            up = F.interpolate(ins[0], scale_factor=2, mode="bilinear", align_corners=True)
            y = torch.cat([up] + ins[1:], 1)
        vals[c.name] = y
    return vals


def _record(net):
    """Forward hooks on every convolution and BatchNorm: [(type, name, input clone)] in call order."""
    log = []
    for name, m in net.named_modules():
        if isinstance(m, (torch.nn.Conv2d, torch.nn.BatchNorm2d)):
            m.register_forward_hook(lambda mod, inp, out, name=name: log.append((type(mod).__name__, name,
                                                                                 inp[0].detach().clone())))
    return log


@pytest.mark.parametrize("ver,seg,dims", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_table_names_every_parameter_once(ver, seg, dims):
    net = _net(ver, seg, dims)
    rows = ts.calls(dims)
    assert len(rows) == 52
    count = {k: sum(c.kind == k for c in rows) for k in ("stem", "bn_act", "bn_add_relu", "conv", "maxpool",
                                                          "upsample_cat", "head")}
    assert count == dict(stem=1, bn_act=14, bn_add_relu=8, conv=24, maxpool=1, upsample_cat=3, head=1)
    names = [p for c in rows for p in c.params()]
    assert len(names) == len(set(names))
    assert sorted(names) == sorted(n for n, _ in net.named_parameters())
    bns = [m for c in rows for m in c.batchnorms()]
    assert sorted(bns) == sorted(n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d))
    # every source is the image, the zero channels, the cat or an earlier call; the cat's operands exist
    seen = {"image", "zeros"}
    for c in rows:
        for s in c.inputs:
            assert s in seen or (s == "cat" and all(o in seen for o in ts.CAT)), (c.name, s)
        seen.add(c.name)
    # convraw.0 reads cat[fm, image, zeros]: its data gradient covers fm's channels only
    raw = [c for c in rows if c.name == "convraw.0"][0]
    assert raw.dgrad_channels == dims[3] and 3 + ts.PAD_CHANNELS == 8


@pytest.mark.parametrize("ver,seg,dims", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_table_order_and_sources_match_forward_torch(ver, seg, dims):
    net = _net(ver, seg, dims)
    twin = copy.deepcopy(net)
    x = torch.randn(2, 3, 32, 48, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    log_t = _record(twin)
    seg_t, ver_t = twin._forward_torch(x)
    log_r = _record(net)
    vals = _replay(net, x, ts.calls(dims))
    out = vals["convraw.3"]
    assert torch.equal(out[:, :seg], seg_t) and torch.equal(out[:, seg:], ver_t)
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        assert torch.equal(p, q), k
    for kind in ("Conv2d", "BatchNorm2d"):
        got = [(n, t) for k, n, t in log_r if k == kind]
        want = [(n, t) for k, n, t in log_t if k == kind]
        assert [n for n, _ in got] == [n for n, _ in want], kind
        for (n, a), (_, b) in zip(got, want):
            assert torch.equal(a, b), n
    # the order of the table's convolutions and BatchNorms is the order they run in
    rows = ts.calls(dims)
    convs = [c.name for c in rows if c.kind in ("stem", "conv", "head")]
    assert convs == [n for k, n, _ in log_t if k == "Conv2d"]
    assert [m for c in rows for m in c.batchnorms()] == [n for k, n, _ in log_t if k == "BatchNorm2d"]
    # the extra zero channels behind the image are zeros, and convraw.0's weight does not reach past them
    up = vals["up2storaw"]
    assert up.shape[1] == dims[3] + 3 + ts.PAD_CHANNELS and not up[:, dims[3] + 3:].any()
