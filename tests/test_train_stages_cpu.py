"""The graph table of forward_train (tests/train_stages.py) against the PyTorch graph, on the CPU.

The table is replayed call by call with the modules' own torch forward (fp64, train mode) and compared with
`_forward_torch` on a copy: the same outputs and buffers, the same module calls in the same order per module type
(convolutions, BatchNorms), each with the same input, and every parameter read by exactly one call."""
import copy

import pytest
import torch
import torch.nn.functional as F

from pvnet_b200.model_repository import Resnet18_8s, Resnet34_8s, Resnet50_8s
from tests import train_stages as ts

CASES = [  # id, network, trunk, ver_dim, seg_dim, decoder widths, calls
    ("default", Resnet18_8s, ts.RESNET18, 18, 2, ts.DEFAULT_DIMS, 52),
    ("narrow-seg3", Resnet18_8s, ts.RESNET18, 18, 3, ts.NARROW_DIMS, 52),
    ("resnet34", Resnet34_8s, ts.RESNET34, 18, 2, ts.DEEP_DIMS, 84),
    ("resnet50", Resnet50_8s, ts.RESNET50, 18, 2, ts.DEEP_DIMS, 117),
]
ACT = {"relu": F.relu, "leaky": lambda t: F.leaky_relu(t, 0.1), None: lambda t: t}


def _net(cls, ver, seg, dims):
    torch.manual_seed(0)
    net = cls(ver_dim=ver, seg_dim=seg, fcdim=dims[0], s8dim=dims[1], s4dim=dims[2], s2dim=dims[3],
              raw_dim=dims[4]).double().train()
    with torch.no_grad():                 # BatchNorms away from their identity initialisation
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.1)
    return net


def _replay(net, x, rows, cat):
    """The table evaluated with the modules' torch forward: {call name: output}."""
    mods = dict(net.named_modules())
    b, _, h, w = x.shape
    vals = {"image": x, "zeros": x.new_zeros(b, ts.PAD_CHANNELS, h, w)}
    for c in rows:
        vals["cat"] = torch.cat([vals[s] for s in cat], 1) if all(s in vals for s in cat) else None
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


@pytest.mark.parametrize("cls,trunk,ver,seg,dims,n", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_table_names_every_parameter_once(cls, trunk, ver, seg, dims, n):
    net = _net(cls, ver, seg, dims)
    rows = ts.calls(trunk._replace(dims=dims))
    assert len(rows) == n
    count = {k: sum(c.kind == k for c in rows) for k in ("stem", "bn_act", "bn_add_relu", "conv", "maxpool",
                                                          "upsample_cat", "head")}
    # per block: a conv and a BatchNorm + ReLU per conv but the last, the last conv, the residual BatchNorm; a
    # downsample in each stage's first block but layer1 of a BasicBlock trunk; fc and four decoder convs
    blocks, per = sum(trunk.blocks), 3 if trunk.bottleneck else 2
    ds = 4 if trunk.bottleneck else 3
    assert count == dict(stem=1, bn_act=1 + blocks * (per - 1) + 5, bn_add_relu=blocks, conv=blocks * per + ds + 5,
                         maxpool=1, upsample_cat=3, head=1)
    if trunk == ts.RESNET18:
        assert count == dict(stem=1, bn_act=14, bn_add_relu=8, conv=24, maxpool=1, upsample_cat=3, head=1)
    names = [p for c in rows for p in c.params()]
    assert len(names) == len(set(names))
    assert sorted(names) == sorted(n for n, _ in net.named_parameters())
    bns = [m for c in rows for m in c.batchnorms()]
    assert sorted(bns) == sorted(n for n, m in net.named_modules() if isinstance(m, torch.nn.BatchNorm2d))
    # every source is the image, the zero channels, the cat or an earlier call; the cat's operands exist
    seen = {"image", "zeros"}
    cat = ts.cat_operands(trunk)
    for c in rows:
        for s in c.inputs:
            assert s in seen or (s == "cat" and all(o in seen for o in cat)), (c.name, s)
        seen.add(c.name)
    # convraw.0 reads cat[fm, image, zeros]: its data gradient covers fm's channels only
    raw = [c for c in rows if c.name == "convraw.0"][0]
    assert raw.dgrad_channels == dims[3] and 3 + ts.PAD_CHANNELS == 8


@pytest.mark.parametrize("cls,trunk,ver,seg,dims,n", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_table_order_and_sources_match_forward_torch(cls, trunk, ver, seg, dims, n):
    net = _net(cls, ver, seg, dims)
    trunk = trunk._replace(dims=dims)
    twin = copy.deepcopy(net)
    x = torch.randn(2, 3, 32, 48, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    log_t = _record(twin)
    seg_t, ver_t = twin._forward_torch(x)
    log_r = _record(net)
    vals = _replay(net, x, ts.calls(trunk), ts.cat_operands(trunk))
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
    rows = ts.calls(trunk)
    convs = [c.name for c in rows if c.kind in ("stem", "conv", "head")]
    assert convs == [n for k, n, _ in log_t if k == "Conv2d"]
    assert [m for c in rows for m in c.batchnorms()] == [n for k, n, _ in log_t if k == "BatchNorm2d"]
    # the extra zero channels behind the image are zeros, and convraw.0's weight does not reach past them
    up = vals["up2storaw"]
    assert up.shape[1] == dims[3] + 3 + ts.PAD_CHANNELS and not up[:, dims[3] + 3:].any()
