"""GPU: one real Resnet18_8s, Resnet34_8s or Resnet50_8s forward_train step, every native call against an fp64
restatement of its own layer.

The whole-step tests (test_gpu_conv_grad.py, test_gpu_bn_train.py, test_gpu_deep_backbones_train.py) bound the network
by torch's own TF32 error, up to 1.7e-1 on a parameter gradient; a weight gradient 1 % wrong on one layer hides in
that.  Here the step runs with capture wrappers on pvnet_b200.conv (tests/train_stages.py): each of the 52, 84 or 117
calls records its inputs, its output, the
gradient that reached its output and the gradient it gave each input.  Every reference below is computed from that
call's own captured tensors, so errors do not accumulate and a failure names the layer.  trunc(.) drops the low 13
mantissa bits (what a TF32 MMA reads from an fp32 activation or gradient), r(.) rounds to TF32 (the packed weights).

  call          forward                                        backward
  conv2d_train  fp64 conv of trunc(x) and r(W);                dX: conv2d_input of trunc(dY) and r(W) (zero insertion
                |got - ref| <= 1e-5 R, R the same operation    for stride 2 is conv2d_input's), on the first
                on absolute values                             dgrad_channels channels, the rest exactly 0;
                                                               dW: conv2d_weight of trunc(x), trunc(dY) against the
                                                               step's own p.grad; both 1e-5 R
  bn_act,       bit for bit oracle/bn_train_oracle.py: y, and  dx, dz, dgamma, dbeta bit for bit the oracle (the
  bn_add_relu   the running statistics updated from the        parameter gradients are p.grad)
                snapshot taken before the call; num_batches_tracked + 1
  upsample2x_   torch.equal to F.interpolate(align_corners=    dlow bit for bit oracle/upsample_oracle.py; each `rest`
  cat           True) + cat                                    gradient equals its channel slice of dY
  stem          fp64 conv of r(x) and r(W), 1e-5 R             dW: conv2d_weight of r(x), trunc(dY) against
                                                               conv1.weight.grad, 1e-5 R
  max-pool      bits equal torch's CUDA max_pool2d             dX bits equal torch's
  head          bit for bit oracle/stem_pool_head_oracle.py    dy, dW, db bit for bit
  losses        --                                             the gradient at the head output: the vertex part bit for
                                                               bit oracle/loss_grad_oracle.py; the seg part bit for bit
                                                               torch's CUDA autograd of the reference's cross-entropy,
                                                               and within 2^-20 gs / (H W) of the oracle (its exp and
                                                               log are numpy's)

The head's forward and dy are per pixel; above 65,536 pixels they are compared on every image's first and last 4096
pixels and 16,384 random ones (the parameter gradients, which sum over all pixels, are compared whole).

Composition: (a) each call's inputs are torch.equal to the outputs the table says feed them; (b) for every tensor with
several consumers the gradient at it is the sum of its consumers' gradients, within 2^-24 (k - 1) sum|terms| for k
consumers, and equal to it with one consumer; (c) every parameter belongs to exactly one call, whose check reads its
.grad; (d) the instrumentation changes nothing: a copy stepped without it has bit-identical outputs, gradients and
buffers.
"""
import copy
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.nn.grad import conv2d_input, conv2d_weight

from oracle import bn_train_oracle as bo
from oracle import loss_grad_oracle as lgo
from oracle import stem_pool_head_oracle as so
from oracle import upsample_oracle as uo
from pvnet_b200 import conv as pc
from pvnet_b200 import net_utils as nu
from pvnet_b200.model_repository import Resnet18_8s, Resnet34_8s, Resnet50_8s
from tests import train_stages as ts
from tests.helpers import seeded_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ACTS = {"relu": pc.ACT_RELU, "leaky": pc.ACT_LEAKY, None: pc.ACT_NONE}
SAMPLE_ABOVE = 65536

# The paths a case must reach, asserted in _run_case: convolutions whose weight gradient is split over more than one
# CTA per tile (layer2.0.conv1: k_conv_wgrad<2,64> on the zero-inserted grid; conv2s.0: <1,128>; the deep networks'
# 1x1 convs at 1/4 resolution and fc.0 over 512 / 2048 channels), and convolutions whose input has a partly filled
# 64-channel Cin tile (channel count of the captured input).
R50 = "resnet50_8s."              # Resnet34_8s keeps its trunk under the same name
SPLIT = {"k9-2x480x640": ("resnet18_8s.layer1.0.conv1", "resnet18_8s.layer2.0.conv1", "conv4s.0", "conv2s.0",
                          "convraw.0"),
         "r34-k9-2x480x640": (R50 + "layer2.0.downsample.0", R50 + "fc.0", "convraw.0"),
         "r50-k9-2x480x640": (R50 + "layer1.0.conv1", R50 + "layer1.1.conv3", R50 + "layer1.0.downsample.0",
                              R50 + "layer2.0.downsample.0", R50 + "fc.0", "convraw.0")}
PARTIAL_CIN = {"k9-2x480x640": {"convraw.0": 40}, "narrow-seg3-2x72x104": {"convraw.0": 72, "conv2s.0": 96},
               "r34-k9-2x480x640": {"convraw.0": 72}, "r50-k9-2x480x640": {"convraw.0": 72}}

CASES = [
    # id, network, trunk, ver_dim, seg_dim, decoder widths, (b, h, w)
    # training resolution; wgrad splits; 150 partials
    ("k9-2x480x640", Resnet18_8s, ts.RESNET18, 18, 2, ts.DEFAULT_DIMS, (2, 480, 640)),
    ("k9-3x72x104", Resnet18_8s, ts.RESNET18, 18, 2, ts.DEFAULT_DIMS, (3, 72, 104)),   # odd 9 x 13 grid at 1/8
    # 1 x 1 at 1/8: every dilated off-centre tap pads
    ("k9-4x8x8", Resnet18_8s, ts.RESNET18, 18, 2, ts.DEFAULT_DIMS, (4, 8, 8)),
    ("k17-2x64x96", Resnet18_8s, ts.RESNET18, 34, 2, ts.DEFAULT_DIMS, (2, 64, 96)),    # head Cout 36
    # convraw.0 reads 72 channels; conv2s.0 Cin 96
    ("narrow-seg3-2x72x104", Resnet18_8s, ts.RESNET18, 18, 3, ts.NARROW_DIMS, (2, 72, 104)),
    # the deep networks: 1x1 Bottleneck convs up to Cin 2048, fc.0 at K = 18 432, BatchNorms of 2048 channels,
    # head_train at Cin 64, convraw.0 reading 72 channels
    ("r34-k9-2x64x96", Resnet34_8s, ts.RESNET34, 18, 2, ts.DEEP_DIMS, (2, 64, 96)),
    ("r34-k9-3x72x104", Resnet34_8s, ts.RESNET34, 18, 2, ts.DEEP_DIMS, (3, 72, 104)),
    ("r34-k9-4x8x8", Resnet34_8s, ts.RESNET34, 18, 2, ts.DEEP_DIMS, (4, 8, 8)),
    ("r34-k9-2x480x640", Resnet34_8s, ts.RESNET34, 18, 2, ts.DEEP_DIMS, (2, 480, 640)),
    ("r50-k9-2x64x96", Resnet50_8s, ts.RESNET50, 18, 2, ts.DEEP_DIMS, (2, 64, 96)),
    ("r50-k9-3x72x104", Resnet50_8s, ts.RESNET50, 18, 2, ts.DEEP_DIMS, (3, 72, 104)),
    ("r50-k9-4x8x8", Resnet50_8s, ts.RESNET50, 18, 2, ts.DEEP_DIMS, (4, 8, 8)),       # dilation 4 under Bottlenecks
    ("r50-k9-2x480x640", Resnet50_8s, ts.RESNET50, 18, 2, ts.DEEP_DIMS, (2, 480, 640)),
]


def _trunc(t):
    return (t.detach().float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def _flat(t):
    """[b,C,H,W] -> numpy [N, C] in NHWC order."""
    return t.detach().permute(0, 2, 3, 1).reshape(-1, t.shape[1]).cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


class Ledger:
    """Failures named by layer, and the largest error/bound ratio per check."""

    def __init__(self):
        self.fail, self.ratio = [], {}

    def bound(self, what, kind, got, ref, absref):
        """|got - ref| <= 1e-5 R."""
        err = (got.detach().double() - ref).abs()
        bnd = 1e-5 * absref
        r = float(torch.where(err == 0, torch.zeros_like(err), err / bnd).max())
        self.ratio[kind] = max(self.ratio.get(kind, 0.0), r)
        if not r <= 1.0:
            self.fail.append(f"{what}: max |got-ref| {float(err.max()):.3e}, {r:.3g} x the bound 1e-5 R")

    def sums(self, what, total, terms):
        if len(terms) == 1:
            if not torch.equal(total, terms[0]):
                self.fail.append(f"{what}: the gradient differs from its one consumer's")
            return
        s = sum(t.double() for t in terms)
        bnd = 2.0 ** -24 * (len(terms) - 1) * sum(t.double().abs() for t in terms)
        err = (total.double() - s).abs()
        r = float(torch.where(err == 0, torch.zeros_like(err), err / bnd).max())
        self.ratio["gradient sums"] = max(self.ratio.get("gradient sums", 0.0), r)
        if not r <= 1.0:
            self.fail.append(f"{what}: sum of {len(terms)} consumers off by {r:.3g} x 2^-24 (k-1) sum|terms|")

    def exact(self, what, ok):
        if not ok:
            self.fail.append(what)


def _model(cls, ver, seg, dims):
    net = cls(ver_dim=ver, seg_dim=seg, fcdim=dims[0], s8dim=dims[1], s4dim=dims[2], s2dim=dims[3], raw_dim=dims[4])
    net.load_state_dict(seeded_state_dict(net))
    return net.to(DEV).train()


def _targets(b, h, w, K, seed):
    """A disc mask per image, keypoints inside the image, their vertex field and 0/1 weights."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    masks = [((yy - rng.uniform(0.3, 0.7) * h) ** 2 + (xx - rng.uniform(0.3, 0.7) * w) ** 2 < (0.25 * h) ** 2)
             for _ in range(b)]
    mask = torch.from_numpy(np.stack(masks).astype(np.int64)).to(DEV)
    hc = np.concatenate([rng.uniform([0, 0], [w, h], (b, K, 2)), np.ones((b, K, 1))], 2)
    return mask, nu.vertex_targets(mask, torch.from_numpy(hc).to(DEV)), mask[:, None].float()


def _keep(store, key, g):
    store[key] = g.clone()


def _step(net, x, mask, field, wgt, keep=None):
    seg, ver = net.forward_train(x)
    ls, lv, _, _ = nu.seg_vertex_training_losses(seg, ver, mask, field, wgt)
    if keep is not None:
        ls.register_hook(functools.partial(_keep, keep, "gs"))
        lv.register_hook(functools.partial(_keep, keep, "gv"))
    (ls.mean() + lv.mean()).backward()
    return seg.detach(), ver.detach()


# ----------------------------------------------------------------------------- per call type
def _check_conv(L, rec, c, mods):
    m = mods[c.name]
    w = m.weight.detach()
    x = rec.inputs[0]
    cin = w.shape[1]
    st, pad, dil = m.stride[0], m.padding[0], m.dilation[0]
    L.exact(f"{c.name}: called with stride {rec.args['stride']}, dilation {rec.args['dilation']}, dgrad_channels "
            f"{rec.args['dgrad_channels']}", (rec.args["stride"], rec.args["dilation"], rec.args["dgrad_channels"])
            == (st, dil, c.dgrad_channels))
    L.exact(f"{c.name}: input channels beyond the weight's are not zero", not x[:, cin:].any())
    xq, wq = _trunc(x[:, :cin]).double(), pc.round_tf32(w).double()
    ref = F.conv2d(xq, wq, None, st, pad, dil)
    L.bound(f"{c.name} forward", "conv2d_train forward", rec.output, ref, F.conv2d(xq.abs(), wq.abs(), None, st, pad,
                                                                                     dil))
    del ref
    gq = _trunc(rec.out_grad).double()
    dx = rec.in_grads[0]
    n = x.shape[1] if c.dgrad_channels is None else c.dgrad_channels
    shape = (x.shape[0], n, x.shape[2], x.shape[3])
    ref = conv2d_input(shape, wq[:, :n], gq, st, pad, dil)
    L.bound(f"{c.name} dX", "conv2d_train dX", dx[:, :n], ref, conv2d_input(shape, wq[:, :n].abs(), gq.abs(), st, pad,
                                                                            dil))
    L.exact(f"{c.name} dX: channels from dgrad_channels on are not 0", not dx[:, n:].any())
    del ref
    ref = conv2d_weight(xq, w.shape, gq, st, pad, dil)
    L.bound(f"{c.name} dW", "conv2d_train dW", m.weight.grad, ref, conv2d_weight(xq.abs(), w.shape, gq.abs(), st, pad,
                                                                                 dil))


def _check_bn(L, rec, c, mods):
    bn = mods[c.name]
    bz = None if c.bn_skip is None else mods[c.bn_skip]
    act = ACTS[c.act] if c.kind == "bn_act" else pc.ACT_RELU
    if c.kind == "bn_act":
        L.exact(f"{c.name}: called with act {rec.args['act']}", rec.args["act"] == act)
    else:
        L.exact(f"{c.name}: called with bn_skip {rec.args['bn_skip']}", rec.args["bn_skip"] == c.bn_skip)
    xs = _flat(rec.inputs[0])
    zs = _flat(rec.inputs[1]) if c.kind == "bn_add_relu" else None
    N = xs.shape[0]

    def stats(m, label, v, snap):
        mean, var, invstd = bo.batch_stats(v, m.eps)
        gamma, beta = m.weight.detach().cpu().numpy(), m.bias.detach().cpu().numpy()
        scale, shift = bo.scale_shift(mean, invstd, gamma, beta)
        rm0, rv0, nbt0 = (t.cpu() for t in snap)
        f = m.momentum
        L.exact(f"{label}: running_mean", torch.equal(
            m.running_mean.cpu(), rm0 * (1 - f) + torch.from_numpy(mean.astype(np.float32)) * f))
        L.exact(f"{label}: running_var", torch.equal(
            m.running_var.cpu(), rv0 * (1 - f) + torch.from_numpy(bo.unbiased32(var, N)) * f))
        L.exact(f"{label}: num_batches_tracked", int(m.num_batches_tracked) == int(nbt0) + 1)
        return scale, shift, mean, invstd, gamma

    scale, shift, mean, invstd, gamma = stats(bn, c.name, xs, rec.snapshots[0])
    if bz is None:
        pre = bo.pre_activation(xs, scale, shift, zs)
    else:
        sz, tz, mz, invz, gz = stats(bz, c.bn_skip, zs, rec.snapshots[1])
        pre = bo.pre_activation(xs, scale, shift, zs, sz, tz)
    L.exact(f"{c.name} forward: y differs from the oracle",
            np.array_equal(_bits(_flat(rec.output)), _bits(bo.act_fwd(pre, act))))
    g = bo.masked_grad(_flat(rec.out_grad), pre, act)
    Sg, Sgx = bo.backward_sums(g, xs, mean)
    coef, (dgam, dbet) = bo.backward_coef(Sg, Sgx, N, mean, invstd, gamma)
    L.exact(f"{c.name} dx differs from the oracle",
            np.array_equal(_bits(_flat(rec.in_grads[0])), _bits(bo.backward_apply(g, xs, coef))))
    L.exact(f"{c.name} dgamma/dbeta differ from the oracle", np.array_equal(_bits(bn.weight.grad.cpu().numpy()),
                                                                            _bits(dgam))
            and np.array_equal(_bits(bn.bias.grad.cpu().numpy()), _bits(dbet)))
    if c.kind == "bn_add_relu" and bz is None:
        L.exact(f"{c.name} skip gradient differs from dy * relu'", np.array_equal(_bits(_flat(rec.in_grads[1])), _bits(g)))
    elif bz is not None:
        Sgz, Sgzz = bo.backward_sums(g, zs, mz)
        coefz, (dgz, dbz) = bo.backward_coef(Sgz, Sgzz, N, mz, invz, gz)
        L.exact(f"{c.name} dz ({c.bn_skip}) differs from the oracle",
                np.array_equal(_bits(_flat(rec.in_grads[1])), _bits(bo.backward_apply(g, zs, coefz))))
        L.exact(f"{c.bn_skip} dgamma/dbeta differ from the oracle",
                np.array_equal(_bits(bz.weight.grad.cpu().numpy()), _bits(dgz))
                and np.array_equal(_bits(bz.bias.grad.cpu().numpy()), _bits(dbz)))


def _check_upsample(L, rec, c):
    low, rest = rec.inputs[0], rec.inputs[1:]
    ref = torch.cat([F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=True), *rest], 1)
    L.exact(f"{c.name} forward differs from F.interpolate + cat", torch.equal(rec.output, ref))
    gy = rec.out_grad
    C = low.shape[1]
    want = uo.upsample2x_backward(gy[:, :C].permute(0, 2, 3, 1).cpu().numpy())
    got = rec.in_grads[0].permute(0, 2, 3, 1).cpu().numpy()
    L.exact(f"{c.name} dlow differs from the oracle", np.array_equal(_bits(got), _bits(want)))
    co = C
    for k, r in enumerate(rest, 1):
        if r.requires_grad:
            L.exact(f"{c.name}: gradient of {c.inputs[k]} is not its channel slice",
                    torch.equal(rec.in_grads[k], gy[:, co:co + r.shape[1]]))
        co += r.shape[1]


def _check_stem(L, rec, c, mods):
    w = mods[c.name].weight
    xq, wq = pc.round_tf32(rec.inputs[0]).double(), pc.round_tf32(w.detach()).double()
    ref = F.conv2d(xq, wq, stride=2, padding=3)
    L.bound("stem forward", "stem forward", rec.output, ref, F.conv2d(xq.abs(), wq.abs(), stride=2, padding=3))
    gq = _trunc(rec.out_grad).double()
    ref = conv2d_weight(xq, w.shape, gq, stride=2, padding=3)
    L.bound("stem dW", "stem dW", w.grad, ref, conv2d_weight(xq.abs(), w.shape, gq.abs(), stride=2, padding=3))


def _check_maxpool(L, rec):
    xi = rec.inputs[0].detach().clone().requires_grad_()
    ref = F.max_pool2d(xi, 3, 2, 1)
    L.exact("max-pool forward differs from torch's", np.array_equal(_bits(_flat(rec.output)), _bits(_flat(ref))))
    (rx,) = torch.autograd.grad(ref, xi, rec.out_grad)
    L.exact("max-pool dX differs from torch's", np.array_equal(_bits(_flat(rec.in_grads[0])), _bits(_flat(rx))))


def _sample_rows(N, b, seed=0):
    """Every row below SAMPLE_ABOVE pixels; above, every image's first and last 4096 and 16384 random ones."""
    if N <= SAMPLE_ABOVE:
        return np.arange(N)
    per = N // b
    rows = [np.arange(i * per, i * per + 4096) for i in range(b)] + [np.arange((i + 1) * per - 4096, (i + 1) * per)
                                                                     for i in range(b)]
    rows.append(np.random.default_rng(seed).choice(N, 16384, replace=False))
    return np.unique(np.concatenate(rows))


def _check_head_call(L, what, y, w, bias, out, gout, gy, gw, gb):
    """The head's forward, dy, dW and db bit for bit against the oracle (forward and dy on _sample_rows)."""
    cout, cin = w.shape[:2]
    yn, gn = _flat(y), _flat(gout)
    wn = w.detach().reshape(cout, cin).cpu().numpy()
    rows = _sample_rows(yn.shape[0], y.shape[0])
    L.exact(f"{what} forward differs from the oracle", np.array_equal(
        _bits(_flat(out)[rows]), _bits(so.head_forward(yn[rows], wn, bias.detach().cpu().numpy()))))
    L.exact(f"{what} dy differs from the oracle", np.array_equal(_bits(_flat(gy)[rows]), _bits(so.head_dy(gn[rows], wn))))
    dw, db = so.head_param_sums(gn, yn)
    L.exact(f"{what} dW differs from the oracle", np.array_equal(_bits(gw.reshape(cout, cin).cpu().numpy()), _bits(dw)))
    L.exact(f"{what} db differs from the oracle", np.array_equal(_bits(gb.cpu().numpy()), _bits(db)))


def _check_losses(L, gout, seg_dim, seg, ver, mask, field, wgt, keep):
    gs, gv = keep["gs"], keep["gv"]
    want = lgo.smooth_l1_grad(ver.cpu().numpy(), field.cpu().numpy(), wgt.cpu().numpy(), gv.cpu().numpy())
    L.exact("vertex gradient at the head output differs from the oracle",
            np.array_equal(_bits(gout[:, seg_dim:].cpu().numpy()), _bits(want)))
    s = seg.contiguous().requires_grad_()
    loss = torch.nn.CrossEntropyLoss(reduction="none")(s, mask)
    (ref,) = torch.autograd.grad(torch.mean(loss.view(loss.shape[0], -1), 1), s, gs)
    got = gout[:, :seg_dim]
    L.exact("seg gradient at the head output differs from torch's autograd", torch.equal(got, ref))
    oracle = lgo.cross_entropy_grad(seg.cpu().numpy(), mask.cpu().numpy(), gs.cpu().numpy())
    n = seg.shape[2] * seg.shape[3]
    bound = (2.0 ** -20 * gs.cpu().numpy() / n)[:, None, None, None]
    L.exact("seg gradient at the head output is not within 2^-20 gs / (H W) of the oracle",
            (np.abs(got.cpu().numpy().astype(np.float64) - oracle) <= bound).all())


def _wgrad_splits(cin, cout, b, H, W, k):
    """How many CTAs share each dW tile of pvnet_conv2d_nhwc_wgrad at this shape (its workspace holds one partial
    tile per split)."""
    import ctypes

    from pvnet_b200 import _native
    n = ctypes.c_size_t()
    with torch.cuda.device(DEV):
        _native.check(_native.lib().pvnet_conv2d_nhwc_wgrad_workspace_bytes(cin, cout, b, H, W, k, ctypes.byref(n)),
                      "pvnet_conv2d_nhwc_wgrad_workspace_bytes")
    return n.value // (cout * cin * k * k * 4)


# ----------------------------------------------------------------------------- the step
def _run_case(case, monkeypatch):
    name, cls, trunk, ver_dim, seg_dim, dims, (b, h, w) = case
    trunk = trunk._replace(dims=dims)
    net = _model(cls, ver_dim, seg_dim, dims)
    twin = copy.deepcopy(net)
    x = torch.randn(b, 3, h, w, device=DEV, generator=torch.Generator(device=DEV).manual_seed(b * h + w))
    mask, field, wgt = _targets(b, h, w, ver_dim // 2, h + w)
    out_twin = _step(twin, x, mask, field, wgt)
    cap = ts.Capture(net, pc)
    cap.install(monkeypatch)
    keep = {}
    try:
        out = _step(net, x, mask, field, wgt, keep)
    finally:
        monkeypatch.undo()
    L = Ledger()
    # (d) the instrumentation changes nothing
    L.exact("instrumented outputs differ", all(torch.equal(p, q) for p, q in zip(out, out_twin)))
    for (k, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        L.exact(f"instrumented {k}.grad differs", torch.equal(p.grad, q.grad))
    for (k, p), (_, q) in zip(net.named_buffers(), twin.named_buffers()):
        L.exact(f"instrumented buffer {k} differs", torch.equal(p, q))
    del twin
    rows, recs = ts.calls(trunk), cap.records
    assert [(r.kind, r.name or c.name) for r, c in zip(recs, rows)] == [(c.kind, c.name) for c in rows]
    assert len(recs) == len(rows)
    # (c) every parameter in exactly one call
    names = [p for c in rows for p in c.params()]
    assert sorted(names) == sorted(k for k, _ in net.named_parameters()) and len(set(names)) == len(names)
    # (a) the wiring
    vals = {c.name: r.output for c, r in zip(rows, recs)}
    vals["image"] = x
    vals["zeros"] = torch.zeros(b, ts.PAD_CHANNELS, h, w, device=DEV)
    cat = ts.cat_operands(trunk)
    vals["cat"] = torch.cat([vals[s] for s in cat], 1)
    for c, r in zip(rows, recs):
        for k, s in enumerate(c.inputs):
            L.exact(f"{c.name}: input {k} is not {s}", torch.equal(r.inputs[k], vals[s]))
    # (b) the gradients of tensors with several consumers add up
    index = {c.name: i for i, c in enumerate(rows)}
    cat_call = [i for i, c in enumerate(rows) if "cat" in c.inputs][0]
    fc = dims[0]
    for s, cons in ts.consumers(rows).items():
        if s not in index:
            continue
        terms = [recs[i].in_grads[k] for i, k in cons]
        if s in cat:
            g = recs[cat_call].in_grads[rows[cat_call].inputs.index("cat")]
            terms.append(g[:, :fc] if s == cat[0] else g[:, fc:])
        L.sums(f"gradient at {s}", recs[index[s]].out_grad, terms)
    for s in cat:             # xfc feeds only the cat
        if s not in ts.consumers(rows):
            g = recs[cat_call].in_grads[0]
            L.sums(f"gradient at {s}", recs[index[s]].out_grad, [g[:, :fc]])
    # the kernel paths this case is meant to reach
    reached = set()
    for c, r in zip(rows, recs):
        if c.kind != "conv":
            continue
        x = r.inputs[0]
        if c.name in SPLIT.get(name, ()):
            splits = _wgrad_splits(x.shape[1], net.get_submodule(c.name).weight.shape[0], *x.shape[:1], *x.shape[2:],
                                   net.get_submodule(c.name).kernel_size[0])
            assert splits > 1, (c.name, splits)
            reached.add(c.name)
        if c.name in PARTIAL_CIN.get(name, {}):
            assert x.shape[1] == PARTIAL_CIN[name][c.name] and x.shape[1] % 64 != 0, (c.name, x.shape)
            reached.add(c.name)
    assert reached == set(SPLIT.get(name, ())) | set(PARTIAL_CIN.get(name, {})), reached
    # per call
    mods = dict(net.named_modules())
    for c, r in zip(rows, recs):
        if c.kind == "conv":
            _check_conv(L, r, c, mods)
        elif c.kind in ("bn_act", "bn_add_relu"):
            _check_bn(L, r, c, mods)
        elif c.kind == "upsample_cat":
            _check_upsample(L, r, c)
        elif c.kind == "stem":
            _check_stem(L, r, c, mods)
        elif c.kind == "maxpool":
            _check_maxpool(L, r)
            print(f"{name}: max-pool input has {int((r.inputs[0] == 0).sum())} exact zeros")
        else:
            m = mods[c.name]
            _check_head_call(L, c.name, r.inputs[0], m.weight, m.bias, r.output, r.out_grad, r.in_grads[0],
                             m.weight.grad, m.bias.grad)
            _check_losses(L, r.out_grad, seg_dim, out[0], out[1], mask, field, wgt, keep)
    for k, v in sorted(L.ratio.items()):
        print(f"{name}: largest error/bound, {k}: {v:.3g}")
    assert not L.fail, "\n".join(L.fail)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_step_native_calls_layer_by_layer(case, monkeypatch):
    _run_case(case, monkeypatch)


# ----------------------------------------------------------------------------- direct head calls
@pytest.mark.parametrize("b,H,W", [(4, 480, 640), (40, 5, 7)], ids=["4x480x640-300-partials", "40x5x7-tiles-span-images"])
def test_head_train_against_oracle(b, H, W):
    # 4 x 480 x 640: 300 partials of HEAD_CHUNK pixels, so the reduce's lanes each add more than one;
    # 40 x 5 x 7: 35 pixels per image, so a 64-pixel tile spans up to three images
    g = torch.Generator(device=DEV).manual_seed(b)
    y = torch.randn(b, 32, H, W, device=DEV, generator=g).contiguous(memory_format=torch.channels_last)
    y.requires_grad_()
    w = (0.2 * torch.randn(20, 32, 1, 1, device=DEV, generator=g)).requires_grad_()
    bias = torch.randn(20, device=DEV, generator=g).requires_grad_()
    out = pc.head_train(y, w, bias)
    gout = torch.randn(out.shape, device=DEV, generator=g)
    gy, gw, gb = torch.autograd.grad(out, (y, w, bias), gout)
    L = Ledger()
    _check_head_call(L, "head_train", y, w, bias, out, gout, gy, gw, gb)
    assert not L.fail, "\n".join(L.fail)
    P = -(-b * H * W // so.HEAD_CHUNK)
    assert (P > 256) == (b == 4), P


# ----------------------------------------------------------------------------- batch 1 at 8 x 8
def test_single_value_per_channel_raises_like_torch():
    # layer2.0.bn1 sees one value per channel: nn.BatchNorm2d raises ValueError after counting the batch
    net = _model(Resnet18_8s, 18, 2, ts.DEFAULT_DIMS)
    start = {k: v.clone() for k, v in net.named_buffers()}
    ref = copy.deepcopy(net)
    x = torch.randn(1, 3, 8, 8, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    with pytest.raises(ValueError, match="more than 1 value"):
        ref._forward_torch(x)
    with pytest.raises(ValueError, match="more than one value"):
        net.forward_train(x)
    got, want = dict(net.named_buffers()), dict(ref.named_buffers())
    for k in got:
        if k.endswith("num_batches_tracked"):
            assert torch.equal(got[k], want[k]), k
        else:           # the same modules updated their statistics, to the same values up to TF32
            assert torch.equal(got[k], start[k]) == torch.equal(want[k], start[k]), k
            rel = float((got[k].double() - want[k].double()).norm() / want[k].double().norm())
            assert rel <= 1e-2, (k, rel)
    assert int(got[ts.RESNET18.prefix + "layer2.0.bn1.num_batches_tracked"]) == 1
    assert int(got[ts.RESNET18.prefix + "layer2.0.bn2.num_batches_tracked"]) == 0
