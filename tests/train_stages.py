"""Resnet*_8s.forward_train as the tests see it: the graph table of its native calls (52 for Resnet18_8s, 84 for
Resnet34_8s, 117 for Resnet50_8s), and wrappers that capture each call's inputs, output and gradients during a real
training step.

The table is written from `_Resnet8s._forward_torch` and pvnet_b200/resnet.py (BasicBlock.forward, Bottleneck.forward,
DilatedResNet.forward), not from `forward_train`: the CPU test (test_train_stages_cpu.py) replays it against
forward hooks on a CPU model, and the GPU test (test_gpu_train_stages.py) holds every captured call to it and to an
fp64 restatement of its own layer.
"""
from __future__ import annotations

import functools
from typing import NamedTuple, Optional, Tuple

import torch

from tests.backbone_stages import DEEP_DIMS, DEFAULT_DIMS, RESNET18, RESNET34, RESNET50, Trunk  # noqa: F401

NARROW_DIMS = (128, 64, 32, 64, 32)
PAD_CHANNELS = 5          # convraw.0 reads cat[fm, image, 5 zero channels] (40 = s2dim + 8 channels by default)

# Sources a call can read besides the outputs of earlier calls:
#   "image"  the input image;
#   "zeros"  the [b, PAD_CHANNELS, H, W] zero channels behind the image;
#   "cat"    torch.cat([xfc, x8s], 1), the one torch op of the step (cat_operands names its operands).


def _last_bn(trunk):
    return "bn3" if trunk.bottleneck else "bn2"


def _stage_output(trunk, layer):
    """The call whose output is layer `layer`'s (1..4): the last block's residual BatchNorm."""
    return f"{trunk.prefix}layer{layer}.{trunk.blocks[layer - 1] - 1}.{_last_bn(trunk)}"


def cat_operands(trunk):
    """The operands of the "cat" source: xfc, then x8s (layer2's output)."""
    return (trunk.prefix + "fc.1", _stage_output(trunk, 2))


class Call(NamedTuple):
    kind: str                      # stem, bn_act, bn_add_relu, conv, maxpool, upsample_cat, head
    name: str                      # the module it stands for: the conv, the BatchNorm, the upsampling, the max-pool
    inputs: Tuple[str, ...]        # where each input comes from: an earlier call's name or a source above
    act: Optional[str] = None      # bn_act: "relu", "leaky" or None
    bn_skip: Optional[str] = None  # bn_add_relu: the downsample's BatchNorm applied to the skip
    dgrad_channels: Optional[int] = None   # conv: input channels that get a data gradient (None: all)

    def params(self):
        """Names of the parameters this call reads."""
        if self.kind in ("stem", "conv"):
            return [self.name + ".weight"]
        if self.kind == "head":
            return [self.name + ".weight", self.name + ".bias"]
        if self.kind in ("bn_act", "bn_add_relu"):
            out = [self.name + ".weight", self.name + ".bias"]
            return out + ([] if self.bn_skip is None else [self.bn_skip + ".weight", self.bn_skip + ".bias"])
        return []

    def batchnorms(self):
        return [m for m in (self.name, self.bn_skip) if m is not None] if self.kind.startswith("bn_") else []


def calls(trunk=RESNET18):
    """The native calls of one forward_train step, in execution order."""
    s2, T = trunk.dims[3], trunk.prefix
    rows = [Call("stem", T + "conv1", ("image",)),
            Call("bn_act", T + "bn1", (T + "conv1",), act="relu"),          # x2s
            Call("maxpool", T + "maxpool", (T + "bn1",))]
    x = T + "maxpool"
    convs = ("conv1", "conv2", "conv3") if trunk.bottleneck else ("conv1", "conv2")
    for layer in range(1, 5):
        for i in range(trunk.blocks[layer - 1]):
            blk = f"{T}layer{layer}.{i}"
            src = x
            # every conv but the last is followed by its BatchNorm + ReLU
            for k, cv in enumerate(convs[:-1]):
                rows += [Call("conv", f"{blk}.{cv}", (src,)),
                         Call("bn_act", f"{blk}.bn{k + 1}", (f"{blk}.{cv}",), act="relu")]
                src = f"{blk}.bn{k + 1}"
            last, bn = f"{blk}.{convs[-1]}", f"{blk}.{_last_bn(trunk)}"
            rows.append(Call("conv", last, (src,)))
            # _stage: a downsample where stride or width changes (layer1 of a Bottleneck trunk widens 64 -> 256)
            if i == 0 and (layer != 1 or trunk.bottleneck):
                rows += [Call("conv", blk + ".downsample.0", (x,)),
                         Call("bn_add_relu", bn, (last, blk + ".downsample.0"), bn_skip=blk + ".downsample.1")]
            else:
                rows.append(Call("bn_add_relu", bn, (last, x)))
            x = bn
    # x4s, x8s, x32s: layer1 / layer2 / layer4's outputs; the decoder's cat order: upsampled features first
    rows += [Call("conv", T + "fc.0", (x,)), Call("bn_act", T + "fc.1", (T + "fc.0",), act="relu"),
             Call("conv", "conv8s.0", ("cat",)), Call("bn_act", "conv8s.1", ("conv8s.0",), act="leaky"),
             Call("upsample_cat", "up8sto4s", ("conv8s.1", _stage_output(trunk, 1))),
             Call("conv", "conv4s.0", ("up8sto4s",)), Call("bn_act", "conv4s.1", ("conv4s.0",), act="leaky"),
             Call("upsample_cat", "up4sto2s", ("conv4s.1", T + "bn1")),
             Call("conv", "conv2s.0", ("up4sto2s",)), Call("bn_act", "conv2s.1", ("conv2s.0",), act="leaky"),
             Call("upsample_cat", "up2storaw", ("conv2s.1", "image", "zeros")),
             Call("conv", "convraw.0", ("up2storaw",), dgrad_channels=s2),
             Call("bn_act", "convraw.1", ("convraw.0",), act="leaky"),
             Call("head", "convraw.3", ("convraw.1",))]
    return rows


def consumers(rows):
    """{source: [(call index, input position), ...]} over the table, in call order."""
    out = {}
    for i, c in enumerate(rows):
        for k, s in enumerate(c.inputs):
            out.setdefault(s, []).append((i, k))
    return out


# ----------------------------------------------------------------------------- capture
class Record:
    """One native call as it ran: its inputs (as passed in), the gradient each of its inputs got from this call alone
    (position -> tensor, for the inputs that require grad), its output and the total gradient that reached the
    output; for BatchNorm calls, the module(s) and their buffers (running_mean, running_var, num_batches_tracked)
    just before the call."""

    def __init__(self, kind, name):
        self.kind, self.name = kind, name
        self.inputs, self.in_grads = [], {}
        self.output = self.out_grad = None
        self.args = {}
        self.snapshots = []


def _store(where, key, grad):
    where[key] = grad.clone()


def _set_out_grad(rec, grad):
    rec.out_grad = grad.clone()


class Capture:
    """Wrappers for the native calls of pvnet_b200.conv that forward_train makes; `install(monkeypatch)` puts them in
    place (forward_train looks `pc.*` up at call time).  Each wrapper records the call, hands it `t.view_as(t)` for
    every input that requires grad with a hook on that view (this consumer's input gradient), and hooks the output
    (the sum over all consumers).  The values passed on are the values received."""

    def __init__(self, net, pc):
        self.pc = pc
        self.maxpool = net._trunk_attr + ".maxpool"
        self.records = []
        self.param_name = {id(p): n for n, p in net.named_parameters()}
        self.module_name = {id(m): n for n, m in net.named_modules()}
        self.orig = {k: getattr(pc, k) for k in ("stem_train", "bn_act", "bn_add_relu", "conv2d_train",
                                                  "maxpool_train", "upsample2x_cat", "upsample2x_into", "head_train")}

    def install(self, monkeypatch):
        for k in self.orig:
            monkeypatch.setattr(self.pc, k, getattr(self, k))

    def _begin(self, kind, name, *inputs):
        rec = Record(kind, name)
        self.records.append(rec)
        passed = []
        for k, t in enumerate(inputs):
            rec.inputs.append(t)
            if isinstance(t, torch.Tensor) and t.requires_grad:
                v = t.view_as(t)
                v.register_hook(functools.partial(_store, rec.in_grads, k))
                passed.append(v)
            else:
                passed.append(t)
        return rec, passed

    @staticmethod
    def _end(rec, y):
        rec.output = y
        if y.requires_grad:
            y.register_hook(functools.partial(_set_out_grad, rec))
        return y

    def _weight_owner(self, w):
        return self.param_name[id(w)].rsplit(".", 1)[0]

    @staticmethod
    def _snapshot(bn):
        return tuple(t.detach().clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked))

    def stem_train(self, x, weight, img, co, mean=None, std=None):
        rec, (xv,) = self._begin("stem", self._weight_owner(weight), x)
        return self._end(rec, self.orig["stem_train"](xv, weight, img, co, mean, std))

    def conv2d_train(self, x, weight, stride=1, dilation=1, dgrad_channels=None):
        rec, (xv,) = self._begin("conv", self._weight_owner(weight), x)
        rec.args = dict(stride=stride, dilation=dilation, dgrad_channels=dgrad_channels)
        return self._end(rec, self.orig["conv2d_train"](xv, weight, stride, dilation, dgrad_channels))

    def bn_act(self, bn, x, act=0):
        rec, (xv,) = self._begin("bn_act", self.module_name[id(bn)], x)
        rec.args = dict(act=act)
        rec.snapshots = [self._snapshot(bn)]
        return self._end(rec, self.orig["bn_act"](bn, xv, act))

    def bn_add_relu(self, bn, a, skip, bn_skip=None):
        rec, (av, sv) = self._begin("bn_add_relu", self.module_name[id(bn)], a, skip)
        rec.args = dict(bn_skip=None if bn_skip is None else self.module_name[id(bn_skip)])
        rec.snapshots = [self._snapshot(m) for m in (bn, bn_skip) if m is not None]
        return self._end(rec, self.orig["bn_add_relu"](bn, av, sv, bn_skip))

    def maxpool_train(self, x):
        rec, (xv,) = self._begin("maxpool", self.maxpool, x)
        return self._end(rec, self.orig["maxpool_train"](xv))

    def upsample2x_cat(self, low, *rest):
        rec, passed = self._begin("upsample_cat", None, low, *rest)
        return self._end(rec, self.orig["upsample2x_cat"](*passed))

    def upsample2x_into(self, low, buf):
        """Recorded as the upsample_cat it stands for: the `rest` inputs are the buffer's channels behind low's (the
        image and zero channels the stem wrote), copied before the call, and the output is the whole buffer."""
        C = low.shape[1]
        rec, (lv,) = self._begin("upsample_cat", None, low)
        rec.inputs += [buf[:, C:C + 3].clone(), buf[:, C + 3:].clone()]
        return self._end(rec, self.orig["upsample2x_into"](lv, buf))

    def head_train(self, y, weight, bias):
        rec, (yv,) = self._begin("head", self._weight_owner(weight), y)
        return self._end(rec, self.orig["head_train"](yv, weight, bias))
