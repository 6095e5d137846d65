"""`Resnet18_8s`, `Resnet34_8s`, `Resnet50_8s` and `Resnet50_8s_2o` with the reference's constructors, forward
signature and state-dict keys (zju3dv/pvnet lib/networks/model_repository.py:7-300), backed in eval mode by the native
sm_90a backbone (wgmma implicit-GEMM convs behind include/pvnet_b200.h).  Resnet50_8s_2o ends at half resolution
(conv2s with a 1x1 head, DESIGN.md §21).  Resnet18_8s_detector and Resnet18_8s_detector_v2 (model_repository.py:302-331)
are the trunk, up to layer4 or layer2, with a 3x3 one-channel score head (DESIGN.md §22).  Resnet34_8s keeps its trunk under the
attribute `resnet50_8s`, as the reference does (model_repository.py:246), so its checkpoints load unchanged.
The notes below are written for Resnet18_8s; the two deeper networks share every mechanism (`_Resnet8s`), with
raw_dim 64, so their head always runs as the separate fp32 `k_head`.

    net = Resnet18_8s(ver_dim=18, seg_dim=2)
    net.load_state_dict(ckpt['net'])          # reference checkpoints load unchanged
    net.cuda().eval()
    seg_pred, ver_pred = net(x)               # [b,2,H,W], [b,18,H,W] views of one tensor

* eval mode on CUDA -> `pvnet_backbone_forward`: BatchNorm folded into TF32 conv weights
  (the reference's cuDNN path also runs TF32 on this hardware: torch's
  `cudnn.allow_tf32` default), fp32 accumulation.  Every convolution runs on wgmma with TF32
  operands: the 7x7/2 stem as a 4x4 conv over the 2x2 space-to-depth image, and convraw.3 (1x1 +
  bias) as a register-A wgmma inside convraw.0's epilogue, fused with torch.argmax over the
  segmentation logits (head weights are rounded to TF32).  When seg_dim + ver_dim > 32 the head runs
  as the separate fp32 `k_head` kernel.  There is no PyTorch fallback in this mode: if the library
  is missing it raises.
* `nn.DataParallel(net, device_ids=[...])` (the reference's own multi-GPU wrapper,
  tools/train_linemod.py:258, tools/demo.py:160) works: replicas share ONE per-device cache of
  native handles and packed weights (keyed by the source module's weight versions), so weights are
  packed once per device, never per forward, and a handle is destroyed exactly once.
* train mode (BatchNorm batch statistics, autograd; also what tools/demo.py runs because it
  never calls .eval(), SURVEY App. C.6) -> `forward` runs the plain PyTorch graph below, as SURVEY.md §7
  prescribes.  `forward_train` is the same graph with every layer on the native kernels: its 24 trunk/decoder
  convolutions (forward, data and weight gradients, DESIGN.md §14), the upsampling (§15), its 25 BatchNorm layers
  with their activations and residual adds (§16), and the stem, max-pool and head (§17).
"""
from __future__ import annotations

import ctypes
import threading
import weakref

import torch
import torch.nn.functional as F
from torch import nn

from . import _native
from . import conv as pc
from .resnet import Bottleneck, resnet18, resnet34, resnet50

# execution-order conv slots of include/pvnet_b200.h (pvnet_backbone_set_conv)
_SLOTS = [
    ("resnet18_8s.conv1", "resnet18_8s.bn1"),
    ("resnet18_8s.layer1.0.conv1", "resnet18_8s.layer1.0.bn1"), ("resnet18_8s.layer1.0.conv2", "resnet18_8s.layer1.0.bn2"),
    ("resnet18_8s.layer1.1.conv1", "resnet18_8s.layer1.1.bn1"), ("resnet18_8s.layer1.1.conv2", "resnet18_8s.layer1.1.bn2"),
    ("resnet18_8s.layer2.0.conv1", "resnet18_8s.layer2.0.bn1"), ("resnet18_8s.layer2.0.downsample.0", "resnet18_8s.layer2.0.downsample.1"),
    ("resnet18_8s.layer2.0.conv2", "resnet18_8s.layer2.0.bn2"),
    ("resnet18_8s.layer2.1.conv1", "resnet18_8s.layer2.1.bn1"), ("resnet18_8s.layer2.1.conv2", "resnet18_8s.layer2.1.bn2"),
    ("resnet18_8s.layer3.0.conv1", "resnet18_8s.layer3.0.bn1"), ("resnet18_8s.layer3.0.downsample.0", "resnet18_8s.layer3.0.downsample.1"),
    ("resnet18_8s.layer3.0.conv2", "resnet18_8s.layer3.0.bn2"),
    ("resnet18_8s.layer3.1.conv1", "resnet18_8s.layer3.1.bn1"), ("resnet18_8s.layer3.1.conv2", "resnet18_8s.layer3.1.bn2"),
    ("resnet18_8s.layer4.0.conv1", "resnet18_8s.layer4.0.bn1"), ("resnet18_8s.layer4.0.downsample.0", "resnet18_8s.layer4.0.downsample.1"),
    ("resnet18_8s.layer4.0.conv2", "resnet18_8s.layer4.0.bn2"),
    ("resnet18_8s.layer4.1.conv1", "resnet18_8s.layer4.1.bn1"), ("resnet18_8s.layer4.1.conv2", "resnet18_8s.layer4.1.bn2"),
    ("resnet18_8s.fc.0", "resnet18_8s.fc.1"),
    ("conv8s.0", "conv8s.1"), ("conv4s.0", "conv4s.1"), ("conv2s.0", "conv2s.1"), ("convraw.0", "convraw.1"),
    ("convraw.3", None),
]


class _NativeEntry:
    """One device's native backbone: the C handle, the packed weight tensors it points into, and the
    weight-version key it was built from.  The handle is destroyed exactly once, when the entry dies."""

    def __init__(self, handle, keep, key):
        self.handle, self.keep, self.key = handle, keep, key
        self.packs = 1
        self._fin = weakref.finalize(self, _NativeEntry._destroy, handle.value)

    @staticmethod
    def _destroy(handle_value):
        try:
            _native.lib().pvnet_backbone_destroy(ctypes.c_void_p(handle_value))
        except Exception:
            pass


class _NativeState:
    """Shared (by reference) between a module and its DataParallel replicas / shallow copies."""

    def __init__(self):
        self.lock = threading.Lock()
        self.entries = {}          # device index -> _NativeEntry
        self.workspaces = {}       # (device index, stream) -> uint8 tensor
        self.pack_count = 0        # how many times weights were folded + packed (tests assert on it)


def _trunk_slots(trunk, prefix, stages=4, fc=True):
    """(conv, BatchNorm) module names of a trunk in the native plan's order: the stem; per block of layer1..`stages`
    conv1, (conv2,) the downsample, and the conv whose epilogue adds the skip (pvnet_backbone_create_trunk); then
    fc.0 unless fc=False."""
    slots = [(prefix + "conv1", prefix + "bn1")]
    for li in range(1, stages + 1):
        for bi, blk in enumerate(getattr(trunk, f"layer{li}")):
            p = f"{prefix}layer{li}.{bi}."
            names = ["1", "2", "3"] if isinstance(blk, Bottleneck) else ["1", "2"]
            slots += [(f"{p}conv{n}", f"{p}bn{n}") for n in names[:-1]]
            if blk.downsample is not None:
                slots.append((p + "downsample.0", p + "downsample.1"))
            slots.append((f"{p}conv{names[-1]}", f"{p}bn{names[-1]}"))
    return slots + ([(prefix + "fc.0", prefix + "fc.1")] if fc else [])


_DECODER_SLOTS = [("conv8s.0", "conv8s.1"), ("conv4s.0", "conv4s.1"), ("conv2s.0", "conv2s.1"),
                  ("convraw.0", "convraw.1"), ("convraw.3", None)]


class _NativeNet(nn.Module):
    """What every network here shares to run on the native backbone: the per-device cache of C handles and packed
    weights (keyed on the weight versions, shared with DataParallel replicas, dropped on pickling), the workspace,
    the eval forward, `run_stages`, and the trunk's layers in `forward_train`.  Subclasses give the plan
    (`_create_handle`, `_slots`, `_pack_slot`), the trunk (`_trunk`) and the output (`_out_channels`,
    `_out_scale`)."""

    _out_scale = 1                  # the output grid is the input's divided by this

    def __init__(self):
        super().__init__()
        self._nat = _NativeState()
        self._src_key = None         # set on DataParallel replicas: the source module's weight-version key
        self._frozen = False

    # ------------------------------------------------------------------ native path
    def _key_modules(self):
        """The modules whose parameters and buffers the native plan reads."""
        return (self,)

    def _weights_key(self):
        """Identity + version of every parameter and buffer of `_key_modules`: changes when weights are loaded, moved
        or modified in place.  A DataParallel replica reports its SOURCE module's key (its own tensors are
        fresh broadcast copies on every forward)."""
        if self._src_key is not None:
            return self._src_key
        mods = self._key_modules()
        return tuple((p.data_ptr(), p._version) for m in mods for p in m.parameters()) + \
               tuple((b.data_ptr(), b._version) for m in mods for b in m.buffers())

    def _replicate_for_data_parallel(self):
        replica = super()._replicate_for_data_parallel()
        replica._src_key = self._weights_key()       # _nat is shared by reference (shallow __dict__ copy)
        return replica

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_nat", None)                      # C handles and device workspaces do not pickle / deep-copy
        state["_src_key"] = None
        return state

    def __setstate__(self, state):
        super().__setstate__(state)
        self._nat = _NativeState()
        self._src_key = None
        self.__dict__.setdefault("_frozen", False)

    def freeze_native(self, frozen=True):
        """Latency knob: with frozen=True the per-forward staleness check of the packed weights (a walk
        over the 152 state tensors, ~40 us) is skipped; call freeze_native(False) after changing weights."""
        self._frozen = bool(frozen)
        return self

    def native_pack_count(self):
        return self._nat.pack_count

    def _prepare_native(self, device):
        """Fold BatchNorm (eval statistics) into the conv weights, pack them K-major, round
        to TF32, hand the pointers to the C handle.  Redone when any parameter changes; cached per
        device and shared with DataParallel replicas."""
        device = torch.device(device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        nat = self._nat
        ent = nat.entries.get(idx)
        if ent is not None and self._frozen:
            return ent.handle
        key = self._weights_key()
        if ent is not None and ent.key == key:
            return ent.handle
        with nat.lock:
            ent = nat.entries.get(idx)
            if ent is not None and ent.key == key:
                return ent.handle
            ent = self._pack_native(device, key)
            nat.entries[idx] = ent               # the previous entry (if any) is destroyed by its finalizer
            nat.pack_count += 1
            # cached tensor maps of older plans point at the old weights: workspaces keep their address,
            # the new handle plans afresh
            return ent.handle

    def _pack_slot(self, slot, conv_name, conv, w):
        """The packed weight of one conv slot (BatchNorm already folded into w)."""
        if slot == 0:                         # stem: a 4x4 conv over the 2x2 space-to-depth image
            return pc.pack_stem_s2d(w)
        return pc.pack_weight(w)

    def _pack_native(self, device, key):
        L = _native.lib()
        mods = dict(self.named_modules())
        handle = ctypes.c_void_p()
        self._create_handle(handle)
        keep = []
        with torch.no_grad():
            for slot, (conv_name, bn_name) in enumerate(self._slots()):
                conv = mods[conv_name]
                if bn_name is not None:
                    bn = mods[bn_name]
                    w, b = pc.fold_bn(conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
                else:
                    w, b = pc.fold_bn(conv.weight, conv_bias=conv.bias)
                w, b = w.to(device), b.to(device).contiguous()
                packed = self._pack_slot(slot, conv_name, conv, w)
                keep += [packed, b]
                _native.check(L.pvnet_backbone_set_conv(handle, slot, packed.data_ptr(), b.data_ptr()),
                              f"pvnet_backbone_set_conv({conv_name})")
        return _NativeEntry(handle, keep, key)

    def forward_native(self, x, with_mask=False, mask_dtype=torch.int64, mean=None, std=None, pixel_major=False):
        """x [b,3,H,W] float32 CUDA (normalised) -- or uint8 [b,H,W,3] raw images with `mean`/`std`
        (normalised on the device) -> out [b,seg+ver,H,W] (and the fused argmax mask [b,H,W]); H/2 x W/2 for
        Resnet50_8s_2o.
        pixel_major=True returns the same values as out [b,H,W,seg+ver] (one contiguous record per pixel:
        `out[..., seg:].view(b,H,W,K,2)` is the contiguous vertex tensor the voting layer likes best)."""
        if not x.is_cuda:
            raise RuntimeError("pvnet_b200: the native backbone needs a CUDA tensor (there is no CPU path)")
        raw_u8 = x.dtype == torch.uint8
        if raw_u8:
            if x.dim() != 4 or x.shape[3] != 3 or mean is None or std is None:
                raise ValueError("uint8 input must be [b,H,W,3] with mean= and std= (ToTensor + Normalize constants)")
            x = x.contiguous()
            b, h, w, _ = x.shape
        else:
            x = x.contiguous().float()
            b, c, h, w = x.shape
            if c != 3:
                raise ValueError(f"input must be [b,3,H,W], got {tuple(x.shape)}")
        if h % 8 or w % 8:
            raise ValueError(f"H,W must be multiples of 8, got {tuple(x.shape)}")
        dev = x.device
        with torch.cuda.device(dev):
            handle = self._prepare_native(dev)
            L = _native.lib()
            n = ctypes.c_size_t()
            _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)),
                          "pvnet_backbone_workspace_bytes")
            ws = self._workspace(n.value, dev)
            ctot = self._out_channels()
            ho, wo = h // self._out_scale, w // self._out_scale
            out = torch.empty([b, ho, wo, ctot] if pixel_major else [b, ctot, ho, wo], dtype=torch.float32,
                              device=dev)
            _native.check(L.pvnet_backbone_set_output_layout(handle, 1 if pixel_major else 0),
                          "pvnet_backbone_set_output_layout")
            mask = torch.empty([b, ho, wo], dtype=mask_dtype, device=dev) if with_mask else None
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            mptr, msz = (None, 0) if mask is None else (mask.data_ptr(), mask.element_size())
            if raw_u8:
                mean3 = (ctypes.c_float * 3)(*[float(v) for v in mean])
                std3 = (ctypes.c_float * 3)(*[float(v) for v in std])
                _native.check(L.pvnet_backbone_forward_u8(handle, x.data_ptr(), mean3, std3, b, h, w, out.data_ptr(), mptr,
                                                          msz, ws.data_ptr(), ws.numel(), stream),
                              "pvnet_backbone_forward_u8")
            else:
                _native.check(L.pvnet_backbone_forward(handle, x.data_ptr(), b, h, w, out.data_ptr(), mptr, msz,
                                                       ws.data_ptr(), ws.numel(), stream), "pvnet_backbone_forward")
        return (out, mask) if with_mask else out

    def run_stages(self, x, out, mask, lo, hi, pixel_major=False):
        """Stages [lo, hi) of the forward pass (pvnet_backbone_run_stage; stage names:
        pvnet_backbone_stage_name) on caller-provided output tensors -- lets a caller interleave other work
        (e.g. the previous batch's voting layer on a second stream) at a stage boundary.  x float32 [b,3,H,W]."""
        b, _, h, w = x.shape
        dev = x.device
        with torch.cuda.device(dev):
            handle = self._prepare_native(dev)
            L = _native.lib()
            n = ctypes.c_size_t()
            _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)), "pvnet_backbone_workspace_bytes")
            ws = self._workspace(n.value, dev)
            _native.check(L.pvnet_backbone_set_output_layout(handle, 1 if pixel_major else 0), "set_output_layout")
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            for i in range(lo, hi):
                _native.check(L.pvnet_backbone_run_stage(handle, i, x.data_ptr(), b, h, w, out.data_ptr(),
                                                         None if mask is None else mask.data_ptr(),
                                                         0 if mask is None else mask.element_size(), ws.data_ptr(), ws.numel(),
                                                         stream), "pvnet_backbone_run_stage")

    def _workspace(self, nbytes, dev):
        # one persistent workspace per (device, stream) (activations of the largest batch seen); reusing
        # the same address also lets the C handle keep its encoded tensor maps
        dev = torch.device(dev)
        key = (dev.index if dev.index is not None else torch.cuda.current_device(),
               torch.cuda.current_stream(dev).cuda_stream)
        ws = self._nat.workspaces.get(key)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            self._nat.workspaces[key] = ws
        return ws

    # ------------------------------------------------------------------ training path
    @staticmethod
    def _conv_bn_act(seq, x, dgrad_channels=None):
        """nn.Sequential(Conv2d, BatchNorm2d, activation) with the convolution and the BatchNorm + activation on the
        native kernels."""
        conv = seq[0]
        y = pc.conv2d_train(x, conv.weight, conv.stride[0], conv.dilation[0], dgrad_channels)
        return pc.bn_act(seq[1], y, pc.act_of(seq[2]))

    @staticmethod
    def _block_train(blk, x):
        """resnet.BasicBlock.forward (resnet.Bottleneck.forward) with its two (three) convolutions and the downsample,
        its BatchNorms, ReLUs and residual add on the native kernels: the last BatchNorm (bn2, bn3), the downsample's
        BatchNorm, the add and the ReLU are one pass."""
        relu = pc.act_of(blk.relu)
        y = pc.bn_act(blk.bn1, pc.conv2d_train(x, blk.conv1.weight, blk.conv1.stride[0], blk.conv1.dilation[0]), relu)
        if isinstance(blk, Bottleneck):
            y = pc.bn_act(blk.bn2, pc.conv2d_train(y, blk.conv2.weight, blk.conv2.stride[0], blk.conv2.dilation[0]),
                          relu)
            last, bn_last = blk.conv3, blk.bn3
        else:
            last, bn_last = blk.conv2, blk.bn2
        y = pc.conv2d_train(y, last.weight, 1, last.dilation[0])
        if blk.downsample is None:
            return pc.bn_add_relu(bn_last, y, x)
        ds = blk.downsample
        return pc.bn_add_relu(bn_last, y, pc.conv2d_train(x, ds[0].weight, ds[0].stride[0], 1), ds[1])

    def _check_train_modules(self):
        """ValueError unless conv1 and the max-pool still have the shapes forward_train's kernels implement."""
        t = self._trunk()
        c1, mp = t.conv1, t.maxpool
        pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)  # noqa: E731
        if not (isinstance(c1, nn.Conv2d) and tuple(c1.weight.shape) == (64, 3, 7, 7) and c1.stride == (2, 2)
                and c1.padding == (3, 3) and c1.dilation == (1, 1) and c1.groups == 1 and c1.bias is None
                and c1.padding_mode == "zeros"):
            raise ValueError("forward_train: conv1 must be a [64,3,7,7] convolution, stride 2, padding 3, no bias")
        if not (isinstance(mp, nn.MaxPool2d) and pair(mp.kernel_size) == (3, 3) and pair(mp.stride) == (2, 2)
                and pair(mp.padding) == (1, 1) and pair(mp.dilation) == (1, 1) and not mp.ceil_mode
                and not mp.return_indices):
            raise ValueError("forward_train: the max-pool must be 3x3, stride 2, padding 1, dilation 1, no ceil_mode")

    @staticmethod
    def _train_input(x, mean, std):
        """forward_train's input checks (see _Resnet8s.forward_train): the float image, or the uint8 one, and (b, h, w)."""
        if x.requires_grad:
            raise ValueError("forward_train: the input image must not require grad (it gets no gradient)")
        raw_u8 = x.dtype == torch.uint8
        if raw_u8:
            if mean is None or std is None:
                raise ValueError("forward_train: a uint8 image needs mean= and std= (the Normalize constants)")
            if x.dim() != 4 or x.shape[3] != 3:
                raise ValueError(f"forward_train: a uint8 image must be [b,H,W,3], got {tuple(x.shape)}")
        elif mean is not None or std is not None:
            raise ValueError("forward_train: mean= and std= apply to a uint8 image; a float image is already "
                             "normalised")
        if not x.is_cuda:
            raise RuntimeError("pvnet_b200: forward_train runs only on CUDA (no CPU fallback)")
        if raw_u8:
            b, h, w, _ = x.shape
        else:
            x = x.float()
            b, h, w = x.shape[0], x.shape[-2], x.shape[-1]      # [b,3,H,W], checked by the stem
        return x, b, h, w


class _Resnet8s(_NativeNet):
    """The Resnet*_8s graph (a dilated trunk under model_repository.py's decoder) on the native kernels: its plan, the
    eval forward's outputs and `forward_train`.  Subclasses name the trunk attribute (`_trunk_attr`) and the trunk;
    `x4c` / `x8c` are layer1 / layer2's output channels."""

    _trunk_attr = None

    def __init__(self, trunk, ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim):
        super().__init__()
        e = 4 if isinstance(trunk.layer1[0], Bottleneck) else 1
        x4c, x8c = 64 * e, 128 * e
        self.ver_dim = ver_dim
        self.seg_dim = seg_dim
        self._dims = (fcdim, s8dim, s4dim, s2dim, raw_dim)
        trunk.fc = nn.Sequential(nn.Conv2d(trunk.inplanes, fcdim, 3, 1, 1, bias=False), nn.BatchNorm2d(fcdim),
                                 nn.ReLU(True))
        setattr(self, self._trunk_attr, trunk)
        self.conv8s = nn.Sequential(nn.Conv2d(x8c + fcdim, s8dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s8dim),
                                    nn.LeakyReLU(0.1, True))
        self.up8sto4s = nn.UpsamplingBilinear2d(scale_factor=2)
        self.conv4s = nn.Sequential(nn.Conv2d(x4c + s8dim, s4dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s4dim),
                                    nn.LeakyReLU(0.1, True))
        self.up4sto2s = nn.UpsamplingBilinear2d(scale_factor=2)
        self._init_tail(ver_dim, seg_dim, s4dim, s2dim, raw_dim)

    # ------------------------------------------------------------------ the decoder's tail
    # What follows conv4s differs between the full-resolution networks (conv2s, x2 upsampling, convraw) and
    # Resnet50_8s_2o (conv2s with a 1x1 head at half resolution).  These hooks and attributes, and _create_handle, are
    # all that differ.
    _decoder_slots = _DECODER_SLOTS
    _image_slot = "convraw.0"       # the convolution that reads the image slice as its second source
    _head_slot = "convraw.3"        # the 1x1 head with bias

    def _init_tail(self, ver_dim, seg_dim, s4dim, s2dim, raw_dim):
        """conv2s and everything after it (model_repository.py:50-57)."""
        self.conv2s = nn.Sequential(nn.Conv2d(64 + s4dim, s2dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s2dim),
                                    nn.LeakyReLU(0.1, True))
        self.up2storaw = nn.UpsamplingBilinear2d(scale_factor=2)
        self.convraw = nn.Sequential(nn.Conv2d(3 + s2dim, raw_dim, 3, 1, 1, bias=False), nn.BatchNorm2d(raw_dim),
                                     nn.LeakyReLU(0.1, True), nn.Conv2d(raw_dim, seg_dim + ver_dim, 1, 1))

    def _tail_torch(self, fm, x2s, x):
        """The PyTorch graph from conv4s's upsampled output to the head's output."""
        fm = self.up2storaw(self.conv2s(torch.cat([fm, x2s], 1)))
        return self.convraw(torch.cat([fm, x], 1))

    def _train_tail_input(self, b, h, w, device):
        """forward_train: the channels_last input buffer of the image-reading convolution, the channel at which the
        stem writes the image and its 5 zero channels, and the stem that writes them.  Here convraw.0's cat[fm, image,
        5 zeros]: pvnet_b200.conv.stem_train fills channels [s2dim, s2dim+8) now, the decoder's upsampling channels
        [0, s2dim) at the end."""
        s2dim = self.conv2s[0].out_channels
        return torch.empty(b, s2dim + 8, h, w, dtype=torch.float32, device=device,
                           memory_format=torch.channels_last), s2dim, pc.stem_train

    def _train_tail(self, fm, x2s, buf):
        """forward_train from conv4s's output to the head's input: (head input, head module)."""
        fm = self._conv_bn_act(self.conv2s, pc.upsample2x_cat(fm, x2s))
        y = self._conv_bn_act(self.convraw, pc.upsample2x_into(fm, buf), dgrad_channels=fm.shape[1])
        return y, self.convraw[3]

    # ------------------------------------------------------------------ PyTorch graph
    def _trunk(self):
        return getattr(self, self._trunk_attr)

    def _slots(self):
        """Execution-order (conv, BatchNorm) module names of the native conv slots."""
        return _trunk_slots(self._trunk(), self._trunk_attr + ".") + self._decoder_slots

    def _out_channels(self):
        return self.seg_dim + self.ver_dim

    def _pack_slot(self, slot, conv_name, conv, w):
        if conv_name == "convraw.3" and self._dims[4] == 32:   # head: fp32 [cout][32]
            return pc.round_tf32(w.reshape(w.shape[0], w.shape[1]))   # fused path feeds it to a tf32 MMA
        if conv_name == self._head_slot:    # head: fp32 [cout][raw], exact in k_head
            return w.reshape(w.shape[0], w.shape[1]).contiguous()
        if conv_name == self._image_slot:   # cat[features, image(3)] -> features+8 input channels
            return pc.pack_weight(w, cin_pad=pc.cin_padded(conv.in_channels + 5))
        return super()._pack_slot(slot, conv_name, conv, w)

    def _create_handle(self, handle):
        """pvnet_backbone_create_trunk for this trunk."""
        t = self._trunk()
        kind = 1 if isinstance(t.layer1[0], Bottleneck) else 0
        blocks = (ctypes.c_int * 4)(*(len(getattr(t, f"layer{i}")) for i in range(1, 5)))
        _native.check(_native.lib().pvnet_backbone_create_trunk(kind, blocks, self.ver_dim, self.seg_dim, *self._dims,
                                                                ctypes.byref(handle)), "pvnet_backbone_create_trunk")

    def _forward_torch(self, x):
        x2s, x4s, x8s, _x16s, _x32s, xfc = self._trunk()(x)
        fm = self.up8sto4s(self.conv8s(torch.cat([xfc, x8s], 1)))
        fm = self.up4sto2s(self.conv4s(torch.cat([fm, x4s], 1)))
        out = self._tail_torch(fm, x2s, x)
        return out[:, :self.seg_dim], out[:, self.seg_dim:]

    def _check_train_modules(self):
        """ValueError unless conv1, the max-pool and the head (convraw.3; conv2s.3 in Resnet50_8s_2o) still have the
        shapes forward_train's kernels implement."""
        super()._check_train_modules()
        hd = self.get_submodule(self._head_slot)
        if not (isinstance(hd, nn.Conv2d) and hd.kernel_size == (1, 1) and hd.stride == (1, 1) and hd.padding == (0, 0)
                and hd.dilation == (1, 1) and hd.groups == 1 and hd.bias is not None):
            seq, i = self._head_slot.split(".")
            raise ValueError(f"forward_train: {seq}[{i}] must be a 1x1 convolution with bias")


    def forward_train(self, x, mean=None, std=None):
        """The train-mode forward (`_forward_torch`) with every layer on the native kernels under autograd:
        * the stem conv1 as pvnet_b200.conv.stem_train (the eval path's space-to-depth tensor-core forward, a wgmma
          weight gradient; the image gets no gradient, so it must not require one: ValueError), which also writes the
          image and 5 zero channels into convraw.0's input buffer, allocated once per step;
        * the 24 convolutions of slots 1..24 as pvnet_b200.conv.Conv2dNHWC (pvnet_conv2d_nhwc forward, its data
          gradient and pvnet_conv2d_nhwc_wgrad backward);
        * the 25 BatchNorm layers with their ReLU/LeakyReLU and residual adds as pvnet_b200.conv.bn_act / bn_add_relu,
          following each module's own `training` flag, momentum and running statistics;
        * the max-pool as pvnet_b200.conv.maxpool_train (torch's argmax rule, a gather backward);
        * the three upsample-and-concatenate steps of the decoder as pvnet_b200.conv.upsample2x_cat (bit for bit
          torch's forward; a fixed-order backward without atomics), the last one as upsample2x_into, which writes the
          upsampled features into convraw.0's input buffer in place: no image copy and no concatenation copy;
        * the head convraw.3 as pvnet_b200.conv.head_train (exact fp32 forward, fixed-order fp64 parameter gradients).
        No step uses cuDNN, and the step runs under torch.use_deterministic_algorithms(True).  Activations are
        channels_last.  convraw.0 reads cat[fm, image, 5 zero channels] like the eval path.  Raises ValueError when
        conv1, the max-pool or convraw.3 no longer have the shapes these kernels implement.

        Returns (seg_pred, ver_pred), the channel slices of one contiguous NCHW tensor that the head writes directly:
        the training losses then write a single gradient for it, and read it on their vectorised path.  NetWrapper's
        change: `seg_pred, vertex_pred = self.net.forward_train(image)`.

        x may also be the loader's raw uint8 [b,H,W,3] image (before ToTensor), with mean= and std= the Normalize
        constants (3 numbers each), as forward_native takes it: the stem's pack normalises it on the device exactly as
        ToTensor + Normalize do on the CPU, so no float image exists.  Every output, gradient and running statistic
        is that of the float path on the normalised image.  ValueError for a uint8 input without mean and std, for
        mean or std with a float input, and for a uint8 input that is not [b,H,W,3]."""
        x, b, h, w = self._train_input(x, mean, std)
        self._check_train_modules()
        t = self._trunk()
        tail_in, co, stem = self._train_tail_input(b, h, w, x.device)
        x2s = pc.bn_act(t.bn1, stem(x, t.conv1.weight, tail_in, co, mean, std), pc.act_of(t.relu))
        x4s = pc.maxpool_train(x2s)
        for blk in t.layer1:
            x4s = self._block_train(blk, x4s)
        x8s = x4s
        for blk in t.layer2:
            x8s = self._block_train(blk, x8s)
        x32s = x8s
        for blk in (*t.layer3, *t.layer4):
            x32s = self._block_train(blk, x32s)
        xfc = self._conv_bn_act(t.fc, x32s)
        fm = self._conv_bn_act(self.conv8s, torch.cat([xfc, x8s], 1))
        fm = self._conv_bn_act(self.conv4s, pc.upsample2x_cat(fm, x4s))
        y, head = self._train_tail(fm, x2s, tail_in)
        out = pc.head_train(y, head.weight, head.bias)
        return out[:, :self.seg_dim], out[:, self.seg_dim:]

    def forward(self, x, feature_alignment=False):
        if self.training or not x.is_cuda:
            if not self.training and not x.is_cuda:
                raise RuntimeError(f"pvnet_b200: eval-mode {type(self).__name__} runs only on CUDA (no CPU fallback)")
            return self._forward_torch(x)
        out = self.forward_native(x)
        return out[:, :self.seg_dim, :, :], out[:, self.seg_dim:, :, :]


class Resnet18_8s(_Resnet8s):
    _trunk_attr = "resnet18_8s"

    def __init__(self, ver_dim, seg_dim, fcdim=256, s8dim=128, s4dim=64, s2dim=32, raw_dim=32):
        super().__init__(resnet18(output_stride=8), ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim)

    def _slots(self):
        return _SLOTS

    def _create_handle(self, handle):
        fcdim, s8dim, s4dim, s2dim, raw_dim = self._dims
        _native.check(_native.lib().pvnet_backbone_create(self.ver_dim, self.seg_dim, fcdim, s8dim, s4dim, s2dim,
                                                          raw_dim, ctypes.byref(handle)), "pvnet_backbone_create")


class Resnet34_8s(_Resnet8s):
    """The reference's Resnet34_8s (model_repository.py:226-300): 3-4-6-3 BasicBlocks, stored as `resnet50_8s`."""
    _trunk_attr = "resnet50_8s"

    def __init__(self, ver_dim, seg_dim, fcdim=384, s8dim=256, s4dim=128, s2dim=64, raw_dim=64):
        super().__init__(resnet34(output_stride=8), ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim)


class Resnet50_8s(_Resnet8s):
    """The reference's Resnet50_8s (model_repository.py:82-156): 3-4-6-3 Bottlenecks."""
    _trunk_attr = "resnet50_8s"

    def __init__(self, ver_dim, seg_dim, fcdim=384, s8dim=256, s4dim=128, s2dim=64, raw_dim=64):
        super().__init__(resnet50(output_stride=8), ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim)


class Resnet50_8s_2o(_Resnet8s):
    """The reference's Resnet50_8s_2o (model_repository.py:158-224): Resnet50_8s's trunk, fc, conv8s and conv4s, then
    conv2s over cat[up(conv4s), x2s, x_ds] -- x_ds = F.interpolate(x, scale_factor=0.5, mode='bilinear') -- with its
    1x1 head conv2s.3.  The output is at half the input's resolution: [b,seg+ver,H/2,W/2] (mask [b,H/2,W/2]).  There
    is no convraw and no x2 upsampling to full resolution.  Keypoints voted from this output are in the pixel
    coordinates of its H/2 x W/2 grid, as the reference's voting layer gives them for this network."""
    _trunk_attr = "resnet50_8s"
    _decoder_slots = [("conv8s.0", "conv8s.1"), ("conv4s.0", "conv4s.1"), ("conv2s.0", "conv2s.1"),
                      ("conv2s.3", None)]
    _image_slot = "conv2s.0"
    _head_slot = "conv2s.3"
    _out_scale = 2

    def __init__(self, ver_dim, seg_dim, fcdim=384, s8dim=256, s4dim=128, s2dim=64):
        super().__init__(resnet50(output_stride=8), ver_dim, seg_dim, fcdim, s8dim, s4dim, s2dim, None)

    def _init_tail(self, ver_dim, seg_dim, s4dim, s2dim, raw_dim):
        self.conv2s = nn.Sequential(nn.Conv2d(3 + 64 + s4dim, s2dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s2dim),
                                    nn.LeakyReLU(0.1, True), nn.Conv2d(s2dim, seg_dim + ver_dim, 1, 1))

    def _tail_torch(self, fm, x2s, x):
        x_ds = F.interpolate(x, scale_factor=0.5, mode="bilinear", align_corners=False)
        return self.conv2s(torch.cat([fm, x2s, x_ds], 1))

    def _create_handle(self, handle):
        t = self._trunk()
        blocks = (ctypes.c_int * 4)(*(len(getattr(t, f"layer{i}")) for i in range(1, 5)))
        _native.check(_native.lib().pvnet_backbone_create_trunk_2o(1, blocks, self.ver_dim, self.seg_dim,
                                                                   *self._dims[:4], ctypes.byref(handle)),
                      "pvnet_backbone_create_trunk_2o")

    def _train_tail_input(self, b, h, w, device):
        """conv2s.0's cat[up(conv4s), x2s, x_ds, 5 zeros] at H/2 x W/2: pvnet_b200.conv.stem_train_half writes x_ds
        and the zeros into channels [s4dim+64, s4dim+72) now, the decoder the channels before them at the end."""
        c = self.conv2s[0].in_channels + 5
        return torch.empty(b, c, h // 2, w // 2, dtype=torch.float32, device=device,
                           memory_format=torch.channels_last), c - 8, pc.stem_train_half

    def _train_tail(self, fm, x2s, buf):
        y = self._conv_bn_act(self.conv2s, pc.upsample2x_into(fm, buf, x2s), dgrad_channels=buf.shape[1] - 8)
        return y, self.conv2s[3]


class _Detector(_NativeNet):
    """What the two detectors share: the dilated ResNet-18 trunk up to layer `_last_stage`, then the 3x3 one-channel
    score head `_score_slot` (Conv2d(C, 1, 3, 1, 1) with bias).  The output is the score map [b,1,H/8,W/8]; there is
    no segmentation output.  Eval mode on CUDA runs pvnet_backbone_create_detector's plan: the trunk stages are
    Resnet18_8s's, then the head in exact fp32 (DESIGN.md §22)."""

    _out_scale = 8
    _last_stage = 4
    _prefix = "resnet18_8s."
    _score_slot = "resnet18_8s.fc"

    def _trunk(self):
        return self.resnet18_8s

    def _out_channels(self):
        return 1

    def _slots(self):
        return _trunk_slots(self._trunk(), self._prefix, self._last_stage, fc=False) + [(self._score_slot, None)]

    def _pack_slot(self, slot, conv_name, conv, w):
        if conv_name == self._score_slot:     # fp32 [9][C], exact in k_head3x3
            return pc.pack_head3x3(w)
        return super()._pack_slot(slot, conv_name, conv, w)

    def _create_handle(self, handle):
        t = self._trunk()
        kind = 1 if isinstance(t.layer1[0], Bottleneck) else 0
        blocks = (ctypes.c_int * 4)(*(len(getattr(t, f"layer{i}")) for i in range(1, 5)))
        _native.check(_native.lib().pvnet_backbone_create_detector(kind, blocks, self._last_stage,
                                                                   ctypes.byref(handle)),
                      "pvnet_backbone_create_detector")

    def forward_native(self, x, with_mask=False, mask_dtype=torch.int64, mean=None, std=None, pixel_major=False):
        """x [b,3,H,W] float32 CUDA (normalised) -- or uint8 [b,H,W,3] raw images with `mean`/`std` -> the score map
        [b,1,H/8,W/8].  ValueError for with_mask=True or pixel_major=True: a detector has no segmentation output."""
        if with_mask or pixel_major:
            raise ValueError(f"{type(self).__name__} returns one score map: with_mask and pixel_major do not apply")
        return super().forward_native(x, mean=mean, std=std)

    def _check_train_modules(self):
        """ValueError unless conv1, the max-pool and the score head still have the shapes forward_train's kernels
        implement."""
        super()._check_train_modules()
        hd = self.get_submodule(self._score_slot)
        if not (isinstance(hd, nn.Conv2d) and hd.out_channels == 1 and hd.kernel_size == (3, 3)
                and hd.stride == (1, 1) and hd.padding == (1, 1) and hd.dilation == (1, 1) and hd.groups == 1
                and hd.bias is not None and hd.padding_mode == "zeros" and hd.in_channels % 32 == 0
                and hd.in_channels <= 512):
            raise ValueError(f"forward_train: {self._score_slot} must be a 3x3 convolution to one channel, padding 1, "
                             "with bias, over at most 512 channels (a multiple of 32)")

    def forward_train(self, x, mean=None, std=None):
        """The train-mode forward (`_forward_torch`) with every layer on the native kernels under autograd, as
        _Resnet8s.forward_train runs the trunk: the stem (pvnet_b200.conv.stem_train_half; its image output goes to
        a scratch buffer), BatchNorm + ReLU, the max-pool, the blocks of layer1..`_last_stage`, and the score head as
        pvnet_b200.conv.head3x3_train (exact fp32 forward, fixed-order fp64 parameter gradients).  The same input
        contract and errors as _Resnet8s.forward_train; returns the score map [b,1,H/8,W/8]."""
        x, _b, _h, _w = self._train_input(x, mean, std)
        self._check_train_modules()
        t = self._trunk()
        y = pc.bn_act(t.bn1, pc.stem_train_half(x, t.conv1.weight, None, 0, mean, std), pc.act_of(t.relu))
        y = pc.maxpool_train(y)
        for li in range(1, self._last_stage + 1):
            for blk in getattr(t, f"layer{li}"):
                y = self._block_train(blk, y)
        hd = self.get_submodule(self._score_slot)
        return pc.head3x3_train(y, hd.weight, hd.bias)

    def forward(self, x):
        if self.training or not x.is_cuda:
            if not self.training and not x.is_cuda:
                raise RuntimeError(f"pvnet_b200: eval-mode {type(self).__name__} runs only on CUDA (no CPU fallback)")
            return self._forward_torch(x)
        return self.forward_native(x)


class Resnet18_8s_detector(_Detector):
    """The reference's Resnet18_8s_detector (model_repository.py:302-316): the dilated ResNet-18 trunk with its fc
    replaced by Conv2d(512, 1, 3, 1, 1) with bias, returning the score map [b,1,H/8,W/8] from layer4's output.  The
    trunk's init loop runs before fc is assigned, so fc keeps nn.Conv2d's default initialisation, as in the
    reference."""

    def __init__(self):
        super().__init__()
        self.resnet18_8s = resnet18(output_stride=8)
        self.resnet18_8s.fc = nn.Conv2d(self.resnet18_8s.inplanes, 1, 3, 1, 1)

    def _forward_torch(self, x):
        _, _, _, _, _, xfc = self.resnet18_8s(x)
        return xfc


class Resnet18_8s_detector_v2(_Detector):
    """The reference's Resnet18_8s_detector_v2 (model_repository.py:318-331): `base_detector`'s stem, layer1 and
    layer2 (its parameters, shared) and out_conv = Conv2d(128, 1, 3, 1, 1) with bias, returning [b,1,H/8,W/8] from
    layer2's output.  The base's layer3, layer4 and fc stay in the state dict but are not used; the native cache is
    keyed on the modules that are, so updating the base's stem or layer1/2 repacks this network."""

    _last_stage = 2
    _prefix = "base_detector.resnet18_8s."
    _score_slot = "out_conv"

    def __init__(self, base_detector):
        super().__init__()
        self.base_detector = base_detector
        self.out_conv = nn.Conv2d(128, 1, 3, 1, 1)

    def _trunk(self):
        return self.base_detector.resnet18_8s

    def _key_modules(self):
        t = self._trunk()
        return (t.conv1, t.bn1, t.layer1, t.layer2, self.out_conv)

    def _forward_torch(self, x):
        t = self._trunk()
        x2s = t.relu(t.bn1(t.conv1(x)))
        x8s = t.layer2(t.layer1(t.maxpool(x2s)))
        return self.out_conv(x8s)
