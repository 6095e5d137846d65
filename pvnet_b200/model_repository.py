"""`Resnet18_8s` with the reference's constructor, forward signature and state-dict keys
(zju3dv/pvnet lib/networks/model_repository.py:7-80), backed in eval mode by the native
sm_90a backbone (wgmma implicit-GEMM convs behind include/pvnet_b200.h).

    net = Resnet18_8s(ver_dim=18, seg_dim=2)
    net.load_state_dict(ckpt['net'])          # reference checkpoints load unchanged
    net.cuda().eval()
    seg_pred, ver_pred = net(x)               # [b,2,H,W], [b,18,H,W] views of one tensor

* eval mode on CUDA -> `pvnet_backbone_forward`: BatchNorm folded into TF32 conv weights
  (the reference's cuDNN path also runs TF32 on this hardware: torch's
  `cudnn.allow_tf32` default), fp32 accumulation.  Every convolution runs on wgmma with TF32
  operands: the 7x7/2 stem as a 4x4 conv over the 2x2 space-to-depth image, and convraw.3 (1x1 +
  bias) as a register-A wgmma inside convraw.0's epilogue, fused with torch.argmax over the
  segmentation logits (head weights are rounded to TF32; the fp32 `k_head`/`k_stem` kernels remain as
  the `pvnet_conv_set_mode(1)` test path).  There is no PyTorch fallback in this mode: if the library
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
from torch import nn

from . import _native
from . import conv as pc
from .resnet import resnet18

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
        self.fuse_up = -1            # what pvnet_backbone_set_fused_upsample was last told (-1: library default)
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
        self.fuse_up = -1          # -1 library default (separate launch), 0 separate upsampling launch, 1 fused


class Resnet18_8s(nn.Module):
    def __init__(self, ver_dim, seg_dim, fcdim=256, s8dim=128, s4dim=64, s2dim=32, raw_dim=32):
        super().__init__()
        trunk = resnet18(output_stride=8)
        self.ver_dim = ver_dim
        self.seg_dim = seg_dim
        self._dims = (fcdim, s8dim, s4dim, s2dim, raw_dim)
        trunk.fc = nn.Sequential(nn.Conv2d(trunk.inplanes, fcdim, 3, 1, 1, bias=False), nn.BatchNorm2d(fcdim),
                                 nn.ReLU(True))
        self.resnet18_8s = trunk
        self.conv8s = nn.Sequential(nn.Conv2d(128 + fcdim, s8dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s8dim),
                                    nn.LeakyReLU(0.1, True))
        self.up8sto4s = nn.UpsamplingBilinear2d(scale_factor=2)
        self.conv4s = nn.Sequential(nn.Conv2d(64 + s8dim, s4dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s4dim),
                                    nn.LeakyReLU(0.1, True))
        self.up4sto2s = nn.UpsamplingBilinear2d(scale_factor=2)
        self.conv2s = nn.Sequential(nn.Conv2d(64 + s4dim, s2dim, 3, 1, 1, bias=False), nn.BatchNorm2d(s2dim),
                                    nn.LeakyReLU(0.1, True))
        self.up2storaw = nn.UpsamplingBilinear2d(scale_factor=2)
        self.convraw = nn.Sequential(nn.Conv2d(3 + s2dim, raw_dim, 3, 1, 1, bias=False), nn.BatchNorm2d(raw_dim),
                                     nn.LeakyReLU(0.1, True), nn.Conv2d(raw_dim, seg_dim + ver_dim, 1, 1))
        self._nat = _NativeState()
        self._src_key = None         # set on DataParallel replicas: the source module's weight-version key
        self._frozen = False

    # ------------------------------------------------------------------ PyTorch graph
    def _forward_torch(self, x):
        x2s, x4s, x8s, _x16s, _x32s, xfc = self.resnet18_8s(x)
        fm = self.up8sto4s(self.conv8s(torch.cat([xfc, x8s], 1)))
        fm = self.up4sto2s(self.conv4s(torch.cat([fm, x4s], 1)))
        fm = self.up2storaw(self.conv2s(torch.cat([fm, x2s], 1)))
        out = self.convraw(torch.cat([fm, x], 1))
        return out[:, :self.seg_dim], out[:, self.seg_dim:]

    # ------------------------------------------------------------------ native path
    def _weights_key(self):
        """Identity + version of every parameter and buffer: changes when weights are loaded, moved or
        modified in place.  A DataParallel replica reports its SOURCE module's key (its own tensors are
        fresh broadcast copies on every forward)."""
        if self._src_key is not None:
            return self._src_key
        return tuple((p.data_ptr(), p._version) for p in self.parameters()) + \
               tuple((b.data_ptr(), b._version) for b in self.buffers())

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

    def set_fused_upsample(self, on=None):
        """A/B switch of the 1/2 -> 1 upsampling inside convraw.0's loader (pvnet_backbone_set_fused_upsample):
        None = library default, False / 0 = separate k_upsample2x launch, True / nonzero = fused."""
        self._nat.fuse_up = -1 if on is None else int(bool(on))
        return self

    def _sync_options(self, dev):
        dev = torch.device(dev)
        ent = self._nat.entries[dev.index if dev.index is not None else torch.cuda.current_device()]
        if ent.fuse_up != self._nat.fuse_up:
            _native.check(_native.lib().pvnet_backbone_set_fused_upsample(ent.handle, self._nat.fuse_up),
                          "pvnet_backbone_set_fused_upsample")
            ent.fuse_up = self._nat.fuse_up

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

    def _pack_native(self, device, key):
        L = _native.lib()
        mods = dict(self.named_modules())
        fcdim, s8dim, s4dim, s2dim, raw_dim = self._dims
        handle = ctypes.c_void_p()
        _native.check(L.pvnet_backbone_create(self.ver_dim, self.seg_dim, fcdim, s8dim, s4dim, s2dim, raw_dim,
                                              ctypes.byref(handle)), "pvnet_backbone_create")
        keep = []
        with torch.no_grad():
            for slot, (conv_name, bn_name) in enumerate(_SLOTS):
                conv = mods[conv_name]
                if bn_name is not None:
                    bn = mods[bn_name]
                    w, b = pc.fold_bn(conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
                else:
                    w, b = pc.fold_bn(conv.weight, conv_bias=conv.bias)
                w, b = w.to(device), b.to(device).contiguous()
                if slot == 0:                         # stem: fp32 [tap][cin][cout]
                    packed = w.permute(2, 3, 1, 0).reshape(49, 3, 64).contiguous()
                elif conv_name == "convraw.3":        # head: fp32 [cout][32]
                    packed = pc.round_tf32(w.reshape(w.shape[0], w.shape[1]))   # fused path feeds it to a tf32 MMA
                elif conv_name == "convraw.0":        # cat[fm(s2dim), image(3)] -> s2dim+8 input channels
                    packed = pc.pack_weight(w, cin_pad=pc.cin_padded(s2dim + 8))
                else:
                    packed = pc.pack_weight(w)
                keep += [packed, b]
                _native.check(L.pvnet_backbone_set_conv(handle, slot, packed.data_ptr(), b.data_ptr()),
                              f"pvnet_backbone_set_conv({conv_name})")
            # slot 26: the stem as a 4x4 conv over the 2x2 space-to-depth image (tensor-core path)
            bn = mods["resnet18_8s.bn1"]
            w, b = pc.fold_bn(mods["resnet18_8s.conv1"].weight, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                              bn.eps)
            w4 = pc.pack_stem_s2d(w.to(device))
            b = b.to(device).contiguous()
            keep += [w4, b]
            _native.check(L.pvnet_backbone_set_conv(handle, len(_SLOTS), w4.data_ptr(), b.data_ptr()),
                          "pvnet_backbone_set_conv(stem s2d)")
        return _NativeEntry(handle, keep, key)

    def forward_native(self, x, with_mask=False, mask_dtype=torch.int64, mean=None, std=None, pixel_major=False):
        """x [b,3,H,W] float32 CUDA (normalised) -- or uint8 [b,H,W,3] raw images with `mean`/`std`
        (normalised on the device) -> out [b,seg+ver,H,W] (and the fused argmax mask).
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
            self._sync_options(dev)
            L = _native.lib()
            n = ctypes.c_size_t()
            _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(n)),
                          "pvnet_backbone_workspace_bytes")
            ws = self._workspace(n.value, dev)
            ctot = self.seg_dim + self.ver_dim
            out = torch.empty([b, h, w, ctot] if pixel_major else [b, ctot, h, w], dtype=torch.float32, device=dev)
            _native.check(L.pvnet_backbone_set_output_layout(handle, 1 if pixel_major else 0),
                          "pvnet_backbone_set_output_layout")
            mask = torch.empty([b, h, w], dtype=mask_dtype, device=dev) if with_mask else None
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
            self._sync_options(dev)
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
        """resnet.BasicBlock.forward with its two (three) convolutions, its BatchNorms, ReLUs and residual add on the
        native kernels: bn2, the downsample's BatchNorm, the add and the ReLU are one pass."""
        relu = pc.act_of(blk.relu)
        y = pc.bn_act(blk.bn1, pc.conv2d_train(x, blk.conv1.weight, blk.conv1.stride[0], blk.conv1.dilation[0]), relu)
        y = pc.conv2d_train(y, blk.conv2.weight, 1, blk.conv2.dilation[0])
        if blk.downsample is None:
            return pc.bn_add_relu(blk.bn2, y, x)
        ds = blk.downsample
        return pc.bn_add_relu(blk.bn2, y, pc.conv2d_train(x, ds[0].weight, ds[0].stride[0], 1), ds[1])

    def _check_train_modules(self):
        """ValueError unless conv1, the max-pool and convraw.3 still have the shapes forward_train's kernels
        implement."""
        t = self.resnet18_8s
        c1, mp, hd = t.conv1, t.maxpool, self.convraw[3]
        pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)  # noqa: E731
        if not (isinstance(c1, nn.Conv2d) and tuple(c1.weight.shape) == (64, 3, 7, 7) and c1.stride == (2, 2)
                and c1.padding == (3, 3) and c1.dilation == (1, 1) and c1.groups == 1 and c1.bias is None
                and c1.padding_mode == "zeros"):
            raise ValueError("forward_train: conv1 must be a [64,3,7,7] convolution, stride 2, padding 3, no bias")
        if not (isinstance(mp, nn.MaxPool2d) and pair(mp.kernel_size) == (3, 3) and pair(mp.stride) == (2, 2)
                and pair(mp.padding) == (1, 1) and pair(mp.dilation) == (1, 1) and not mp.ceil_mode
                and not mp.return_indices):
            raise ValueError("forward_train: the max-pool must be 3x3, stride 2, padding 1, dilation 1, no ceil_mode")
        if not (isinstance(hd, nn.Conv2d) and hd.kernel_size == (1, 1) and hd.stride == (1, 1) and hd.padding == (0, 0)
                and hd.dilation == (1, 1) and hd.groups == 1 and hd.bias is not None):
            raise ValueError("forward_train: convraw[3] must be a 1x1 convolution with bias")

    def forward_train(self, x):
        """The train-mode forward (`_forward_torch`) with every layer on the native kernels under autograd:
        * the stem conv1 as pvnet_b200.conv.stem_train (the eval path's space-to-depth tensor-core forward, a wgmma
          weight gradient; the image gets no gradient, so it must not require one: ValueError);
        * the 24 convolutions of slots 1..24 as pvnet_b200.conv.Conv2dNHWC (pvnet_conv2d_nhwc forward, its data
          gradient and pvnet_conv2d_nhwc_wgrad backward);
        * the 25 BatchNorm layers with their ReLU/LeakyReLU and residual adds as pvnet_b200.conv.bn_act / bn_add_relu,
          following each module's own `training` flag, momentum and running statistics;
        * the max-pool as pvnet_b200.conv.maxpool_train (torch's argmax rule, a gather backward);
        * the three upsample-and-concatenate steps of the decoder as pvnet_b200.conv.upsample2x_cat (bit for bit
          torch's forward; a fixed-order backward without atomics);
        * the head convraw.3 as pvnet_b200.conv.head_train (exact fp32 forward, fixed-order fp64 parameter gradients).
        No step uses cuDNN, and the step runs under torch.use_deterministic_algorithms(True).  Activations are
        channels_last.  convraw.0 reads cat[fm, image, 5 zero channels] like the eval path.  Raises ValueError when
        conv1, the max-pool or convraw.3 no longer have the shapes these kernels implement.

        Returns (seg_pred, ver_pred), the channel slices of one contiguous NCHW tensor that the head writes directly:
        the training losses then write a single gradient for it, and read it on their vectorised path.  NetWrapper's
        change: `seg_pred, vertex_pred = self.net.forward_train(image)`."""
        if x.requires_grad:
            raise ValueError("forward_train: the input image must not require grad (it gets no gradient)")
        if not x.is_cuda:
            raise RuntimeError("pvnet_b200: forward_train runs only on CUDA (no CPU fallback)")
        self._check_train_modules()
        cl = torch.channels_last
        x = x.float()
        x_nchw = x.contiguous()                       # the stem's space-to-depth pack reads NCHW
        x = x.contiguous(memory_format=cl)            # convraw.0's concatenated input
        t = self.resnet18_8s
        x2s = pc.bn_act(t.bn1, pc.stem_train(x_nchw, t.conv1.weight), pc.act_of(t.relu))
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
        fm = self._conv_bn_act(self.conv2s, pc.upsample2x_cat(fm, x2s))
        b, _, h, w = x.shape
        pad = torch.zeros(b, 5, h, w, dtype=torch.float32, device=x.device).contiguous(memory_format=cl)
        y = self._conv_bn_act(self.convraw, pc.upsample2x_cat(fm, x, pad), dgrad_channels=fm.shape[1])
        head = self.convraw[3]
        out = pc.head_train(y, head.weight, head.bias)
        return out[:, :self.seg_dim], out[:, self.seg_dim:]

    def forward(self, x, feature_alignment=False):
        if self.training or not x.is_cuda:
            if not self.training and not x.is_cuda:
                raise RuntimeError("pvnet_b200: eval-mode Resnet18_8s runs only on CUDA (no CPU fallback)")
            return self._forward_torch(x)
        out = self.forward_native(x)
        return out[:, :self.seg_dim, :, :], out[:, self.seg_dim:, :, :]
