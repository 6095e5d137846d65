"""Validation losses on the device: the reference's lib/utils/net_utils.py (`smooth_l1_loss`,
`compute_precision_recall`) and the cross-entropy of NetWrapper.forward (tools/train_linemod.py:79-91), over the C ABI
(`pvnet_seg_vertex_losses` in include/pvnet_b200.h, pvnet_b200/csrc/losses.cu), plus the host-side helpers the
reference's entry points import from that module.

    smooth_l1_loss(vertex_pred, vertex_targets, vertex_weights, sigma=1.0, normalize=True, reduce=True)
    compute_precision_recall(scores, target, reduce=False)
    seg_vertex_losses(seg_pred, vertex_pred, mask, vertex, vertex_weights)
                                   -> (loss_seg, loss_vertex, precision, recall), all four in one launch pair
    vertex_targets(mask, hcoords, use_motion=False)
                                   the loader's ground-truth vertex field [b,2K,h,w] (compute_vertex_hcoords)
    seg_vertex_losses_from_keypoints(seg_pred, vertex_pred, mask, hcoords, vertex_weights, use_motion=False)
                                   seg_vertex_losses with that field computed in registers, never stored
    NetWrapper(net)                the reference's NetWrapper with the fused call in eval / no_grad
    AverageMeter, Recorder, load_model, save_model, adjust_learning_rate, set_learning_rate

Inputs are read in place through their strides (seg_pred / vertex_pred may be channel slices of the network's one
output tensor).  When grad is enabled and an input requires grad (training; tools/demo.py, which runs the network in
train mode) the functions evaluate the same semantics as torch expressions so that backward() works, as
Resnet18_8s runs its train mode in PyTorch.  Otherwise there is no CPU path: CPU tensors raise RuntimeError.
Importing this module loads neither tensorboardX, easydict, torchvision nor matplotlib.
"""
from __future__ import annotations

import ctypes
import os
import re

import torch
from torch import nn
from torch.nn import functional as F

from . import _native

IGNORE_INDEX = -100                         # nn.CrossEntropyLoss's default
_MASK_DTYPES = (torch.int64, torch.int32, torch.uint8, torch.bool)


def _use_torch(*xs):
    return torch.is_grad_enabled() and any(isinstance(x, torch.Tensor) and x.requires_grad for x in xs)


def _strides(x, n):
    """Element strides of x as a ctypes int64[n] (the stride along the last dimension forced to 1, as the C ABI
    requires; a tensor whose last dimension is not unit-stride is copied first)."""
    if x.shape[-1] != 1 and x.stride(-1) != 1:
        x = x.contiguous()
    s = list(x.stride())
    s[-1] = 1
    return x, (ctypes.c_int64 * n)(*s)


def _check_float(name, x):
    if x.dtype != torch.float32:
        raise ValueError(f"{name} must be float32, got {x.dtype}")


def _check_vertex(vertex_pred, vertex_targets, vertex_weights):
    for name, x in (("vertex_pred", vertex_pred), ("vertex_targets", vertex_targets),
                    ("vertex_weights", vertex_weights)):
        _check_float(name, x)
    if vertex_pred.dim() != 4 or vertex_targets.shape != vertex_pred.shape:
        raise ValueError(f"vertex_pred {tuple(vertex_pred.shape)} and vertex_targets {tuple(vertex_targets.shape)} "
                         "must both be [b,ver_dim,h,w]")
    b, _, h, w = vertex_pred.shape
    if tuple(vertex_weights.shape) != (b, 1, h, w):
        raise ValueError(f"vertex_weights must be [b,1,h,w] = {(b, 1, h, w)}, got {tuple(vertex_weights.shape)}")


def _check_keypoints(mask, hcoords):
    if mask.dim() != 3:
        raise ValueError(f"mask must be [b,h,w], got {tuple(mask.shape)}")
    if mask.dtype not in _MASK_DTYPES:
        raise ValueError(f"mask dtype {mask.dtype} is not one of int64, int32, uint8, bool")
    if hcoords.dim() != 3 or hcoords.shape[0] != mask.shape[0] or hcoords.shape[1] < 1 or hcoords.shape[2] != 3:
        raise ValueError(f"hcoords must be [b,K,3] with b = {mask.shape[0]} and K >= 1, got {tuple(hcoords.shape)}")
    if hcoords.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"hcoords must be float32 or float64, got {hcoords.dtype}")


def _check_seg(scores, target):
    _check_float("seg_pred", scores)
    if scores.dim() != 4:
        raise ValueError(f"seg_pred must be [b,C,h,w], got {tuple(scores.shape)}")
    b, _, h, w = scores.shape
    if tuple(target.shape) != (b, h, w):
        raise ValueError(f"mask must be [b,h,w] = {(b, h, w)}, got {tuple(target.shape)}")
    if target.dtype not in _MASK_DTYPES:
        raise ValueError(f"mask dtype {target.dtype} is not one of int64, int32, uint8, bool")


def _native_losses(seg=None, mask=None, pred=None, tgt=None, wgt=None, sigma=1.0, normalize=True,
                   want=("seg", "ver", "precision", "recall"), hcoords=None, use_motion=False):
    """One pvnet_seg_vertex_losses call (pvnet_seg_vertex_losses_keypoints when `hcoords` replaces `tgt`); returns
    {part: tensor} for the parts in `want`."""
    xs = [x for x in (seg, mask, pred, tgt, wgt, hcoords) if x is not None]
    if not all(x.is_cuda for x in xs):
        raise RuntimeError("pvnet_b200: the validation losses need CUDA tensors (there is no CPU path)")
    dev = xs[0].device
    if any(x.device != dev for x in xs):
        raise ValueError("all inputs must be on the same device")
    ref = seg if seg is not None else pred
    b, _, h, w = ref.shape
    L = _native.lib()
    args = []
    C = vd = 0
    if seg is not None:
        seg, s_seg = _strides(seg, 4)
        C = seg.shape[1]
        args += [seg.data_ptr(), s_seg]
    else:
        args += [None, None]
    if mask is not None:
        mask, s_mask = _strides(mask, 3)
        args += [mask.data_ptr(), mask.element_size(), s_mask]
    else:
        args += [None, 0, None]
    if pred is not None:
        pred, s_pred = _strides(pred, 4)
        vd = pred.shape[1]
        args += [pred.data_ptr(), s_pred]
        if hcoords is None:
            tgt, s_tgt = _strides(tgt, 4)
            args += [tgt.data_ptr(), s_tgt]
        else:
            hcoords = hcoords.detach().contiguous()
            args += [hcoords.data_ptr(), int(hcoords.dtype == torch.float64), int(bool(use_motion))]
        wgt, s_wgt = _strides(wgt, 4)
        args += [wgt.data_ptr(), s_wgt]
    else:
        args += [None] * (6 if hcoords is None else 7)
    out = {}
    for part in want:
        shape = [b, vd, h, w] if part == "ver" and not normalize else [b]
        out[part] = torch.empty(shape, dtype=torch.float32, device=dev)
    nbytes = ctypes.c_size_t()
    _native.check(L.pvnet_seg_vertex_losses_workspace_bytes(b, h, w, ctypes.byref(nbytes)),
                  "pvnet_seg_vertex_losses_workspace_bytes")
    ws = torch.empty([nbytes.value], dtype=torch.uint8, device=dev)
    ptr = {k: v.data_ptr() for k, v in out.items()}
    name = "pvnet_seg_vertex_losses" if hcoords is None else "pvnet_seg_vertex_losses_keypoints"
    with torch.cuda.device(dev):
        _native.check(getattr(L, name)(*args, b, h, w, C, vd, float(sigma), int(bool(normalize)),
                                       ptr.get("seg"), ptr.get("ver"), ptr.get("precision"), ptr.get("recall"),
                                       ws.data_ptr(), nbytes.value,
                                       ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                      name)
    return out


# ----------------------------------------------------------------------------- torch expressions (grad mode)
def _smooth_l1_torch(vertex_pred, vertex_targets, vertex_weights, sigma, normalize):
    s2 = sigma ** 2
    diff = vertex_weights * (vertex_pred - vertex_targets)
    ad = diff.abs()
    inside = (ad < 1.0 / s2).detach().float()
    in_loss = diff * diff * (s2 / 2.0) * inside + (ad - 0.5 / s2) * (1.0 - inside)
    if normalize:
        b, vd = vertex_pred.shape[:2]
        in_loss = in_loss.reshape(b, -1).sum(1) / (vd * vertex_weights.reshape(b, -1).sum(1) + 1e-3)
    return in_loss


def _cross_entropy_torch(seg_pred, mask):
    """Per-image mean of the per-pixel cross-entropy with ignore_index -100; an image holding any other target
    outside [0,C) gets NaN (where nn.CrossEntropyLoss would raise a device-side assert)."""
    b, C = seg_pred.shape[:2]
    t = mask.long()
    ignored = t == IGNORE_INDEX
    valid = (t >= 0) & (t < C)
    logp = F.log_softmax(seg_pred, 1).gather(1, t.clamp(0, C - 1)[:, None])[:, 0]
    term = torch.where(valid, -logp, torch.zeros_like(logp))
    loss = term.reshape(b, -1).mean(1)
    bad = (~(valid | ignored)).reshape(b, -1).any(1)
    return loss.masked_fill(bad, float("nan"))


def _precision_recall_torch(scores, target):
    b = scores.shape[0]
    p = scores.argmax(1).long().reshape(b, -1)
    t = target.long().reshape(b, -1)
    tp, fp, fn = (p * t).sum(1), (p * (1 - t)).sum(1), ((1 - p) * t).sum(1)
    num = tp.float() + 1
    return num / ((tp.float() + fp.float()) + 1), num / ((tp.float() + fn.float()) + 1)


# ------------------------------------------------------------------------------------------ public functions
def smooth_l1_loss(vertex_pred, vertex_targets, vertex_weights, sigma=1.0, normalize=True, reduce=True):
    """net_utils.py:54-80.  vertex_pred, vertex_targets [b,ver_dim,h,w], vertex_weights [b,1,h,w], float32.
    normalize: per-image sum(in) / (ver_dim * sum(w) + 1e-3) -> [b]; otherwise the elementwise loss [b,ver_dim,h,w],
    bit-identical to torch's fp32 ops.  `reduce` is accepted and, as in the reference (whose mean is discarded),
    leaves the result per image."""
    _check_vertex(vertex_pred, vertex_targets, vertex_weights)
    if _use_torch(vertex_pred, vertex_targets, vertex_weights):
        return _smooth_l1_torch(vertex_pred, vertex_targets, vertex_weights, sigma, normalize)
    return _native_losses(pred=vertex_pred, tgt=vertex_targets, wgt=vertex_weights, sigma=sigma, normalize=normalize,
                          want=("ver",))["ver"]


def compute_precision_recall(scores, target, reduce=False):
    """net_utils.py:329-348.  scores [b,C,h,w] float32, target [b,h,w] (int64, int32, uint8 or bool) ->
    precision, recall float32 [b] (their batch means with reduce=True)."""
    _check_seg(scores, target)
    if _use_torch(scores):
        precision, recall = _precision_recall_torch(scores, target)
    else:
        r = _native_losses(seg=scores, mask=target, want=("precision", "recall"))
        precision, recall = r["precision"], r["recall"]
    if reduce:
        precision, recall = torch.mean(precision), torch.mean(recall)
    return precision, recall


def seg_vertex_losses(seg_pred, vertex_pred, mask, vertex, vertex_weights):
    """The four per-image figures of NetWrapper.forward (train_linemod.py:87-90) in one pass:
    loss_seg (cross-entropy, mean over pixels), loss_vertex (smooth_l1_loss, normalize=True), precision, recall;
    each float32 [b]."""
    _check_seg(seg_pred, mask)
    _check_vertex(vertex_pred, vertex, vertex_weights)
    if seg_pred.shape[0] != vertex_pred.shape[0] or seg_pred.shape[2:] != vertex_pred.shape[2:]:
        raise ValueError(f"seg_pred {tuple(seg_pred.shape)} and vertex_pred {tuple(vertex_pred.shape)} differ in b,h,w")
    if _use_torch(seg_pred, vertex_pred, vertex, vertex_weights):
        precision, recall = _precision_recall_torch(seg_pred, mask)
        return (_cross_entropy_torch(seg_pred, mask),
                _smooth_l1_torch(vertex_pred, vertex, vertex_weights, 1.0, True), precision, recall)
    r = _native_losses(seg_pred, mask, vertex_pred, vertex, vertex_weights)
    return r["seg"], r["ver"], r["precision"], r["recall"]


def vertex_targets(mask, hcoords, use_motion=False):
    """The loader's ground-truth vertex field on the device: compute_vertex_hcoords
    (lib/datasets/linemod_dataset.py:68-81) for every image, as the loader collates it (`.permute(2,0,1)`).
    mask [b,h,w] (int64, int32, uint8 or bool; foreground is mask == 1), hcoords [b,K,3] float32 or float64 with rows
    (hx, hy, hw) -> float32 [b,2K,h,w].  Bit-identical to the reference's numpy for the hcoords passed in; the
    loader's keypoints are float64, so pass those (not their float32 rounding) where exact equality with the loader
    matters.  tools/demo.py's compute_vertex(mask, points_2d) is hcoords = [points_2d, 1]."""
    _check_keypoints(mask, hcoords)
    if not (mask.is_cuda and hcoords.is_cuda):
        raise RuntimeError("pvnet_b200: vertex_targets needs CUDA tensors (there is no CPU path)")
    if mask.device != hcoords.device:
        raise ValueError("mask and hcoords must be on the same device")
    dev = mask.device
    b, h, w = mask.shape
    K = hcoords.shape[1]
    mask, s_mask = _strides(mask, 3)
    hc = hcoords.detach().contiguous()
    out = torch.empty([b, 2 * K, h, w], dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _native.check(_native.lib().pvnet_vertex_targets(
            mask.data_ptr(), mask.element_size(), s_mask, hc.data_ptr(), int(hc.dtype == torch.float64), b, h, w, K,
            int(bool(use_motion)), out.data_ptr(), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
            "pvnet_vertex_targets")
    return out


def seg_vertex_losses_from_keypoints(seg_pred, vertex_pred, mask, hcoords, vertex_weights, use_motion=False):
    """seg_vertex_losses with the vertex targets built from the keypoints instead of read from a [b,2K,h,w] tensor:
    the same four float32 [b] figures, bit-identical to seg_vertex_losses(seg_pred, vertex_pred, mask,
    vertex_targets(mask, hcoords, use_motion), vertex_weights), in one launch pair that never materialises the field.
    hcoords [b,K,3] float32 or float64, with ver_dim == 2K.  In grad mode the field is materialised with
    vertex_targets and the torch expressions evaluated on it."""
    _check_seg(seg_pred, mask)
    for name, x in (("vertex_pred", vertex_pred), ("vertex_weights", vertex_weights)):
        _check_float(name, x)
    if vertex_pred.dim() != 4:
        raise ValueError(f"vertex_pred must be [b,ver_dim,h,w], got {tuple(vertex_pred.shape)}")
    b, vd, h, w = vertex_pred.shape
    if tuple(vertex_weights.shape) != (b, 1, h, w):
        raise ValueError(f"vertex_weights must be [b,1,h,w] = {(b, 1, h, w)}, got {tuple(vertex_weights.shape)}")
    if seg_pred.shape[0] != b or seg_pred.shape[2:] != vertex_pred.shape[2:]:
        raise ValueError(f"seg_pred {tuple(seg_pred.shape)} and vertex_pred {tuple(vertex_pred.shape)} differ in b,h,w")
    _check_keypoints(mask, hcoords)
    if vd != 2 * hcoords.shape[1]:
        raise ValueError(f"ver_dim {vd} is not 2 x the {hcoords.shape[1]} keypoints of hcoords")
    if _use_torch(seg_pred, vertex_pred, vertex_weights):
        vertex = vertex_targets(mask, hcoords, use_motion)
        precision, recall = _precision_recall_torch(seg_pred, mask)
        return (_cross_entropy_torch(seg_pred, mask),
                _smooth_l1_torch(vertex_pred, vertex, vertex_weights, 1.0, True), precision, recall)
    r = _native_losses(seg_pred, mask, vertex_pred, None, vertex_weights, hcoords=hcoords, use_motion=use_motion)
    return r["seg"], r["ver"], r["precision"], r["recall"]


class NetWrapper(nn.Module):
    """tools/train_linemod.py:79-91 (and tools/demo.py:31-43): forward(image, mask, vertex, vertex_weights) ->
    (seg_pred, vertex_pred, loss_seg, loss_vertex, precision, recall).  With no gradient to carry (eval under
    no_grad) the four figures come from one `seg_vertex_losses` call; in grad mode from the torch expressions."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, image, mask, vertex, vertex_weights):
        seg_pred, vertex_pred = self.net(image)
        loss_seg, loss_vertex, precision, recall = seg_vertex_losses(seg_pred, vertex_pred, mask, vertex,
                                                                     vertex_weights)
        return seg_pred, vertex_pred, loss_seg, loss_vertex, precision, recall


# ------------------------------------------------------------------------------------------ host-side helpers
class AverageMeter(dict):
    """Running average (val, avg, sum, count), readable as attributes or as dict items."""

    def __init__(self):
        super().__init__()
        self.reset()

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name) from None

    def __setattr__(self, name, value):
        self[name] = value

    def reset(self):
        self.val = 0
        self.avg = 0
        self.sum = 0
        self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


_CKPT = re.compile(r"^(\d+)\.pth$")


def load_model(model, optim, model_dir, epoch=-1):
    """Load `<model_dir>/<epoch>.pth` ({'net', 'optim', 'epoch'}; the latest epoch when epoch == -1) into model and
    optim.  Returns the epoch to continue from (stored epoch + 1), or 0 when there is no checkpoint."""
    if not os.path.isdir(model_dir):
        return 0
    epochs = [int(m.group(1)) for m in map(_CKPT.match, os.listdir(model_dir)) if m]
    if not epochs:
        return 0
    pick = max(epochs) if epoch == -1 else epoch
    ckpt = torch.load(os.path.join(model_dir, f"{pick}.pth"))
    model.load_state_dict(ckpt["net"])
    optim.load_state_dict(ckpt["optim"])
    print(f"load model {model_dir} epoch {ckpt['epoch']}")
    return ckpt["epoch"] + 1


def save_model(net, optim, epoch, model_dir):
    """Write {'net', 'optim', 'epoch'} to `<model_dir>/<epoch>.pth`, creating the directory."""
    os.makedirs(model_dir, exist_ok=True)
    torch.save({"net": net.state_dict(), "optim": optim.state_dict(), "epoch": epoch},
               os.path.join(model_dir, f"{epoch}.pth"))


def adjust_learning_rate(optimizer, epoch, lr_decay_rate, lr_decay_epoch, min_lr=1e-5):
    """Every lr_decay_epoch epochs (when (epoch + 1) is a multiple), multiply each group's lr by lr_decay_rate,
    not going below min_lr."""
    if (epoch + 1) % lr_decay_epoch != 0:
        return
    for group in optimizer.param_groups:
        before = group["lr"]
        group["lr"] = max(before * lr_decay_rate, min_lr)
    print(f"changing learning rate {before:5f} to {group['lr']:.5f}")


def set_learning_rate(optimizer, lr):
    """Set every parameter group's lr."""
    for group in optimizer.param_groups:
        before = group["lr"]
        group["lr"] = lr
    print(f"reset learning rate {before:5f} to {lr:.5f}")


def _optional(module, what):
    import importlib
    try:
        return importlib.import_module(module)
    except ImportError as e:
        raise ImportError(f"{what} needs the `{module}` package, which is not installed "
                          f"(Recorder(rec=False) logs to stdout and dump_fn without it)") from e


class Recorder(object):
    """Loss logging to stdout, an optional dump file and (rec=True) a tensorboardX SummaryWriter.  tensorboardX is
    imported when a recording Recorder is built; torchvision and matplotlib when an image is logged."""

    def __init__(self, rec=True, rec_dir=None, dump_fn=None):
        if rec:
            self.writer = _optional("tensorboardX", "Recorder(rec=True)").SummaryWriter(log_dir=rec_dir)
        else:
            self.writer = None
        self.dump_fn = dump_fn

    def _log(self, msg):
        print(msg)
        if self.dump_fn is not None:
            with open(self.dump_fn, "a") as f:
                f.write(msg + "\n")

    def rec_loss(self, loss, step, name='data/loss'):
        self._log(f"{name} {step} {loss}")
        if self.writer is not None:
            self.writer.add_scalar(name, loss, step)

    def rec_loss_batch(self, losses_batch, step, epoch, prefix='train'):
        msg = f"{prefix} epoch {epoch} step {step}"
        for k, v in losses_batch.items():
            msg += f" {k.split('/')[-1]} {v:.8f} "
        self._log(msg)
        if self.writer is not None:
            for k, v in losses_batch.items():
                self.writer.add_scalar(k, v, step)

    def rec_segmentation(self, seg, num_classes, nrow, step, name='seg'):
        """The argmax class map of seg [b,C,h,w] as an RGB image grid (one colour of matplotlib's tab20 per class)."""
        if self.writer is None:
            return
        vutils = _optional("torchvision.utils", "Recorder.rec_segmentation")
        cm = _optional("matplotlib.cm", "Recorder.rec_segmentation")
        palette = torch.tensor([cm.tab20(i % 20)[:3] for i in range(num_classes)], dtype=torch.float32) * 255
        labels = torch.argmax(seg, dim=1).long().cpu().clamp(0, num_classes - 1)
        rgb = palette[labels].permute(0, 3, 1, 2).to(torch.uint8)
        self.writer.add_image(name, vutils.make_grid(rgb, nrow), step)

    def rec_vertex(self, vertex, mask, nrow, step, name='vertex'):
        """The first vertex channel pair, masked and mapped from [-1,1] to [0,1], through the default colormap."""
        if self.writer is None:
            return
        vutils = _optional("torchvision.utils", "Recorder.rec_vertex")
        cm = _optional("matplotlib.cm", "Recorder.rec_vertex")
        v = (vertex[:, :2] * mask + 1) / 2
        h, w = v.shape[2:]
        rgb = cm.get_cmap()(v.reshape(-1, h, w).detach().cpu().numpy())[..., :3]
        self.writer.add_image(name, vutils.make_grid(torch.from_numpy(rgb).permute(0, 3, 1, 2), nrow), step)
