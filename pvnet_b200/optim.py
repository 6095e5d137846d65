"""`torch.optim.Adam` as the reference trains with it (tools/train_linemod.py:260), stepped by one multi-tensor launch.

`Adam(net.parameters(), lr=...)` is a drop-in for `torch.optim.Adam(net.parameters(), lr=...)`: the same `state`
(`step` a float32 CPU scalar, `exp_avg`, `exp_avg_sq`), the same `param_groups` keys the training loop touches (`lr`,
`betas`, `eps`, `weight_decay`), and a `state_dict()` that loads into torch's Adam and back, so a checkpoint written by
`net_utils.save_model` with either resumes with the other.  `step()` hands every parameter of a group that has a
gradient to `pvnet_adam_step` (pvnet_b200/csrc/optim.cu): one pass over `p, g, m, v` in the floating-point sequence of
torch's `foreach=False` Adam, stated in DESIGN.md §19.

There is no fallback: a CPU parameter is an error, and so is anything the kernel does not compute (AMSGrad, maximize,
decoupled weight decay, sparse gradients, dtypes other than float32).
"""
from __future__ import annotations

import ctypes

import torch

from . import _native

_UNSUPPORTED = ("amsgrad", "maximize", "foreach", "capturable", "differentiable", "fused", "decoupled_weight_decay")
# options a loaded torch.optim.Adam state_dict may carry that change what a step computes or where `step` lives;
# `foreach` only chooses among torch's own implementations and is ignored
_REFUSED_WHEN_SET = ("amsgrad", "maximize", "capturable", "differentiable", "fused", "decoupled_weight_decay")


def _dense(t):
    """Non-overlapping and dense: some permutation of the dimensions is contiguous."""
    if t.is_contiguous():
        return True
    expect = 1
    for stride, size in sorted((st, sz) for sz, st in zip(t.shape, t.stride()) if sz != 1):
        if stride != expect:
            return False
        expect *= size
    return True


def _like(p, t):
    """t is a float32 tensor on p's device with p's shape and, over the dimensions longer than 1, p's strides."""
    if t.dtype != torch.float32 or t.device != p.device or t.shape != p.shape:
        return False
    return t.stride() == p.stride() or all(a == b for a, b, n in zip(p.stride(), t.stride(), p.shape) if n != 1)


class Adam(torch.optim.Optimizer):
    """Adam with torch.optim.Adam's defaults, state and checkpoint format; CUDA float32 parameters only."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, **unsupported):
        if unsupported:
            names = ", ".join(sorted(unsupported))
            raise ValueError(f"pvnet_b200.optim.Adam takes lr, betas, eps and weight_decay only (got {names}): "
                             f"it computes torch.optim.Adam's default step and has no {' / '.join(_UNSUPPORTED)} option")
        for name, value in (("lr", lr), ("eps", eps), ("weight_decay", weight_decay)):
            if isinstance(value, torch.Tensor):
                raise ValueError(f"{name} must be a Python number, not a tensor")
        _check_hyper(lr, betas, eps, weight_decay)
        super().__init__(params, {"lr": lr, "betas": tuple(betas), "eps": eps, "weight_decay": weight_decay})
        self._checked_state = {}                      # parameter -> the (exp_avg, exp_avg_sq, step) already checked

    def __setstate__(self, state):
        super().__setstate__(state)                   # unpickling and load_state_dict both come through here
        self._checked_state = {}

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        # every check first: nothing is launched and no step count advances when something is refused
        plans = [(group, self._plan(group)) for group in self.param_groups]
        for group, entries in plans:
            if not entries:
                continue
            # a CPU tensor addend: the scalar 1 would be wrapped into a tensor once per step tensor
            torch._foreach_add_([state["step"] for _, _, state in entries], torch.tensor(1.0), alpha=1.0)
            calls = {}                                # (device, step reached) -> [(p, g, m, v)]
            for p, g, state in entries:
                calls.setdefault((p.device, int(state["step"].item())), []).append((p, g, state["exp_avg"],
                                                                                     state["exp_avg_sq"]))
            beta1, beta2 = group["betas"]
            for (dev, step), tensors in calls.items():
                _adam_step(dev, tensors, float(group["lr"]), float(beta1), float(beta2), float(group["eps"]),
                           float(group["weight_decay"]), step)
        return loss

    def _plan(self, group):
        """The (parameter, gradient, state) triples of one group's step, state created lazily as torch creates it."""
        for name in _REFUSED_WHEN_SET:
            if group.get(name):
                raise ValueError(f"pvnet_b200.optim.Adam: this parameter group has {name}={group[name]!r} (loaded from "
                                 f"a torch.optim.Adam that used it); only torch's default Adam step is computed")
        _check_hyper(group["lr"], group["betas"], group["eps"], group["weight_decay"])
        entries = []
        for p in group["params"]:
            g = p.grad
            if g is None:
                continue
            if g.is_sparse:
                raise ValueError("pvnet_b200.optim.Adam does not support sparse gradients")
            if p.dtype != torch.float32 or g.dtype != torch.float32:
                raise ValueError(f"pvnet_b200.optim.Adam steps float32 parameters only, got {p.dtype} with a "
                                 f"{g.dtype} gradient")
            _check_device(p)
            if not _dense(p):
                raise ValueError(f"pvnet_b200.optim.Adam: a parameter of shape {tuple(p.shape)} and strides "
                                 f"{p.stride()} is not dense in memory")
            state = self.state[p]
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            # the state tensors are checked once, and again only when they have been replaced (load_state_dict)
            m, v = state["exp_avg"], state["exp_avg_sq"]
            seen = self._checked_state.get(p)
            fresh = seen is None or seen[0] is not m or seen[1] is not v or seen[2] is not state["step"]
            for name, t in (("gradient", g),) + ((("exp_avg", m), ("exp_avg_sq", v)) if fresh else ()):
                if not _like(p, t):
                    raise ValueError(
                        f"pvnet_b200.optim.Adam: the {name} of a parameter of shape {tuple(p.shape)} must be a float32 "
                        f"tensor on {p.device} with the parameter's strides {p.stride()}; got {t.dtype} on {t.device}, "
                        f"shape {tuple(t.shape)}, strides {t.stride()}")
            if fresh:
                if state["step"].is_cuda:
                    raise ValueError("pvnet_b200.optim.Adam keeps `step` on the host, as torch's default Adam does; "
                                     "this state came from a capturable or fused optimizer")
                self._checked_state[p] = (m, v, state["step"])
            entries.append((p, g, state))
        return entries


def _check_device(p):
    if not p.is_cuda:
        raise RuntimeError("pvnet_b200: optim.Adam runs only on CUDA (no CPU fallback)")


def _adam_step(dev, tensors, lr, beta1, beta2, eps, weight_decay, step):
    """pvnet_adam_step over [(p, g, m, v)] on dev's current stream; `step` is the count these tensors reach."""
    table = (_native.AdamTensor * len(tensors))(
        *(_native.AdamTensor(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel())
          for p, g, m, v in tensors))
    with torch.cuda.device(dev):
        _native.check(_native.lib().pvnet_adam_step(
            table, len(tensors), lr, beta1, beta2, eps, weight_decay, step,
            ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)), "pvnet_adam_step")


def _check_hyper(lr, betas, eps, weight_decay):
    if not 0.0 <= lr < float("inf"):
        raise ValueError(f"Invalid learning rate: {lr}")
    if not 0.0 <= eps < float("inf"):
        raise ValueError(f"Invalid epsilon value: {eps}")
    if not 0.0 <= betas[0] < 1.0:
        raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
    if not 0.0 <= betas[1] < 1.0:
        raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
    if not 0.0 <= weight_decay < float("inf"):
        raise ValueError(f"Invalid weight_decay value: {weight_decay}")
