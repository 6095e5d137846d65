"""The training losses forward + backward: the torch expressions against the device backward, one JSON line.

Batch 16 and 32, 480 x 640, K = 9 (ver_dim 18), C = 2, int64 disc masks of 20 000 foreground pixels, 0/1 weights,
float64 keypoints; seg_pred and vertex_pred are the channel slices of one [b,20,480,640] tensor that requires grad.
For each form, the device time of forward + torch.autograd.grad(mean(loss_seg) + mean(loss_vertex), output) (CUDA
events around INNER back-to-back steps, warmed, median of REPS) and the peak of the memory allocated during one step
above what was allocated before it:
  (1) seg_vertex_losses in grad mode: the reference's torch expressions;
  (2) seg_vertex_training_losses on a materialised field;
  (3) seg_vertex_training_losses_from_keypoints.
Also the backward call alone for (2) and (3) (the four launches of pvnet_seg_vertex_losses[_keypoints]_backward),
with the compulsory bytes H*W*(4C + 4vd [+ 4vd field] + 4 + 8 + 4(C+vd)) over its time against 3.35 TB/s.
Then one training step at batch 16: train-mode Resnet18_8s (the PyTorch graph) + the losses + backward() + an SGD
step, with the torch losses and the native ones alternated step by step in the same run, median of STEPS each.
    python benchmarks/train_losses.py > profiles/train_losses_<gpu>_<power>.json
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402

H, W, K, C, NFG = 480, 640, 9, 2, 20000
VD = 2 * K
BATCHES = (16, 32)
STEP_BATCH = 16
REPS = int(os.environ.get("REPS", "20"))
INNER = int(os.environ.get("INNER", "5"))
STEPS = int(os.environ.get("STEPS", "10"))
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def device_ms(fn, warm=3):
    for _ in range(warm):
        fn()
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(INNER):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / INNER)
    times.sort()
    return times[len(times) // 2]


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def inputs(b, dev, seed=0):
    rng = np.random.default_rng(seed)
    masks = [syn.disc_mask(NFG, center=(320 + int(rng.integers(-40, 41)), 240 + int(rng.integers(-40, 41))))
             for _ in range(b)]
    hc = np.concatenate([rng.uniform([0, 0], [W, H], (b, K, 2)), np.ones((b, K, 1))], 2)
    mask = torch.from_numpy(np.stack(masks)).to(dev)
    hcoords = torch.from_numpy(hc).to(dev)
    field = nu.vertex_targets(mask, hcoords)
    weights = mask[:, None].float()
    return mask, hcoords, field, weights


def loss_forms(mask, hcoords, field, weights):
    return {
        "torch_expressions": lambda s, v: nu.seg_vertex_losses(s, v, mask, field, weights),
        "native_field": lambda s, v: nu.seg_vertex_training_losses(s, v, mask, field, weights),
        "native_keypoints": lambda s, v: nu.seg_vertex_training_losses_from_keypoints(s, v, mask, hcoords, weights),
    }


def losses_rows(b, dev):
    mask, hcoords, field, weights = inputs(b, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    out = torch.randn(b, C + VD, H, W, device=dev, generator=g).requires_grad_()
    rows, grads = {}, {}
    for name, fn in loss_forms(mask, hcoords, field, weights).items():
        def step(fn=fn):
            ls, lv, _, _ = fn(out[:, :C], out[:, C:])
            return torch.autograd.grad(torch.mean(ls) + torch.mean(lv), out)[0]
        grads[name] = step()
        rows[name] = {"fwd_bwd_ms": device_ms(step), "peak_mb": peak_mb(step)}
    ref = grads["torch_expressions"]
    for name in ("native_field", "native_keypoints"):
        d = grads[name] - ref
        rows[name]["max_abs_diff_vs_torch"] = float(d.abs().max())
        rows[name]["grad_bit_identical_to_torch"] = bool(torch.equal(grads[name], ref))
    # the backward call alone: pvnet_seg_vertex_losses[_keypoints]_backward into a preallocated output gradient
    gout = torch.empty_like(out)
    ones = torch.full([b], 1.0 / b, device=dev)
    seg, ver = out.detach()[:, :C], out.detach()[:, C:]
    for name, tgt, hc in (("native_field", field, None), ("native_keypoints", None, hcoords)):
        def bwd(tgt=tgt, hc=hc):
            nu._native_losses_backward(seg, mask, ver, tgt, weights, hc, False, ones, ones, gout[:, :C], gout[:, C:])
        ms = device_ms(bwd)
        nbytes = b * H * W * (4 * C + 4 * VD + (4 * VD if tgt is not None else 0) + 4 + 8 + 4 * (C + VD))
        rows[name].update({"backward_call_ms": ms, "backward_compulsory_bytes": nbytes,
                           "backward_tb_per_s": nbytes / (ms * 1e-3) / 1e12,
                           "backward_fraction_of_hbm_3_35_tb_s": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S,
                           "backward_lower_bound_ms": nbytes / HBM_BYTES_PER_S * 1e3})
    return rows


def train_step_rows(dev):
    from pvnet_b200.model_repository import Resnet18_8s
    torch.manual_seed(0)
    net = Resnet18_8s(ver_dim=VD, seg_dim=C).to(dev).train()
    opt = torch.optim.SGD(net.parameters(), lr=1e-5, momentum=0.9)
    mask, hcoords, field, weights = inputs(STEP_BATCH, dev, seed=1)
    x = torch.randn(STEP_BATCH, 3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    forms = loss_forms(mask, hcoords, field, weights)

    def step(fn):
        seg, ver = net(x)
        ls, lv, _, _ = fn(seg, ver)
        loss = torch.mean(ls) + torch.mean(lv)
        opt.zero_grad()
        loss.backward()
        opt.step()

    times = {k: [] for k in forms}
    for _ in range(2):
        for fn in forms.values():
            step(fn)
    for _ in range(STEPS):
        for name, fn in forms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(fn)
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b))
    res = {}
    for name, fn in forms.items():
        t = sorted(times[name])
        res[name] = {"step_ms": t[len(t) // 2], "step_peak_mb": peak_mb(lambda fn=fn: step(fn))}
    return res


def main():
    if not torch.cuda.is_available():
        raise SystemExit("train_losses.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    name, power, clock = gpu_info()
    rows = {str(b): losses_rows(b, dev) for b in BATCHES}
    step = train_step_rows(dev)
    print(json.dumps({
        "bench": "train_losses", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
        "h": H, "w": W, "keypoints": K, "classes": C, "foreground_pixels": NFG, "mask_dtype": "torch.int64",
        "reps": REPS, "inner": INNER, "steps": STEPS, "losses": rows,
        "train_step_batch": STEP_BATCH, "train_step": step}))


if __name__ == "__main__":
    main()
