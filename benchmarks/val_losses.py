"""The validation losses of NetWrapper.forward on the device against the reference's torch expressions, one JSON line.

Batch 16, 480 x 640, K = 9 (ver_dim 18), 2 classes, int64 mask; seg_pred / vertex_pred are channel slices of one
[16,20,480,640] tensor, as Resnet18_8s.forward returns them.  For each form:
  - fused:    seg_vertex_losses, one launch pair for loss_seg, loss_vertex, precision and recall;
  - separate: the three native calls (cross-entropy alone, smooth_l1_loss, compute_precision_recall);
  - torch:    the reference's expressions (nn.CrossEntropyLoss(reduce=False) + mean, net_utils.py's smooth_l1_loss and
              compute_precision_recall), restated here;
device time per call (CUDA events around INNER back-to-back calls, warmed, median of REPS), the peak of the memory
allocated during one call, and for the fused call the compulsory bytes H*W*(4C + 8 ver_dim + 4 + 8) per image over
its time, against the H100 SXM's 3.35 TB/s.
    python benchmarks/val_losses.py > profiles/val_losses_<gpu>.json
"""
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvnet_b200 import net_utils as nu  # noqa: E402

B, H, W, K, C = 16, 480, 640, 9, 2
VD = 2 * K
REPS = int(os.environ.get("REPS", "30"))
INNER = int(os.environ.get("INNER", "10"))
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def torch_reference(seg, ver, mask, vertex, weights):
    """NetWrapper.forward's four figures with the reference's torch expressions."""
    loss_seg = nn.CrossEntropyLoss(reduction="none")(seg, mask)
    loss_seg = torch.mean(loss_seg.view(loss_seg.shape[0], -1), 1)
    b, vd = ver.shape[:2]
    s2 = 1.0
    diff = weights * (ver - vertex)
    ad = torch.abs(diff)
    sign = (ad < 1. / s2).detach().float()
    in_loss = torch.pow(diff, 2) * (s2 / 2.) * sign + (ad - (0.5 / s2)) * (1. - sign)
    loss_vertex = torch.sum(in_loss.view(b, -1), 1) / (vd * torch.sum(weights.view(b, -1), 1) + 1e-3)
    p = torch.argmax(seg, 1).float()
    t = mask.float()
    tp, fp, fn = (torch.sum(x.view(b, -1), 1) for x in (p * t, p * (1 - t), (1 - p) * t))
    return loss_seg, loss_vertex, (tp + 1) / (tp + fp + 1), (tp + 1) / (tp + fn + 1)


def separate(seg, ver, mask, vertex, weights):
    loss_seg = nu._native_losses(seg=seg, mask=mask, want=("seg",))["seg"]
    loss_vertex = nu.smooth_l1_loss(ver, vertex, weights)
    precision, recall = nu.compute_precision_recall(seg, mask)
    return loss_seg, loss_vertex, precision, recall


def device_ms(fn, args):
    for _ in range(5):
        fn(*args)
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(INNER):
            fn(*args)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / INNER)
    times.sort()
    return times[len(times) // 2]


def peak_mb(fn, args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn(*args)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    if not torch.cuda.is_available():
        raise SystemExit("val_losses.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    g = torch.Generator(device=dev).manual_seed(0)
    out = torch.randn(B, C + VD, H, W, device=dev, generator=g)
    seg, ver = out[:, :C], out[:, C:]
    mask = torch.randint(0, 2, (B, H, W), device=dev, generator=g)
    vertex = torch.randn(B, VD, H, W, device=dev, generator=g)
    weights = (mask > 0).float()[:, None]
    args = (seg, ver, mask, vertex, weights)
    name, power, clock = gpu_info()
    rows = {}
    with torch.no_grad():
        fused = nu.seg_vertex_losses(*args)
        ref = torch_reference(*args)
        max_rel = max(float(((a - b).abs() / b.abs()).max()) for a, b in zip(fused, ref))
        for key, fn in (("fused", nu.seg_vertex_losses), ("separate", separate), ("torch", torch_reference)):
            rows[key] = {"ms": device_ms(fn, args), "peak_mb": peak_mb(fn, args)}
    compulsory = B * H * W * (4 * C + 4 * VD * 2 + 4 + mask.element_size())
    gbps = compulsory / (rows["fused"]["ms"] * 1e-3) / 1e9
    print(json.dumps({
        "bench": "val_losses", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
        "batch": B, "h": H, "w": W, "ver_dim": VD, "classes": C, "mask_dtype": str(mask.dtype), "reps": REPS,
        "inner": INNER, "compulsory_bytes": compulsory, "fused_gb_per_s": gbps,
        "fused_fraction_of_hbm_3_35_tb_s": gbps * 1e9 / HBM_BYTES_PER_S,
        "speedup_fused_vs_torch": rows["torch"]["ms"] / rows["fused"]["ms"],
        "speedup_fused_vs_separate": rows["separate"]["ms"] / rows["fused"]["ms"],
        "max_rel_diff_fused_vs_torch": max_rel, "rows": rows}))


if __name__ == "__main__":
    main()
