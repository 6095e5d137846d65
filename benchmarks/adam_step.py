"""The optimizer step of a Resnet18_8s training iteration; one JSON line.

1. The step alone, on Resnet18_8s's 77 parameter tensors (ver_dim 18, seg_dim 2) with resident random gradients, four
   forms on their own copies of the parameters: `native` (pvnet_b200.optim.Adam: pvnet_adam_step, one launch),
   `torch_foreach` (torch.optim.Adam's default on CUDA), `torch_single` (foreach=False, the sequence the native kernel
   states) and `torch_fused` (fused=True, torch's own multi-tensor kernel: the honest baseline).  Every form is warmed,
   then the forms alternate inside the timed loop, REPS repetitions, each timed by CUDA events around `step()`; the
   median is reported with min and max.  With an idle device those events span the host's enqueue as well: where
   `enqueue_ms` (the host's wall clock for `step()` without a synchronise: time to enqueue, not to compute) is close
   to `ms`, the form is host-bound in this loop, and `kernel_ms` says what the device itself executes: the summed
   device time of the step's kernels under torch.profiler in a separate run, with `device_ops`, their number per
   step (for the native form also read from the library's launch counter).  `gb_per_s` and `kernel_gb_per_s` are
   the compulsory bytes (read p, g, m, v and write p, m, v: 7 x 4 B x parameters) over `ms` and `kernel_ms`, the
   `share_of_hbm_peak` figures those rates over the H100 SXM data sheet's 3.35 TB/s: the step is bandwidth-bound and
   its 0.36 GB are several times the 50 MB L2.
2. A full training step (forward_train, seg_vertex_training_losses_from_keypoints, backward(), optimizer) at
   16 x 480 x 640, 32 x 480 x 640 and 32 x 256 x 320 with the native optimizer and torch's default alternated step by
   step, median of STEPS, with torch.use_deterministic_algorithms off and on, and the peak memory of one step.
    python benchmarks/adam_step.py > profiles/adam_step_<gpu>_<power>.json
"""
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from pvnet_b200 import _native, optim  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402
from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402
from train_step import gpu_info, peak_mb  # noqa: E402

K = 9
REPS = int(os.environ.get("REPS", "200"))
STEPS = int(os.environ.get("STEPS", "10"))
WARM = int(os.environ.get("WARM", "3"))
CONFIGS = [tuple(int(v) for v in c.split("x")) for c in
           os.environ.get("CONFIGS", "16x480x640,32x480x640,32x256x320").split(",")]
HBM_PEAK = 3.35e12
FORMS = {
    "native": lambda ps: optim.Adam(ps, lr=1e-3),
    "torch_foreach": lambda ps: torch.optim.Adam(ps, lr=1e-3),
    "torch_single": lambda ps: torch.optim.Adam(ps, lr=1e-3, foreach=False),
    "torch_fused": lambda ps: torch.optim.Adam(ps, lr=1e-3, fused=True),
}


def stats(ts):
    return {"ms": float(np.median(ts)), "ms_min": float(min(ts)), "ms_max": float(max(ts))}


PROFILED_STEPS = 5


def device_ops(fn):
    """(kernels and memory operations per step, their summed device time per step in ms) over PROFILED_STEPS steps
    under torch.profiler: what the device executes, without the host's enqueue time between launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(PROFILED_STEPS):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA]
    return (sum(e.count for e in ev) / PROFILED_STEPS,
            sum(e.self_device_time_total for e in ev) / 1e3 / PROFILED_STEPS)


def optimizer_alone(dev):
    torch.manual_seed(0)
    shapes = [p.shape for p in Resnet18_8s(ver_dim=2 * K, seg_dim=2).parameters()]
    numel = sum(s.numel() for s in shapes)
    g = torch.Generator(device=dev).manual_seed(0)
    opts = {}
    for name, make in FORMS.items():
        ps = [torch.nn.Parameter(torch.randn(s, device=dev, generator=g) * 0.1) for s in shapes]
        for p in ps:
            p.grad = torch.randn(p.shape, device=dev, generator=g) * 0.01
        opts[name] = make(ps)
    for _ in range(WARM):
        for opt in opts.values():
            opt.step()
    torch.cuda.synchronize()
    dev_ms = {k: [] for k in opts}
    host_ms = {k: [] for k in opts}
    for _ in range(REPS):
        for name, opt in opts.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            opt.step()
            e.record()
            e.synchronize()
            dev_ms[name].append(a.elapsed_time(e))
    for _ in range(REPS):
        for name, opt in opts.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            opt.step()
            host_ms[name].append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    bytes_ = 7 * 4 * numel
    rows = {}
    for name, opt in opts.items():
        row = stats(dev_ms[name])
        row["gb_per_s"] = bytes_ / (row["ms"] * 1e-3) / 1e9
        row["share_of_hbm_peak"] = bytes_ / (row["ms"] * 1e-3) / HBM_PEAK
        row["enqueue_ms"] = float(np.median(host_ms[name]))
        row["device_ops"], row["kernel_ms"] = device_ops(opt.step)
        row["kernel_gb_per_s"] = bytes_ / (row["kernel_ms"] * 1e-3) / 1e9
        row["kernel_share_of_hbm_peak"] = bytes_ / (row["kernel_ms"] * 1e-3) / HBM_PEAK
        rows[name] = row
    _native.launch_count_reset()
    opts["native"].step()
    rows["native"]["launches"] = _native.launch_count()
    return {"tensors": len(shapes), "parameters": numel, "compulsory_bytes": bytes_, "reps": REPS, "forms": rows}


def batch(b, H, W, dev, seed):
    rng = np.random.default_rng(seed)
    nfg = max(H * W // 15, 64)
    masks = [syn.disc_mask(nfg, center=(W // 2 + int(rng.integers(-W // 16, W // 16 + 1)),
                                        H // 2 + int(rng.integers(-H // 16, H // 16 + 1))), h=H, w=W)
             for _ in range(b)]
    hc = np.concatenate([rng.uniform([0, 0], [W, H], (b, K, 2)), np.ones((b, K, 1))], 2)
    x = torch.randn(b, 3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
    return x, torch.from_numpy(np.stack(masks)).to(dev), torch.from_numpy(hc).to(dev)


def full_step(b, H, W, dev):
    torch.manual_seed(0)
    base = Resnet18_8s(ver_dim=2 * K, seg_dim=2).to(dev).train()
    x, mask, hc = batch(b, H, W, dev, seed=b + H)
    steps = {}
    for name in ("native", "torch_foreach"):
        net = copy.deepcopy(base)
        opt = FORMS[name](net.parameters())

        def step(net=net, opt=opt):
            seg, ver = net.forward_train(x)
            ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
            opt.zero_grad(set_to_none=True)
            (ls.mean() + lv.mean()).backward()
            opt.step()
        steps[name] = step
    row = {"b": b, "H": H, "W": W}
    for det in (False, True):
        torch.use_deterministic_algorithms(det)
        try:
            for _ in range(WARM):
                for fn in steps.values():
                    fn()
            ts = {k: [] for k in steps}
            for _ in range(STEPS):
                for name, fn in steps.items():
                    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    fn()
                    e.record()
                    e.synchronize()
                    ts[name].append(a.elapsed_time(e))
            row["deterministic" if det else "default"] = {
                name: {**{"step_" + k: v for k, v in stats(ts[name]).items()}, "step_peak_mb": peak_mb(fn)}
                for name, fn in steps.items()}
        finally:
            torch.use_deterministic_algorithms(False)
    return row


def main():
    if not torch.cuda.is_available():
        raise SystemExit("adam_step.py measures on a GPU; none is available (no GPU, no fallback)")
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    alone = optimizer_alone(dev)
    rows = []
    for b, H, W in CONFIGS:
        rows.append(full_step(b, H, W, dev))
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "adam_step", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
                      "hbm_peak_bytes_per_s": HBM_PEAK, "optimizer_alone": alone, "steps": STEPS, "warmup": WARM,
                      "full_step": rows}))


if __name__ == "__main__":
    main()
