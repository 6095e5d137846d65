"""Train-mode BatchNorm on the native kernels against torch's modules; one JSON line.

Part one, per BatchNorm site of Resnet18_8s.forward_train at batch B (default 32), 480 x 640: the native forward
(pvnet_batchnorm_act_forward: statistics, finalise, apply) and backward (pvnet_batchnorm_act_backward: reduce,
coefficients, elementwise) against torch's channels_last BatchNorm2d + ReLU / LeakyReLU(0.1) modules (+ the residual
add and ReLU of a block tail, + the downsample's BatchNorm), forward and autograd backward (torch.autograd.grad of the
same inputs and parameters).  CUDA events, WARM warm-up calls, REPS timed calls with the native and torch forms
alternated, the median.  Bytes: the passes each native call makes over [N, C] fp32 tensors (forward: statistics read
x (and z), apply reads x (and z) and writes y; backward: the reduce reads dy, x (and z), the elementwise pass reads
them again and writes dx (and dz)), as GB/s and as a share of 3.35 TB/s (H100 SXM data sheet).

Part two, a forward_train step (seg_vertex_training_losses_from_keypoints, backward(), Adam) at batch 16 and 32:
native against the same network with torch's modules swapped back in for pc.bn_act / pc.bn_add_relu, alternated
step by step in one run; median step time and the peak memory allocated during a step.
    python benchmarks/bn_train.py > profiles/bn_train_<gpu>_<power>.json
"""
import copy
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from pvnet_b200 import conv as pc  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402
from train_step import gpu_info, inputs, peak_mb  # noqa: E402

H, W, K = 480, 640, 9
B = int(os.environ.get("B", "32"))
BATCHES = tuple(int(b) for b in os.environ.get("BATCHES", "16,32").split(","))
REPS = int(os.environ.get("REPS", "20"))
WARM = int(os.environ.get("WARM", "3"))
STEPS = int(os.environ.get("STEPS", "10"))
HBM = 3.35e12
R, L = pc.ACT_RELU, pc.ACT_LEAKY

# (sites, form, act, C, downsampling of the 480 x 640 image)
SITES = [("bn1", 0, R, 64, 2), ("layer1.*.bn1", 0, R, 64, 4), ("layer1.*.bn2+add", 1, R, 64, 4),
         ("layer2.0.bn1", 0, R, 128, 8), ("layer2.0.bn2+downsample.1+add", 2, R, 128, 8), ("layer2.1.bn1", 0, R, 128, 8),
         ("layer2.1.bn2+add", 1, R, 128, 8), ("layer3.0.bn1", 0, R, 256, 8),
         ("layer3.0.bn2+downsample.1+add", 2, R, 256, 8), ("layer3.1.bn1", 0, R, 256, 8),
         ("layer3.1.bn2+add", 1, R, 256, 8), ("layer4.0.bn1", 0, R, 512, 8),
         ("layer4.0.bn2+downsample.1+add", 2, R, 512, 8), ("layer4.1.bn1", 0, R, 512, 8),
         ("layer4.1.bn2+add", 1, R, 512, 8), ("fc.1", 0, R, 256, 8), ("conv8s.1", 0, L, 128, 8),
         ("conv4s.1", 0, L, 64, 4), ("conv2s.1", 0, L, 32, 2), ("convraw.1", 0, L, 32, 1)]
# sites that occur twice in the network (layer1's two blocks)
COUNT = {"layer1.*.bn1": 2, "layer1.*.bn2+add": 2}
PASSES = {0: (3, 5), 1: (4, 8), 2: (5, 8)}          # (forward, backward) passes over one [N, C] fp32 tensor


def _act(act, t):
    return F.relu(t, inplace=True) if act == R else F.leaky_relu(t, 0.1, inplace=True)


def torch_bn_act(bn, x, act=pc.ACT_NONE):
    y = bn(x)
    return y if act == pc.ACT_NONE else _act(act, y)


def torch_bn_add_relu(bn, a, skip, bn_skip=None):
    return F.relu(bn(a) + (skip if bn_skip is None else bn_skip(skip)), inplace=True)


def timed(fns, reps):
    """Median ms of each fn, the fns alternated call by call."""
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            e.record()
            e.synchronize()
            ts[k].append(a.elapsed_time(e))
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()}


def site_row(name, form, act, C, down, dev):
    b, h, w = B, H // down, W // down
    g = torch.Generator(device=dev).manual_seed(C + down)
    cl = torch.channels_last
    mk = lambda: torch.randn(b, C, h, w, device=dev, generator=g).contiguous(memory_format=cl)  # noqa: E731
    x, dy = mk(), mk()
    z = mk() if form else None
    bn = torch.nn.BatchNorm2d(C).to(dev).train()
    bz = torch.nn.BatchNorm2d(C).to(dev).train() if form == 2 else None
    tb, tz = copy.deepcopy(bn), copy.deepcopy(bz)
    xh, zh, dyh = pc._nhwc(x), None if z is None else pc._nhwc(z), pc._nhwc(dy)
    state = {}

    def nat_fwd():
        st, sz = pc.BatchNormState(bn, dev), pc.BatchNormState(bz, dev) if form == 2 else None
        state["y"] = pc.batchnorm_forward(form, act, xh, zh, st, bn.weight, bn.bias, sz,
                                          None if bz is None else bz.weight, None if bz is None else bz.bias)
        state["st"], state["sz"] = st, sz

    def nat_bwd():
        pc.batchnorm_backward(form, act, dyh, xh, zh, state["st"], bn.weight, state["sz"],
                              None if bz is None else bz.weight)

    xt = x.detach().requires_grad_()
    zt = None if z is None else z.detach().requires_grad_()
    params = [xt, tb.weight, tb.bias] + ([zt] if form else []) + ([tz.weight, tz.bias] if form == 2 else [])

    def torch_fwd():
        state["yt"] = torch_bn_act(tb, xt, act) if form == 0 else torch_bn_add_relu(tb, xt, zt, tz)

    def torch_bwd():
        torch.autograd.grad(state["yt"], params, dy, retain_graph=True)

    nat_fwd()
    torch_fwd()
    for _ in range(WARM):
        nat_fwd(), nat_bwd(), torch_fwd(), torch_bwd()
    t = timed({"native_fwd": nat_fwd, "torch_fwd": torch_fwd}, REPS)
    t.update(timed({"native_bwd": nat_bwd, "torch_bwd": torch_bwd}, REPS))
    tensor_bytes = 4.0 * b * h * w * C
    pf, pb = PASSES[form]
    row = {"site": name, "count": COUNT.get(name, 1), "form": form, "act": act, "C": C, "hw": [h, w],
           "tensor_mb": tensor_bytes / 2 ** 20, "fwd_bytes": pf * tensor_bytes, "bwd_bytes": pb * tensor_bytes}
    for k, ms in t.items():
        row[k + "_ms"] = ms
    for part in ("fwd", "bwd"):
        gbps = row[f"{part}_bytes"] / (row[f"native_{part}_ms"] * 1e-3)
        row[f"native_{part}_GBps"] = gbps / 1e9
        row[f"native_{part}_fraction_of_hbm_peak"] = gbps / HBM
    return row


def step_rows(b, dev):
    x, mask, hc, wgt = inputs(b, dev, seed=1)
    torch.manual_seed(0)
    base = Resnet18_8s(ver_dim=2 * K, seg_dim=2).to(dev).train()
    nets = {"native": base, "torch_modules": copy.deepcopy(base)}
    opts = {k: torch.optim.Adam(m.parameters(), lr=1e-3) for k, m in nets.items()}
    orig = pc.bn_act, pc.bn_add_relu

    def make(k):
        def step():
            if k == "torch_modules":
                pc.bn_act, pc.bn_add_relu = torch_bn_act, torch_bn_add_relu
            try:
                seg, ver = nets[k].forward_train(x)
            finally:
                pc.bn_act, pc.bn_add_relu = orig
            ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
            opts[k].zero_grad(set_to_none=True)
            (torch.mean(ls) + torch.mean(lv)).backward()
            opts[k].step()
        return step
    steps = {k: make(k) for k in nets}
    for _ in range(WARM):
        for fn in steps.values():
            fn()
    t = timed(steps, STEPS)
    return {k: {"step_ms": t[k], "step_peak_mb": peak_mb(fn)} for k, fn in steps.items()}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("bn_train.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    name, power, clock = gpu_info()
    sites = []
    for s in SITES:
        sites.append(site_row(*s, dev))
        torch.cuda.empty_cache()
    tot = {k: sum(r[k] * r["count"] for r in sites) for k in ("native_fwd_ms", "native_bwd_ms", "torch_fwd_ms",
                                                               "torch_bwd_ms")}
    steps = {}
    for b in BATCHES:
        steps[str(b)] = step_rows(b, dev)
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "bn_train", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock, "h": H, "w": W,
                      "sites_batch": B, "reps": REPS, "warm": WARM, "steps": STEPS, "hbm_peak_Bps": HBM,
                      "sites": sites, "site_totals_ms": tot, "forward_train_step": steps}))


if __name__ == "__main__":
    main()
