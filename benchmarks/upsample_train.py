"""The decoder's bilinear x2 upsampling in training, native against torch; one JSON line.

Per stage of forward_train's decoder (conv8s -> 1/4: C = 128 at 60 x 80 into a 192-channel concat buffer; conv4s ->
1/2: 64 at 120 x 160 into 128; conv2s -> full resolution: 32 at 240 x 320 into 40), at batch 16 and 32:
  forward   pvnet_upsample2x_nhwc into the concat buffer's first C channels, against torch's
            F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) on the channels_last input;
  backward  pvnet_upsample2x_backward_nhwc reading the buffer gradient's first C channels in place, against
            aten.upsample_bilinear2d_backward on the same channel slice (what CatBackward hands the graph's
            UpsampleBilinear2DBackward; its output zero-fill and atomics included).
CUDA events around ITERS launches, the two forms alternated REPS times, median; achieved GB/s of the compulsory bytes
(read the input once, write the output once) and its share of 3.35 TB/s (H100 SXM HBM3 data sheet).

Then one Resnet18_8s.forward_train step (forward, seg_vertex_training_losses_from_keypoints, backward(), Adam) at
480 x 640, K = 9, with torch.use_deterministic_algorithms off and on, alternated step by step, median of STEPS steps.
    python benchmarks/upsample_train.py > profiles/upsample_train_<gpu>_<power>.json
"""
import copy
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvnet_b200 import _native  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402

STAGES = (("up8sto4s", 128, 60, 80, 192), ("up4sto2s", 64, 120, 160, 128), ("up2storaw", 32, 240, 320, 40))
BATCHES = tuple(int(b) for b in os.environ.get("BATCHES", "16,32").split(","))
ITERS = int(os.environ.get("ITERS", "20"))
REPS = int(os.environ.get("REPS", "7"))
STEPS = int(os.environ.get("STEPS", "8"))
HBM = 3.35e12
H, W, K = 480, 640, 9


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def timed(fn, iters=ITERS):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def stage_rows(b):
    L = _native.lib()
    rows = []
    for name, C, h, w, cs in STAGES:
        g = torch.Generator(device="cuda").manual_seed(C)
        low = torch.randn(b, C, h, w, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        buf = torch.empty(b, cs, 2 * h, 2 * w, device="cuda").contiguous(memory_format=torch.channels_last)
        gbuf = torch.randn(b, cs, 2 * h, 2 * w, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        dlow = torch.empty(b, h, w, C, device="cuda")
        s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def nat_fwd():
            _native.check(L.pvnet_upsample2x_nhwc(ctypes.c_void_p(low.data_ptr()), C, ctypes.c_void_p(buf.data_ptr()),
                                                  cs, 0, b, h, w, s), "pvnet_upsample2x_nhwc")

        def nat_bwd():
            _native.check(L.pvnet_upsample2x_backward_nhwc(ctypes.c_void_p(gbuf.data_ptr()), cs, 0, C,
                                                           ctypes.c_void_p(dlow.data_ptr()), b, h, w, s),
                          "pvnet_upsample2x_backward_nhwc")

        gslice = gbuf[:, :C]

        def t_fwd():
            F.interpolate(low, scale_factor=2, mode="bilinear", align_corners=True)

        def t_bwd():
            torch.ops.aten.upsample_bilinear2d_backward(gslice, [2 * h, 2 * w], [b, C, h, w], True, None, None)

        forms = {"native_fwd": nat_fwd, "torch_fwd": t_fwd, "native_bwd": nat_bwd, "torch_bwd": t_bwd}
        for fn in forms.values():
            timed(fn, 3)
        ms = {k: [] for k in forms}
        for _ in range(REPS):
            for k, fn in forms.items():
                ms[k].append(timed(fn))
        small, big = b * h * w * C * 4, b * 4 * h * w * C * 4
        row = {"stage": name, "batch": b, "C": C, "h": h, "w": w, "concat_channels": cs, "bytes": small + big}
        for k, v in ms.items():
            t = float(np.median(v))
            row[k + "_ms"] = round(t, 4)
            row[k + "_GBps"] = round((small + big) / (t * 1e-3) / 1e9, 1)
            row[k + "_of_hbm"] = round((small + big) / (t * 1e-3) / HBM, 3)
        rows.append(row)
    return rows


def step_rows(b):
    torch.manual_seed(0)
    net0 = Resnet18_8s(ver_dim=2 * K, seg_dim=2).cuda().train()
    nets = {"default": net0, "deterministic": copy.deepcopy(net0)}
    opts = {k: torch.optim.Adam(n.parameters(), lr=1e-3) for k, n in nets.items()}
    rng = np.random.default_rng(0)
    x = torch.randn(b, 3, H, W, device="cuda")
    mask = torch.from_numpy((rng.random((b, H, W)) < 0.1).astype(np.int64)).cuda()
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [W, H], (b, K, 2)), np.ones((b, K, 1))], 2)).cuda()
    wgt = mask[:, None].float()

    def step(k):
        torch.use_deterministic_algorithms(k == "deterministic")
        try:
            net, opt = nets[k], opts[k]
            opt.zero_grad()
            seg, ver = net.forward_train(x)
            ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
            (ls.mean() + lv.mean()).backward()
            opt.step()
        finally:
            torch.use_deterministic_algorithms(False)

    ms = {k: [] for k in nets}
    for i in range(STEPS + 2):
        for k in nets:
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            step(k)
            e.record()
            e.synchronize()
            if i >= 2:
                ms[k].append(a.elapsed_time(e))
    out = {"batch": b}
    for k, v in ms.items():
        out[k + "_step_ms"] = round(float(np.median(v)), 2)
    del nets, opts
    torch.cuda.empty_cache()
    return out


def main():
    if not torch.cuda.is_available():
        raise SystemExit("upsample_train.py needs a CUDA device")
    name, power, clock = gpu_info()
    stages = [r for b in BATCHES for r in stage_rows(b)]
    steps = [step_rows(b) for b in BATCHES]
    print(json.dumps({"bench": "upsample_train", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
                      "hbm_peak_Bps": HBM, "stages": stages, "forward_train_step": steps}))


if __name__ == "__main__":
    main()
