"""Device time of the full-resolution tail of the bench forward -- `upsample 1/2->1` and `convraw.0` (with its
fused 1x1 head and argmax) -- in both output layouts, by CUDA events around each stage (run_stages).

bench.py's `stages_ms` table times the stages with the NCHW head output; the timed step writes the pixel-major
one.  The two layouts store the same bytes in a different order, so this times both.  Batch 16, 480x640, K = 9,
uint8 mask, the bench's weights and foreground calibration; 5 warm-up repetitions, then 200 enqueued back to back
(one synchronize at the end) and the median per stage.  Prints one JSON line with the GPU's name, power limit and
the SM clocks sampled while the stages ran."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvnet_b200 import _native  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402

STAGES = ("upsample 1/2->1", "convraw.0")


def time_tail(net, x, pixel_major, warm=5, reps=200):
    L = _native.lib()
    names = [L.pvnet_backbone_stage_name(i).decode() for i in range(L.pvnet_backbone_num_stages())]
    idx = [names.index(s) for s in STAGES]
    b, _, h, w = x.shape
    ctot = net.seg_dim + net.ver_dim
    out = torch.empty([b, h, w, ctot] if pixel_major else [b, ctot, h, w], dtype=torch.float32, device=x.device)
    mask = torch.empty([b, h, w], dtype=torch.uint8, device=x.device)
    with torch.no_grad():
        net.run_stages(x, out, mask, 0, idx[0], pixel_major)          # the tail's inputs
        evs = []
        for rep in range(warm + reps):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(idx) + 1)]
            ev[0].record()
            for j, i in enumerate(idx):
                net.run_stages(x, out, mask, i, i + 1, pixel_major)
                ev[j + 1].record()
            if rep >= warm:
                evs.append(ev)
        torch.cuda.synchronize()
    ms = np.median(np.array([[ev[j].elapsed_time(ev[j + 1]) for j in range(len(idx))] for ev in evs]), axis=0)
    head_bytes = out.numel() * out.element_size() + mask.numel()
    res = {s: round(float(t), 4) for s, t in zip(STAGES, ms)}
    res["convraw.0 head+mask write GB/s"] = round(head_bytes / (ms[1] * 1e-3) / 1e9, 1)
    return res


def main():
    dev = torch.device("cuda", 0)
    net = bench.build_model(torch, dev)
    x = torch.from_numpy(syn.backbone_input(bench.BATCH, 2000)).to(dev)
    bench.calibrate_foreground(torch, net, x)
    sampler = bench.ClockSampler(0)
    sampler.start()
    rows = {("pixel-major" if pm else "nchw"): time_tail(net, x, pm) for pm in (True, False)}
    clocks = sampler.stop()
    print(json.dumps(dict(gpu=bench.gpu_identity(0), clocks=clocks, batch=bench.BATCH, h=bench.H, w=bench.W,
                          k=bench.K_KP, stages_ms=rows)))


if __name__ == "__main__":
    main()
