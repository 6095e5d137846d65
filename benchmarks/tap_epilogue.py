"""Device time of the per-tap convolution (`k_conv_tap`) at the stage shapes of the bench forward, set against
the time its MMAs alone would take.

Batch 16, 60x80 outputs: the layer2, layer3, layer4, fc.0 and conv8s.0 forms, with and without residual.  Each
layer is `pvnet_conv2d_nhwc` in MODE_PER_TAP on seeded inputs, timed with CUDA events: 5 warm-up calls, then 20
timed calls back to back, per sweep; the sweep over all layers is repeated (--sweeps, default 5) so that the clock
sampler sees a second or more of load, and a layer's time is the median of all its timed calls.

Per layer the JSON line carries: ms; the algorithmic TFLOP/s (2 x b x Ho x Wo x Cout x Cin x taps over ms); the
MMA-issue floor in ms at the SM clock sampled during the run -- items per CTA (rounds of the persistent CTAs) x
K-blocks x 1024 clocks at a 256-channel N tile, scaled by BN/256 for the narrower tiles, i.e. what the layer
would take if the tensor cores never waited; and the bytes its epilogue moves (output written, residual read).
The line also names the GPU, its power limit and the sampled SM clock.  Needs a GPU: without one it prints the
shape table's static columns to stderr and fails.

  python benchmarks/tap_epilogue.py [--label TEXT] [--sweeps N]
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BATCH, HO, WO = 16, 60, 80
SMS_H100 = 132
# name, Cin, Cout, ksize, stride, dilation, act (0 none, 1 ReLU, 2 LeakyReLU), residual
LAYERS = [
    ("layer2.0.conv1", 64, 128, 3, 2, 1, 1, False),
    ("layer2.0.downsample", 64, 128, 1, 2, 1, 0, False),
    ("layer2.x.conv2", 128, 128, 3, 1, 1, 1, True),
    ("layer2.1.conv1", 128, 128, 3, 1, 1, 1, False),
    ("layer3.0.conv1", 128, 256, 3, 1, 2, 1, False),
    ("layer3.0.downsample", 128, 256, 1, 1, 1, 0, False),
    ("layer3.x.conv2", 256, 256, 3, 1, 2, 1, True),
    ("layer3.1.conv1", 256, 256, 3, 1, 2, 1, False),
    ("layer4.0.conv1", 256, 512, 3, 1, 4, 1, False),
    ("layer4.0.downsample", 256, 512, 1, 1, 1, 0, False),
    ("layer4.x.conv2", 512, 512, 3, 1, 4, 1, True),
    ("layer4.1.conv1", 512, 512, 3, 1, 4, 1, False),
    ("fc.0", 512, 256, 3, 1, 1, 1, False),
    ("conv8s.0", 384, 128, 3, 1, 1, 2, False),
]


def plan_bn(cout, m_tiles, sms):
    """conv_plan's N tile: the divisor of Cout among 256/128/64/32 with the lowest rounds x bytes-per-K-block cost,
    the wider tile on a tie."""
    best = None
    for bn in (256, 128, 64, 32):
        if cout % bn:
            continue
        cost = -(-(m_tiles * (cout // bn)) // sms) * (128 * 32 * 4 + bn * 32 * 4)
        if best is None or cost < best[0]:
            best = (cost, bn)
    return best[1]


def static_row(layer, sms):
    """What follows from the shapes alone: N tile, rounds, K-blocks, MMA-issue clocks, FLOPs, epilogue bytes."""
    name, cin, cout, k, stride, dil, act, with_res = layer
    m_tiles = BATCH * (-(-HO // 8)) * (-(-WO // 16))
    bn = plan_bn(cout, m_tiles, sms)
    rounds = -(-(m_tiles * (cout // bn)) // sms)
    kblocks = k * k * (-(-cin // 32))
    px = BATCH * HO * WO
    return dict(layer=name, cin=cin, cout=cout, ksize=k, stride=stride, dilation=dil, residual=with_res, bn=bn,
                rounds=rounds, k_blocks=kblocks, mma_issue_clocks=rounds * kblocks * 1024 * bn // 256,
                gflop=round(2.0 * px * cout * cin * k * k / 1e9, 2),
                epilogue_write_bytes=px * cout * 4, epilogue_residual_bytes=px * cout * 4 if with_res else 0)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--label", default="", help="free text copied into the line (which build this is)")
    ap.add_argument("--sweeps", type=int, default=5)
    ap.add_argument("--warm", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if args.sweeps < 1 or args.reps < 1:
        ap.error("--sweeps and --reps must be at least 1")

    import torch
    if not torch.cuda.is_available():
        for layer in LAYERS:
            print(json.dumps(static_row(layer, SMS_H100)), file=sys.stderr)
        raise RuntimeError("tap_epilogue.py needs a CUDA device: a time is only measured on the GPU")

    import bench
    from pvnet_b200 import conv as pc

    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    gen = torch.Generator().manual_seed(31)
    work = []
    for layer in LAYERS:
        name, cin, cout, k, stride, dil, act, with_res = layer
        x = pc.round_tf32(torch.randn(BATCH, HO * stride, WO * stride, cin, generator=gen).to(dev))
        w = pc.pack_weight((torch.randn(cout, cin, k, k, generator=gen) / np.sqrt(cin * k * k)).to(dev))
        bias = torch.randn(cout, generator=gen).to(dev)
        res = torch.randn(BATCH, HO, WO, cout, generator=gen).to(dev) if with_res else None
        out = torch.empty(BATCH, HO, WO, cout, device=dev)
        work.append((layer, x, w, bias, res, out))

    def call(item):
        (name, cin, cout, k, stride, dil, act, with_res), x, w, bias, res, out = item
        pc.conv2d_nhwc(x, 0, cin, w, bias, out, 0, cout, k, stride, dil, act, res, 0, round_out=True)

    times = {layer[0]: [] for layer in LAYERS}
    sampler = bench.ClockSampler(0)
    pc.set_mode(pc.MODE_PER_TAP)
    try:
        for item in work:                       # first launches load the module and set the kernel attributes
            call(item)
        torch.cuda.synchronize()
        sampler.start()
        for _ in range(args.sweeps):
            evs = []
            for item in work:
                for _ in range(args.warm):
                    call(item)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.reps + 1)]
                ev[0].record()
                for i in range(args.reps):
                    call(item)
                    ev[i + 1].record()
                evs.append(ev)
            torch.cuda.synchronize()
            for item, ev in zip(work, evs):
                times[item[0][0]] += [ev[i].elapsed_time(ev[i + 1]) for i in range(args.reps)]
        clocks = sampler.stop()
    finally:
        pc.set_mode(pc.MODE_AUTO)

    mhz = clocks.get("sm_mhz")
    rows = []
    for layer in LAYERS:
        row = static_row(layer, sms)
        ms = float(np.median(times[layer[0]]))
        row["ms"] = round(ms, 4)
        row["tflops"] = round(row["gflop"] / ms, 1)
        row["mma_floor_ms"] = round(row["mma_issue_clocks"] / (mhz * 1e3), 4) if mhz else None
        rows.append(row)
    print(json.dumps(dict(benchmark="tap_epilogue", label=args.label, gpu=bench.gpu_identity(0), clocks=clocks, sms=sms,
                          batch=BATCH, ho=HO, wo=WO, warm=args.warm, reps=args.reps, sweeps=args.sweeps,
                          total_ms=round(sum(r["ms"] for r in rows), 4), layers=rows)))


if __name__ == "__main__":
    main()
