"""Resnet18_8s_detector / Resnet18_8s_detector_v2 on one GPU: eval (native vs the torch graph on cuDNN-TF32 in
channels_last and NCHW), per-stage times of the native eval forward (the score head stage included), and one training
step (forward_train + BCE-with-logits + backward() + the native Adam, vs the torch graph in channels_last +
torch.optim.Adam), with the helpers and conventions of benchmarks/backbones.py.

    python benchmarks/detectors.py [--batch 16] [--train-batch 16] [--iters 20] [--out FILE.jsonl]

Prints one JSON line per measurement (and appends them to --out), each carrying the GPU's name and power limit.
Batch 16 at 480x640, seeded weights; v2 runs on a fresh base detector.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from backbones import H, W, flops_per_image, gpu_info, stage_rows, timed  # noqa: E402

from pvnet_b200 import model_repository as mr  # noqa: E402
from pvnet_b200.optim import Adam  # noqa: E402

NETS = ("Resnet18_8s_detector", "Resnet18_8s_detector_v2")


def make(name, dev, seed=0):
    torch.manual_seed(seed)
    net = mr.Resnet18_8s_detector() if name == "Resnet18_8s_detector" else \
        mr.Resnet18_8s_detector_v2(mr.Resnet18_8s_detector())
    return net.to(dev)


def eval_rows(name, dev, batch, iters, info):
    net = make(name, dev).eval()
    x = torch.randn(batch, 3, H, W, device=dev)
    flops = flops_per_image(net)
    rows = []
    with torch.no_grad():
        ms, ms_min = timed(lambda: net.forward_native(x), iters)
        rows.append(dict(what="eval", net=name, arm="native", batch=batch, ms=ms, ms_min=ms_min,
                         images_s=batch / ms * 1e3, gflop_per_image=flops / 1e9, tflop_s=flops * batch / ms / 1e9))
        for fmt, mf in (("channels_last", torch.channels_last), ("nchw", torch.contiguous_format)):
            tnet = make(name, dev).eval().to(memory_format=mf)
            xt = x.contiguous(memory_format=mf)
            with torch.backends.cudnn.flags(enabled=True, benchmark=True, allow_tf32=True):
                ms, ms_min = timed(lambda: tnet._forward_torch(xt), iters)
            rows.append(dict(what="eval", net=name, arm="cudnn_tf32_" + fmt, batch=batch, ms=ms, ms_min=ms_min,
                             images_s=batch / ms * 1e3, gflop_per_image=flops / 1e9,
                             tflop_s=flops * batch / ms / 1e9))
            del tnet
    for r in rows:
        r.update(info)
    return rows, net, x


def train_rows(name, dev, batch, iters, info):
    x = torch.randn(batch, 3, H, W, device=dev)
    lab = (torch.rand(batch, 1, H // 8, W // 8, device=dev) < 0.3).float()
    rows = []
    net = make(name, dev).train()
    opt = Adam(net.parameters(), lr=1e-4)

    def native_step():
        F.binary_cross_entropy_with_logits(net.forward_train(x), lab).backward()
        opt.step()
        opt.zero_grad()

    flops = 3 * flops_per_image(net)
    ms, ms_min = timed(native_step, iters)
    rows.append(dict(what="train", net=name, arm="native", batch=batch, ms=ms, ms_min=ms_min,
                     images_s=batch / ms * 1e3, tflop_s=flops * batch / ms / 1e9))
    del net, opt
    torch.cuda.empty_cache()
    tnet = make(name, dev).train().to(memory_format=torch.channels_last)
    topt = torch.optim.Adam(tnet.parameters(), lr=1e-4)
    xt = x.contiguous(memory_format=torch.channels_last)

    def torch_step():
        F.binary_cross_entropy_with_logits(tnet._forward_torch(xt), lab).backward()
        topt.step()
        topt.zero_grad()

    with torch.backends.cudnn.flags(enabled=True, benchmark=True, allow_tf32=True):
        ms, ms_min = timed(torch_step, iters)
    rows.append(dict(what="train", net=name, arm="torch_cudnn_tf32_channels_last", batch=batch, ms=ms, ms_min=ms_min,
                     images_s=batch / ms * 1e3, tflop_s=flops * batch / ms / 1e9))
    del tnet, topt
    torch.cuda.empty_cache()
    for r in rows:
        r.update(info)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--train-batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--nets", default=",".join(NETS))
    ap.add_argument("--out", default=None, help="append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("benchmarks/detectors.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    rows = []
    for name in args.nets.split(","):
        start = len(rows)
        er, net, x = eval_rows(name, dev, args.batch, args.iters, info)
        rows += er + stage_rows(name, net, x, args.iters, info)
        del net, x
        torch.cuda.empty_cache()
        rows += train_rows(name, dev, args.train_batch, max(5, args.iters // 2), info)
        for r in rows[start:]:
            print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
