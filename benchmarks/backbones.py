"""Resnet18_8s / Resnet34_8s / Resnet50_8s / Resnet50_8s_2o on one GPU: eval images/s (native vs the torch graph on cuDNN), per-stage
times of the native eval forward, and one training step (native vs the torch graph), with FLOPs per image counted
from the layer shapes.

    python benchmarks/backbones.py [--batch 16] [--train-batch 16] [--iters 20] [--out FILE.jsonl]

Prints one JSON line per measurement (and appends them to --out), each carrying the GPU's name and power limit.
Eval: batch 16 at 480x640, ver_dim 18 / seg_dim 2, eval mode, seeded weights.  `native` is forward_native (fused or
separate head, NCHW output); `cudnn_*` is _forward_torch under torch.no_grad() with cuDNN's TF32 convolutions (torch's
default), in channels_last and in NCHW.  Stages: pvnet_backbone_run_stage one at a time, CUDA events around each,
median over --iters passes; each stage's time includes the host's launch gap before it, so they sum to more than the
whole forward.  Train: forward_train + the native training losses + backward() + the native Adam, vs
_forward_torch in channels_last + torch's cross-entropy / smooth-L1 + torch.optim.Adam, both in train mode; cuDNN TF32.
FLOPs: 2 * MACs of every convolution (the head included) at the layer's output resolution; the train step is
counted as 3x the forward's (forward, data and weight gradients).  Workspace: pvnet_backbone_workspace_bytes of the
eval batch, next to the stage times.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvnet_b200 import _native  # noqa: E402
from pvnet_b200 import model_repository as mr  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200.optim import Adam  # noqa: E402

H, W = 480, 640
NETS = ("Resnet18_8s", "Resnet34_8s", "Resnet50_8s", "Resnet50_8s_2o")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = (v.strip() for v in out.split(","))
        return {"gpu": name, "power_limit_w": float(pl)}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "error": str(e)[:100]}


def flops_per_image(net, h=H, w=W):
    """2 * MACs of every Conv2d for one h x w image, from the layer shapes seen by forward hooks on one forward."""
    total = 0
    hooks = []

    def hook(m, inp, out):
        nonlocal total
        k = m.kernel_size[0] * m.kernel_size[1]
        total += 2 * out.shape[2] * out.shape[3] * m.out_channels * (m.in_channels // m.groups) * k

    for m in net.modules():
        if isinstance(m, torch.nn.Conv2d):
            hooks.append(m.register_forward_hook(hook))
    with torch.no_grad():
        net._forward_torch(torch.zeros(1, 3, h, w, device=next(net.parameters()).device))
    for hk in hooks:
        hk.remove()
    return total


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts))


def make(name, dev, seed=0):
    torch.manual_seed(seed)
    return getattr(mr, name)(18, 2).to(dev)


def eval_rows(name, dev, batch, iters, info):
    net = make(name, dev).eval()
    x = torch.randn(batch, 3, H, W, device=dev)
    flops = flops_per_image(net)
    rows = []
    with torch.no_grad():
        ms, ms_min = timed(lambda: net.forward_native(x), iters)
        rows.append(dict(what="eval", net=name, arm="native", batch=batch, ms=ms, ms_min=ms_min,
                         images_s=batch / ms * 1e3, gflop_per_image=flops / 1e9,
                         tflop_s=flops * batch / ms / 1e9))
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


def stage_rows(name, net, x, iters, info):
    L = _native.lib()
    dev = x.device
    handle = net._prepare_native(dev)
    n = L.pvnet_backbone_handle_num_stages(handle)
    names = [L.pvnet_backbone_handle_stage_name(handle, i).decode() for i in range(n)]
    b, _, h, w = x.shape
    out = torch.empty(b, 20, h // net._out_scale, w // net._out_scale, device=dev)
    ws = ctypes.c_size_t()
    _native.check(L.pvnet_backbone_workspace_bytes(handle, b, h, w, ctypes.byref(ws)), "workspace_bytes")
    net.freeze_native(True)          # no per-call walk over the weights between two stages
    with torch.no_grad():
        net.run_stages(x, out, None, 0, n)
        torch.cuda.synchronize()
        times = np.zeros((iters, n))
        for it in range(iters):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
            ev[0].record()
            for i in range(n):
                net.run_stages(x, out, None, i, i + 1)
                ev[i + 1].record()
            ev[-1].synchronize()
            times[it] = [ev[i].elapsed_time(ev[i + 1]) for i in range(n)]
    net.freeze_native(False)
    med = np.median(times, 0)
    row = dict(what="stages", net=name, batch=b, total_ms=float(med.sum()), workspace_bytes=ws.value,
               stages=[{"name": s, "ms": round(float(t), 4)} for s, t in zip(names, med)])
    row.update(info)
    return [row]


def train_rows(name, dev, batch, iters, info):
    rng = np.random.default_rng(0)
    ho, wo = H // getattr(mr, name)._out_scale, W // getattr(mr, name)._out_scale    # targets on the output grid
    mask = torch.from_numpy((rng.random((batch, ho, wo)) < 0.3).astype(np.int64)).to(dev)
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [wo, ho], (batch, 9, 2)), np.ones((batch, 9, 1))],
                                         2)).to(dev)
    x = torch.randn(batch, 3, H, W, device=dev)
    rows = []
    net = make(name, dev).train()
    opt = Adam(net.parameters(), lr=1e-4)

    def native_step():
        seg, ver = net.forward_train(x)
        ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc)
        (ls.mean() + lv.mean()).backward()
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
    field = nu.vertex_targets(mask, hc)
    wgt = mask[:, None].float()

    def torch_step():
        seg, ver = tnet._forward_torch(xt)
        loss = torch.nn.functional.cross_entropy(seg, mask) + \
            nu._smooth_l1_torch(ver, field, wgt, 1.0, True).mean()
        loss.backward()
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
        raise SystemExit("benchmarks/backbones.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = gpu_info()
    rows = []
    for name in args.nets.split(","):
        start = len(rows)
        er, net, x = eval_rows(name, dev, args.batch, args.iters, info)
        rows += er
        if name != "Resnet18_8s":
            rows += stage_rows(name, net, x, args.iters, info)
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
