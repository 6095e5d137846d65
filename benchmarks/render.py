"""Mesh rendering on the device (`pvnet_b200.render.render_mesh`, csrc/render.cu) by CUDA events: depth and
RGB+depth at b = 1, 16, 64, 480x640, icospheres of 20 480, 81 920 and 327 680 faces at LINEMOD-like poses; next to it
the numpy oracle (oracle/render_oracle.py) per image on the host.  Appends one JSON line per measurement to
profiles/render_h100_<power>w.jsonl (or --out), with the card name and power limit read in the same run.

Derived numbers, computed here from shapes and outputs:
  fragments/s  2 x covered pixels / time: every covered pixel of a closed convex mesh with both sides inside the clip
               range is covered by one front and one back face, so that is how many fragments pass the test;
  resolve      bytes = 8 (key read) + 4 (depth) and/or 3 (RGB) per pixel, and that over 3.35 TB/s (the H100 SXM data
               sheet's HBM3 bandwidth) as the least time the resolve pass could take."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import render_oracle as ro  # noqa: E402
from pvnet_b200.render import render_mesh  # noqa: E402
from tests import render_cases as rc  # noqa: E402

H, W = 480, 640
HBM_BPS = 3.35e12


def device_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    card, power = q[0], float(q[1])
    out = args.out or os.path.join(ROOT, "profiles", f"render_h100_{int(round(power))}w.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    dev = "cuda:0"
    K = torch.from_numpy(rc.K_LINEMOD).to(dev)
    recs = []
    for subdiv in (5, 6, 7):
        v, f = rc.icosphere(subdiv, 90.0)
        vd, fd = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
        cd = torch.from_numpy(np.random.default_rng(0).uniform(0, 1, (len(v), 3)).astype(np.float32)).to(dev)
        for b in (1, 16, 64):
            P = torch.from_numpy(rc.poses(b, np.random.default_rng(b))).to(dev)
            for mode in ("depth", "rgb+depth"):
                res = render_mesh(vd, fd, K, P, H, W, 100, 2000, colors=cd, mode=mode)
                depth = res if mode == "depth" else res[1]
                covered = int((depth > 0).sum())
                ms = device_ms(lambda: render_mesh(vd, fd, K, P, H, W, 100, 2000, colors=cd, mode=mode), args.iters)
                rbytes = b * H * W * (8 + 4 + (3 if mode != "depth" else 0))
                recs.append({"card": card, "power_limit_w": power, "faces": int(len(f)), "b": b, "h": H, "w": W,
                             "mode": mode, "device_ms": ms, "covered_pixels": covered,
                             "fragments_per_s": 2 * covered / (ms * 1e-3), "resolve_bytes": rbytes,
                             "resolve_bound_ms": rbytes / HBM_BPS * 1e3})
                print(json.dumps(recs[-1]), flush=True)
    # the oracle evaluates every face at every pixel, so its time is linear in the faces: a 320-face icosphere
    v, f = rc.icosphere(2, 90.0)
    P = rc.poses(1, np.random.default_rng(1))
    t0 = time.perf_counter()
    ro.render(v, f, rc.K_LINEMOD, P, H, W, 100, 2000, colors=np.full((len(v), 3), 0.5, np.float32))
    recs.append({"card": card, "power_limit_w": power, "faces": int(len(f)), "b": 1, "h": H, "w": W,
                 "mode": "rgb+depth", "oracle_host_ms_per_image": (time.perf_counter() - t0) * 1e3})
    print(json.dumps(recs[-1]))
    with open(out, "a") as fh:
        for r in recs:
            fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
