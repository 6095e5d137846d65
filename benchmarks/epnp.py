"""EPnP on the device (`pnp(..., method=SOLVEPNP_EPNP)`, csrc/epnp.cu) by CUDA events, next to the LM solver
(`pnp(method=0)`) and, where cv2 imports, the reference's per-image `cv2.solvePnP(..., SOLVEPNP_EPNP)` loop by host
wall clock.  Writes one JSON line to profiles/epnp_h100_<power>w.jsonl (or --out), with the card name and power limit
read in the same run."""
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

from pvnet_b200 import evaluation as ev  # noqa: E402
from tests import pnp_cases as pc  # noqa: E402


def problems(b, pn, seed=0):
    rng = np.random.default_rng(seed)
    P = pc.object_points("cloud", pn, rng)
    K = pc.camera("cloud")
    R, t = pc.poses("cloud", b, rng)
    x = (pc.project(P, R, t, K) + rng.normal(0, 1.0, (b, pn, 2))).astype(np.float32)
    return P, K, x


def device_ms(fn, iters=200, warmup=20):
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
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    card, power = q[0], float(q[1])
    dev = "cuda:0"
    rec = {"card": card, "power_limit_w": power, "epnp_ms": {}, "lm_ms": {}, "cv2_epnp_ms": {}}
    for b, pn in ((16, 9), (256, 9), (4096, 9), (256, 1024)):
        P, K, x = problems(b, pn)
        xd, pd = torch.from_numpy(x).to(dev), torch.from_numpy(P).to(dev)
        rec["epnp_ms"][f"b{b}_pn{pn}"] = device_ms(lambda: ev.pnp(pd, xd, K, method=ev.SOLVEPNP_EPNP))
    for b in (16, 256):
        P, K, x = problems(b, 9)
        xd, pd = torch.from_numpy(x).to(dev), torch.from_numpy(P).to(dev)
        rec["lm_ms"][f"b{b}_pn9"] = device_ms(lambda: ev.pnp(pd, xd, K, method=0))
    try:
        import cv2
        rec["cv2_version"] = cv2.__version__
        for b, pn in ((16, 9), (256, 9), (256, 1024)):
            P, K, x = problems(b, pn)
            t0 = time.perf_counter()
            for i in range(b):
                cv2.solvePnP(P.astype(np.float64)[None], x[i].astype(np.float64)[None], K, np.zeros((8, 1)),
                             flags=cv2.SOLVEPNP_EPNP)
            rec["cv2_epnp_ms"][f"b{b}_pn{pn}"] = (time.perf_counter() - t0) * 1e3
    except ImportError:
        print("cv2 is not installed: the per-image cv2.solvePnP loop is not measured")
        rec["cv2_epnp_ms"] = None
    out = args.out or os.path.join(ROOT, "profiles", f"epnp_h100_{int(round(power))}w.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    with open(out, "a") as f:
        f.write(json.dumps(rec) + "\n")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
