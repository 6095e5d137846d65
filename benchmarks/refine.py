"""Silhouette pose refinement on the device (`pvnet_b200.refine.refine_poses`, csrc/refine.cu) by CUDA events:
device time per call (rounds = 8) and per round at b = 1, 16, 64, 480x640, on a 20 480-face mesh at LINEMOD-like
poses 3 degrees and 1 cm from the truth whose coverage is the mask.  Beside it, in the same run: the pose step it
follows (`uncertainty_pnp_batched`, 9 keypoints with covariances) at the same batch, and the numpy oracle
(oracle/refine_oracle.py) on the host for one image and one round of a 320-face mesh (its renderer evaluates every
face at every pixel, so a 20 480-face round would take minutes).  Prints one JSON line per measurement, with the
card's name and power limit read in the same run; --out also appends them to a file."""
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

from oracle import refine_oracle as rfo  # noqa: E402
from pvnet_b200 import extend_utils as eu  # noqa: E402
from pvnet_b200.refine import refine_poses  # noqa: E402
from pvnet_b200.render import render_mesh  # noqa: E402
from tests import refine_cases as rf  # noqa: E402
from tests import render_cases as rc  # noqa: E402

H, W = 480, 640
DEV = "cuda:0"


def device_ms(fn, iters, warmup=2):
    """Median of `iters` single-call CUDA-event timings after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else ("?", "?")
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--batches", default="1,16,64")
    ap.add_argument("--oracle-faces-subdiv", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = gpu_info()
    lines = []

    def emit(d):
        d.update(gpu=name, power_limit=power)
        print(json.dumps(d), flush=True)
        lines.append(d)

    verts, faces = rf.lumpy_mesh(5)
    v, f = torch.from_numpy(verts).to(DEV), torch.from_numpy(faces).to(DEV)
    K = torch.from_numpy(rc.K_LINEMOD).to(DEV)
    kp3 = torch.from_numpy(np.random.default_rng(9).normal(0, 0.04, (9, 3)).astype(np.float32)).to(DEV)
    for b in [int(x) for x in a.batches.split(",")]:
        rng = np.random.default_rng(b)
        Pt = rf.true_poses(b, rng)
        P0 = torch.from_numpy(rf.perturb(Pt, rng)).to(DEV)
        mask = (render_mesh(v, f, K, torch.from_numpy(Pt).float().to(DEV), H, W, rf.NEAR, rf.FAR) > 0).to(torch.uint8)
        call = device_ms(lambda: refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds), a.iters)
        eval_only = device_ms(lambda: refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=0), a.iters)
        out, info = refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds, return_info=True)
        # the pose step before it: uncertainty PnP on 9 keypoints per image
        kp2 = torch.from_numpy(rng.uniform(100, 500, (b, 9, 2)).astype(np.float32)).to(DEV)
        cov = torch.eye(2, device=DEV).expand(b, 9, 2, 2).contiguous()
        pnp = device_ms(lambda: eu.uncertainty_pnp_batched(kp2, kp3, K, cov=cov), a.iters)
        d0, d1 = info["dist_before"].cpu().numpy(), info["dist_after"].cpu().numpy()
        emit(dict(what="refine_poses", b=b, h=H, w=W, faces=int(len(faces)), rounds=a.rounds, call_ms=call,
                  per_round_ms=(call - eval_only) / max(a.rounds, 1), evaluation_only_ms=eval_only,
                  uncertainty_pnp_batched_ms=pnp, mean_dist_before_px=float(np.nanmean(d0)),
                  mean_dist_after_px=float(np.nanmean(d1)), pairs_mean=float(info["pairs"].float().mean().item())))
    # the oracle on the host: one image, one round
    ov, of = rf.lumpy_mesh(a.oracle_faces_subdiv)
    rng = np.random.default_rng(0)
    Pt = rf.true_poses(1, rng)
    P0 = rf.perturb(Pt, rng)
    ovd, ofd = torch.from_numpy(ov).to(DEV), torch.from_numpy(of).to(DEV)
    m = (render_mesh(ovd, ofd, K, torch.from_numpy(Pt).float().to(DEV), H, W, rf.NEAR, rf.FAR) > 0)[0].cpu().numpy()
    t0 = time.perf_counter()
    rfo.refine_image(m, P0[0], rc.K_LINEMOD, ov, of, rf.NEAR, rf.FAR, rounds=1)
    host = time.perf_counter() - t0
    mo, Po = torch.from_numpy(m[None].astype(np.uint8)).to(DEV), torch.from_numpy(P0).to(DEV)
    dev1 = device_ms(lambda: refine_poses(mo, Po, K, ovd, ofd, rf.NEAR, rf.FAR, rounds=1), a.iters)
    emit(dict(what="oracle_host_vs_device", b=1, h=H, w=W, faces=int(len(of)), rounds=1, oracle_host_s=host,
              device_ms=dev1))
    if a.out:
        with open(a.out, "a") as fh:
            for d in lines:
                fh.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
