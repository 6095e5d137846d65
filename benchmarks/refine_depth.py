"""Depth-anchored pose refinement (`refine_poses_depth`, DESIGN.md §28) by CUDA events and on known answers.
benchmarks/refine_keypoints.py's setup: 480x640, LINEMOD K, a 20 480-face mesh, 9 farthest-point keypoints with 1-3 px
of noise and their covariances, the start from `uncertainty_pnp_batched`, b = 1, 16, 64.  The observed depth is the
mesh's render at the true pose plus 1 mm of seeded Gaussian noise.  Device time per call (8 rounds; median of 10
after 2 warm-ups) and per round; then the rotation, translation (and its optical-axis component), 2D projection and
ADD errors of the PnP start, the keypoint-anchored refinement, and the keypoint-anchored refinement followed by depth
refinement.  Prints one JSON line per measurement with the card's name and power limit read in the same run; --out
also appends them to a file."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from refine_keypoints import device_ms, errors, farthest_points, gpu_info  # noqa: E402

from oracle import refine_oracle as rfo  # noqa: E402
from pvnet_b200 import extend_utils as eu  # noqa: E402
from pvnet_b200.refine import refine_poses, refine_poses_depth  # noqa: E402
from pvnet_b200.render import render_mesh  # noqa: E402
from tests import refine_cases as rf  # noqa: E402
from tests import refine_depth_cases as rdc  # noqa: E402
from tests import refine_keypoint_cases as rkc  # noqa: E402
from tests import render_cases as rc  # noqa: E402

H, W = 480, 640
DEV = "cuda:0"
NOISE = 1e-3                                     # metres of depth noise


def axis_error_mm(P, Pt):
    """Mean |t_z - t_z,true| in mm: the translation error along the optical axis."""
    return float(np.mean(np.abs(np.asarray(P)[:, 2, 3] - np.asarray(Pt)[:, 2, 3])) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=8)
    ap.add_argument("--batches", default="1,16,64")
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
    pts = farthest_points(verts, 9)
    p3 = torch.from_numpy(pts).to(DEV)
    for b in [int(x) for x in a.batches.split(",")]:
        rng = np.random.default_rng(b)
        Pt = rf.true_poses(b, rng)
        clean = render_mesh(v, f, K, torch.from_numpy(Pt).float().to(DEV), H, W, rf.NEAR, rf.FAR)
        mask = (clean > 0).to(torch.uint8)
        sig = rng.uniform(1.0, 3.0, (b, len(pts)))
        kp_np, cov_np = rkc.keypoint_votes(Pt, rc.K_LINEMOD, pts, 1.0, rng)
        kp_true = np.stack([np.stack(rfo.project(pts.astype(np.float64), Pt[i], rc.K_LINEMOD), -1) for i in range(b)])
        kp_np = (kp_true + (kp_np - kp_true) * sig[..., None]).astype(np.float32)
        cov_np = (cov_np * (sig ** 2)[..., None, None]).astype(np.float32)
        kp, cov = torch.from_numpy(kp_np).to(DEV), torch.from_numpy(cov_np).to(DEV)
        depth = torch.from_numpy(rdc.noisy(clean.cpu().numpy(), NOISE, np.random.default_rng(1000 + b))).to(DEV)
        P0 = eu.uncertainty_pnp_batched(kp, p3, K, cov=cov)
        anchored = refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds, keypoints=kp, points_3d=p3,
                                cov=cov)
        ms = device_ms(lambda: refine_poses_depth(mask, depth, anchored, K, v, f, rf.NEAR, rf.FAR, rdc.GATE,
                                                  rounds=a.rounds), a.iters)
        ms0 = device_ms(lambda: refine_poses_depth(mask, depth, anchored, K, v, f, rf.NEAR, rf.FAR, rdc.GATE,
                                                   rounds=0), a.iters)
        emit(dict(what="refine_depth_time", b=b, h=H, w=W, faces=int(len(faces)), rounds=a.rounds, call_ms=ms,
                  rounds0_ms=ms0, per_round_ms=(ms - ms0) / max(a.rounds, 1)))
        out, info = refine_poses_depth(mask, depth, anchored, K, v, f, rf.NEAR, rf.FAR, rdc.GATE, rounds=a.rounds,
                                       return_info=True)
        res = {}
        for key, P in (("pnp_start", P0), ("keypoint_anchored", anchored), ("anchored_then_depth", out)):
            P = P.cpu().numpy()
            res[key] = errors(P, Pt, rc.K_LINEMOD, verts)
            res[key]["axis_mm"] = axis_error_mm(P, Pt)
        res["anchored_then_depth"]["status_nonzero"] = int((info["status"] & ~16 != 0).sum().item())
        res["anchored_then_depth"]["dist_rose"] = int((info["dist_after"] > info["dist_before"]).sum().item())
        emit(dict(what="refine_depth_accuracy", b=b, h=H, w=W, faces=int(len(faces)), keypoints=len(pts),
                  noise_px="1-3", depth_noise_m=NOISE, gate_m=rdc.GATE, start="uncertainty_pnp_batched",
                  rounds=a.rounds, **res))
    if a.out:
        with open(a.out, "a") as fh:
            for d in lines:
                fh.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
