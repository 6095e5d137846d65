"""Keypoint-anchored pose refinement (`refine_poses(..., keypoints=)`, DESIGN.md §27) by CUDA events and on known
answers.  Device time per call (8 rounds; median of 10 after 2 warm-ups) with and without the keypoint term at
b = 1, 16, 64, 480x640, on a 20 480-face mesh.  Then, on the same seeded scenes -- the truth's coverage as the mask,
9 keypoints at the true projections plus noise of 1-3 px with their covariances, the start from
`uncertainty_pnp_batched` on those keypoints -- the rotation, translation, 2D projection and ADD errors of the PnP
start, the silhouette-only refinement and the keypoint-anchored one at lambda = 0.25, 1 and 4.  Prints one JSON line
per measurement with the card's name and power limit read in the same run; --out also appends them to a file."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refine_oracle as rfo  # noqa: E402
from pvnet_b200 import extend_utils as eu  # noqa: E402
from pvnet_b200.refine import refine_poses  # noqa: E402
from pvnet_b200.render import render_mesh  # noqa: E402
from tests import refine_cases as rf  # noqa: E402
from tests import refine_keypoint_cases as rkc  # noqa: E402
from tests import render_cases as rc  # noqa: E402

H, W = 480, 640
DEV = "cuda:0"
LAMBDAS = (0.25, 1.0, 4.0)


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


def farthest_points(verts, n):
    """n of the mesh's vertices by farthest-point sampling from the one farthest from the centroid."""
    v = np.asarray(verts, np.float64)
    idx = [int(np.argmax(np.linalg.norm(v - v.mean(0), axis=1)))]
    d = np.linalg.norm(v - v[idx[0]], axis=1)
    for _ in range(n - 1):
        idx.append(int(np.argmax(d)))
        d = np.minimum(d, np.linalg.norm(v - v[idx[-1]], axis=1))
    return v[idx].astype(np.float32)


def errors(P, Pt, K, verts):
    """Mean over images: rotation error (deg), translation error (mm), 2D projection error (px), ADD (mm)."""
    v = np.asarray(verts, np.float64)
    out = []
    for p, q in zip(P, Pt):
        r, tr = rf.pose_error(p, q)
        a, b = np.stack(rfo.project(v, p, K), -1), np.stack(rfo.project(v, q, K), -1)
        add = np.linalg.norm((v @ p[:, :3].T + p[:, 3]) - (v @ q[:, :3].T + q[:, 3]), axis=1).mean()
        out.append((r, tr * 1e3, np.linalg.norm(a - b, axis=1).mean(), add * 1e3))
    e = np.array(out)
    return dict(rot_deg=float(e[:, 0].mean()), trans_mm=float(e[:, 1].mean()), proj2d_px=float(e[:, 2].mean()),
                add_mm=float(e[:, 3].mean()), rot_deg_median=float(np.median(e[:, 0])))


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
        mask = (render_mesh(v, f, K, torch.from_numpy(Pt).float().to(DEV), H, W, rf.NEAR, rf.FAR) > 0).to(torch.uint8)
        sig = rng.uniform(1.0, 3.0, (b, len(pts)))
        kp_np, cov_np = rkc.keypoint_votes(Pt, rc.K_LINEMOD, pts, 1.0, rng)
        kp_true = np.stack([np.stack(rfo.project(pts.astype(np.float64), Pt[i], rc.K_LINEMOD), -1) for i in range(b)])
        kp_np = (kp_true + (kp_np - kp_true) * sig[..., None]).astype(np.float32)
        cov_np = (cov_np * (sig ** 2)[..., None, None]).astype(np.float32)
        kp, cov = torch.from_numpy(kp_np).to(DEV), torch.from_numpy(cov_np).to(DEV)
        P0 = eu.uncertainty_pnp_batched(kp, p3, K, cov=cov)
        plain = device_ms(lambda: refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds), a.iters)
        anchored = device_ms(lambda: refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds, keypoints=kp,
                                                  points_3d=p3, cov=cov), a.iters)
        emit(dict(what="refine_keypoints_time", b=b, h=H, w=W, faces=int(len(faces)), keypoints=len(pts),
                  rounds=a.rounds, silhouette_only_ms=plain, keypoint_anchored_ms=anchored,
                  keypoint_term_per_round_ms=(anchored - plain) / max(a.rounds, 1)))
        res = dict(pnp_start=errors(P0.cpu().numpy(), Pt, rc.K_LINEMOD, verts))
        out, info = refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds, return_info=True)
        res["silhouette_only"] = errors(out.cpu().numpy(), Pt, rc.K_LINEMOD, verts)
        res["silhouette_only"]["status_nonzero"] = int((info["status"] & ~16 != 0).sum().item())
        for lam in LAMBDAS:
            out, info = refine_poses(mask, P0, K, v, f, rf.NEAR, rf.FAR, rounds=a.rounds, keypoints=kp, points_3d=p3,
                                     cov=cov, keypoint_weight=lam, return_info=True)
            r = errors(out.cpu().numpy(), Pt, rc.K_LINEMOD, verts)
            r["status_nonzero"] = int((info["status"] & ~16 != 0).sum().item())
            r["cost_rose"] = int((info["cost_after"] > info["cost_before"]).sum().item())
            res[f"anchored_lambda_{lam:g}"] = r
        emit(dict(what="refine_keypoints_accuracy", b=b, h=H, w=W, faces=int(len(faces)), keypoints=len(pts),
                  noise_px="1-3", start="uncertainty_pnp_batched", rounds=a.rounds, **res))
    if a.out:
        with open(a.out, "a") as fh:
            for d in lines:
                fh.write(json.dumps(d) + "\n")


if __name__ == "__main__":
    main()
