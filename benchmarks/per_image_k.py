"""Uncertainty PnP with one camera matrix per image (the truncated-LINEMOD evaluation), one JSON line per run.

For batches of 16 and 64 images of the LINEMOD cat's 9 keypoints, each with its own K (principal points shifted as
by a crop), the covariance form of the solver:
  - batched:        one `uncertainty_pnp_batched` call with the cameras as a CUDA [b,3,3]
                    (`pvnet_uncertainty_pnp_per_image_k`);
  - loop_host_k:    one single-K call per image with that image's K as a host array (`pvnet_uncertainty_pnp`), the
                    loop the truncated mode needed before the per-image entry existed;
  - loop_device_k:  the same loop with the cameras on the device as the loader delivers them (`Ks.cuda()`), each
                    read back with `.cpu()` first -- what the single-K entry made a caller do: one synchronisation per
                    image;
and the whole evaluation of a batch (poses and the ADD / 2-D projection / 5 cm 5 degree metrics on a 2 k-vertex
model):
  - eval_batched:   `Evaluator.evaluate_keypoints_batch` with CUDA keypoints, covariances, poses and cameras;
  - eval_per_image: `Evaluator.evaluate_uncertainty(..., 'use_intrinsic', intri_matrix=K)` per image on numpy
                    inputs, the reference's loop (tools/train_linemod.py:199-205).
Each figure is host wall-clock per batch, from the first call to a device synchronisation after the last (median of
REPS batches, after warm-up): the loops are bound by host work and launches, which device-event timing would not
show.  `batched_device_ms` is the batched call's own device time (CUDA events).  The batched poses are checked to
equal the loop's bit for bit before anything is timed.
    python benchmarks/per_image_k.py > profiles/per_image_k_<gpu>.json
"""
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pnp_oracle as pno  # noqa: E402
from pvnet_b200 import evaluation as ev  # noqa: E402
from pvnet_b200 import extend_utils as eu  # noqa: E402

BATCHES = (16, 64)
REPS = int(os.environ.get("REPS", "30"))
K_LINEMOD = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])
GOLDEN = os.path.join(ROOT, "tests", "golden", "pnp_cases.npz")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def inputs(b, seed=0):
    """points_3d [9,3], cameras [b,3,3], float32 keypoints [b,9,2] and covariances [b,9,2,2], poses [b,3,4]."""
    rng = np.random.default_rng(seed)
    P = np.load(GOLDEN)["points_3d"]
    K = np.stack([K_LINEMOD] * b)
    K[:, 0, 2] -= rng.uniform(-200, 200, b)
    K[:, 1, 2] -= rng.uniform(-150, 150, b)
    kp, pose = [], []
    for i in range(b):
        R = pno.rodrigues(rng.normal(0, 1, 3))
        t = np.array([rng.uniform(-.1, .1), rng.uniform(-.1, .1), rng.uniform(0.5, 1.2)])
        X = P @ R.T + t
        kp.append(np.stack([K[i, 0, 0] * X[:, 0] / X[:, 2] + K[i, 0, 2], K[i, 1, 1] * X[:, 1] / X[:, 2] + K[i, 1, 2]],
                           1) + rng.normal(0, 1, (9, 2)))
        pose.append(np.concatenate([R, t[:, None]], 1))
    A = rng.normal(0, 1, (b, 9, 2, 2))
    cov = A @ A.transpose(0, 1, 3, 2) + 0.2 * np.eye(2)
    return P, K, np.stack(kp).astype(np.float32), cov.astype(np.float32), np.stack(pose).astype(np.float32)


def wall_ms(fn, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def device_ms(fn):
    for _ in range(3):
        fn()
    t = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        t.append(a.elapsed_time(b))
    return float(np.median(t))


class _ModelDB:
    def __init__(self, model):
        self.model = model

    def get_ply_model(self, class_type):
        return self.model

    def get_diameter(self, class_type):
        return 0.12


class _Projector:
    intrinsic_matrix = {"linemod": K_LINEMOD}


def main():
    name, power, clock_mhz = gpu_info()
    dev = torch.device("cuda", 0)
    rows = []
    for b in BATCHES:
        P, K, kp, cov, pose = inputs(b)
        p3 = torch.from_numpy(P.astype(np.float32)).to(dev)
        kp_d, cov_d, pose_d, K_d = (torch.from_numpy(x).to(dev) for x in (kp, cov, pose, K))

        def batched():
            return eu.uncertainty_pnp_batched(kp_d, p3, K_d, cov=cov_d)

        def loop_host_k():
            return [eu.uncertainty_pnp_batched(kp_d[i:i + 1], p3, K[i], cov=cov_d[i:i + 1]) for i in range(b)]

        def loop_device_k():
            return [eu.uncertainty_pnp_batched(kp_d[i:i + 1], p3, K_d[i].cpu().numpy(), cov=cov_d[i:i + 1])
                    for i in range(b)]
        same = bool(torch.equal(torch.nan_to_num(batched()), torch.nan_to_num(torch.cat(loop_host_k()))))
        if not same:
            raise SystemExit("batched per-image-K poses differ from the per-image loop")

        # the evaluation: the reference tree's VotingType stands in for the dataset module
        vt = types.ModuleType("lib.datasets.linemod_dataset")
        vt.VotingType = type("VotingType", (), {"BB8": 0, "get_pts_3d": staticmethod(lambda v, c: P)})
        sys.modules.setdefault("lib.datasets", types.ModuleType("lib.datasets"))
        sys.modules["lib.datasets.linemod_dataset"] = vt
        model = np.random.default_rng(1).uniform(-0.05, 0.05, (2048, 3)).astype(np.float32)
        e_batch = ev.Evaluator(model_db=_ModelDB(model), projector=_Projector())
        e_one = ev.Evaluator(model_db=_ModelDB(model), projector=_Projector())

        def eval_batched():
            return e_batch.evaluate_keypoints_batch(kp_d, pose_d, "cat", K_d, covar=cov_d)

        def eval_per_image():
            return [e_one.evaluate_uncertainty(kp[i], cov[i], pose[i], "cat", "use_intrinsic", intri_matrix=K[i])
                    for i in range(b)]
        rows.append({"batch": b, "poses_equal_loop": same,
                     "batched_ms": wall_ms(batched), "batched_device_ms": device_ms(batched),
                     "loop_host_k_ms": wall_ms(loop_host_k), "loop_device_k_ms": wall_ms(loop_device_k),
                     "eval_batched_ms": wall_ms(eval_batched), "eval_per_image_ms": wall_ms(eval_per_image)})
    print(json.dumps({"bench": "per_image_k", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock_mhz,
                      "points": 9, "reps": REPS, "rows": rows}))


if __name__ == "__main__":
    main()
