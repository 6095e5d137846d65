"""Pose metrics on the device against the reference's host path, one JSON line per run.

For batch 16 and model clouds of 2 k, 8 k and 32 k vertices:
  - `pose_metrics` device time (CUDA events, median of REPS) with ADD and with ADD-S (the in-kernel nearest-point
    search; both with the plain 2-D projection, as the reference's evaluate / evaluate_uncertainty);
  - the reference's path on the same inputs: its numpy metrics (evaluation_utils.py:75-141) per image, with the
    reference's own nearest-point kernel (oracle/_ref/libpvnet_refnn.so, called per image as extend_utils.py:39-60
    does) for ADD-S -- when oracle/_ref is present;
  - ADD-S pair tests per second against the FP32 issue bound (SMs x 128 lanes x SM clock / 8 instructions per pair).
    python benchmarks/eval_metrics.py > profiles/eval_metrics_<gpu>.json
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import eval_oracle as eo  # noqa: E402
from oracle import pnp_oracle as pno  # noqa: E402
from pvnet_b200 import evaluation as ev  # noqa: E402

B = 16
SIZES = (2048, 8192, 32768)
REPS = int(os.environ.get("REPS", "20"))
K = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def inputs(n, seed=0):
    rng = np.random.default_rng(seed)
    gt, pred = [], []
    for _ in range(B):
        R = pno.rodrigues(rng.normal(0, 1, 3))
        t = np.array([rng.uniform(-.1, .1), rng.uniform(-.1, .1), rng.uniform(0.5, 1.2)])
        gt.append(np.concatenate([R, t[:, None]], 1))
        pred.append(np.concatenate([pno.rodrigues(rng.normal(0, 0.05, 3)) @ R, (t + rng.normal(0, .01, 3))[:, None]], 1))
    return np.stack(pred), np.stack(gt), rng.uniform(-0.06, 0.06, (n, 3)).astype(np.float32)


def device_ms(pp, pg, m, symmetric):
    for _ in range(10):
        ev.pose_metrics(pp, pg, m, K, symmetric)
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ev.pose_metrics(pp, pg, m, K, symmetric)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def reference_ms(pred, gt, model, symmetric, reps=3):
    def run():
        out = []
        for i in range(B):
            mp = np.dot(model, pred[i][:, :3].T) + pred[i][:, 3]
            mt = np.dot(model, gt[i][:, :3].T) + gt[i][:, 3]
            if symmetric:
                idx = eo.ref_find_nearest_point_idx(mp[None].astype(np.float32), mt[None].astype(np.float32))[0]
                add = np.mean(np.linalg.norm(mp[idx] - mt, 2, 1))
            else:
                add = np.mean(np.linalg.norm(mp - mt, axis=-1))
            p2 = [np.matmul(np.matmul(model, P[:, :3].T) + P[:, 3:].T, K.T) for P in (pred[i], gt[i])]
            proj = np.mean(np.linalg.norm(p2[0][:, :2] / p2[0][:, 2:] - p2[1][:, :2] / p2[1][:, 2:], axis=-1))
            out.append((add, proj))
        return out
    run()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        run()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main():
    name, power, clock_mhz = gpu_info()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bound = sms * 128 * clock_mhz * 1e6 / 8.0
    rows = []
    for n in SIZES:
        pred, gt, model = inputs(n)
        pp, pg, m = (torch.from_numpy(x).cuda() for x in (pred, gt, model))
        row = {"n": n, "add_ms": device_ms(pp, pg, m, False), "adds_ms": device_ms(pp, pg, m, True)}
        row["adds_pair_tests_per_s"] = B * n * n / (row["adds_ms"] * 1e-3)
        row["adds_fraction_of_fp32_issue_bound"] = row["adds_pair_tests_per_s"] / bound
        if eo.ref_nn_available():
            row["ref_add_ms"] = reference_ms(pred, gt, model, False)
            row["ref_adds_ms"] = reference_ms(pred, gt, model, True, reps=1 if n > 8192 else 3)
        rows.append(row)
    print(json.dumps({"bench": "eval_metrics", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock_mhz,
                      "sms": sms, "batch": B, "reps": REPS, "fp32_issue_bound_pairs_per_s": bound, "rows": rows}))


if __name__ == "__main__":
    main()
