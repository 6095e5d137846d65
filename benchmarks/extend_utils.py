"""Farthest point sampling and binary mesh rasterisation on the device, one JSON line.

  - FPS (init_center mode) at pn in {10 k, 100 k, 1 M} x sn in {8, 64, 512} x b in {1, 13} clouds of N(0, 0.05) points:
    device time per call, the time per round (call time / sn), and whether the cloud stays on chip;
  - the reference's own single-threaded farthest_point_sampling_init_center (oracle/_ref/libpvnet_refextend.so,
    when present) on the host CPU for b = 1, where pn * sn <= 6.4e7;
  - rasterisation of projected sphere meshes of 10 k and 100 k triangles at 480 x 640, b = 16.
Device times are CUDA events around INNER back-to-back calls, warmed, median of REPS (>= 20) windows.  Indices of
every FPS shape with b = 1 and sn = 8 are checked against the C oracle first.
    python benchmarks/extend_utils.py > profiles/extend_utils_<gpu>.json
"""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import extend_oracle as eo  # noqa: E402
from pvnet_b200 import _native  # noqa: E402
from pvnet_b200 import extend_utils as eu  # noqa: E402
from tests import extend_cases as ec  # noqa: E402

REPS = max(20, int(os.environ.get("REPS", "21")))
INNER = int(os.environ.get("INNER", "3"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def device_ms(fn):
    for _ in range(3):
        fn()
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(INNER):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / INNER)
    times.sort()
    return times[len(times) // 2]


def host_ref_ms(pts, sn):
    times = []
    for _ in range(3):
        t0 = time.perf_counter()
        eo.ref_farthest_point_sampling(pts, sn)
        times.append((time.perf_counter() - t0) * 1e3)
    return sorted(times)[1]


def main():
    if not torch.cuda.is_available():
        raise SystemExit("extend_utils.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    name, power, clock = gpu_info()
    L = _native.lib()
    fps_rows = []
    for pn in (10_000, 100_000, 1_000_000):
        for b in (1, 13):
            clouds = (np.random.default_rng(pn + b).normal(size=(b, pn, 3)) * 0.05).astype(np.float32)
            d = torch.from_numpy(clouds).to(dev)
            need = ctypes.c_size_t()
            L.pvnet_farthest_point_sampling_workspace_bytes(b, pn, ctypes.byref(need))
            check = eu.farthest_point_sampling(d[:1], 8, True, return_indices=True).cpu().numpy()
            assert np.array_equal(check, eo.farthest_point_sampling(clouds[:1], 8)), (pn, b)
            for sn in (8, 64, 512):
                ms = device_ms(lambda: eu.farthest_point_sampling(d, sn, True, return_indices=True))
                row = {"pn": pn, "sn": sn, "b": b, "on_chip": need.value == 0, "ms": ms,
                       "us_per_round": ms * 1e3 / sn}
                if b == 1 and pn * sn <= 6.4e7 and eo.ref_available():
                    row["ref_host_ms"] = host_ref_ms(clouds[0], sn)
                fps_rows.append(row)
    raster_rows = []
    for case in ("sphere_10k", "sphere_100k"):
        tris, h, w = ec.raster_case(case)
        batch = np.stack([tris + np.float32(8 * i) for i in range(16)])
        d = torch.from_numpy(batch).to(dev)
        got = eu.mesh_binary_rasterization(d, h, w).cpu().numpy()
        assert np.array_equal(got, eo.mesh_binary_rasterization(batch, h, w)), case
        ms = device_ms(lambda: eu.mesh_binary_rasterization(d, h, w))
        raster_rows.append({"case": case, "triangles": int(tris.shape[0]), "b": 16, "h": h, "w": w, "ms": ms,
                            "covered_fraction": float(got.mean())})
    print(json.dumps({"bench": "extend_utils", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
                      "reps": REPS, "inner": INNER, "fps_mode": "init_center", "fps": fps_rows,
                      "raster": raster_rows}))


if __name__ == "__main__":
    main()
