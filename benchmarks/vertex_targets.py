"""The loader's ground-truth vertex field on the host against the device, and the validation losses computed from the
keypoints against the losses read from a materialised field, one JSON line.

Batch 16, 480 x 640, K = 9 (ver_dim 18), disc masks of 20 000 foreground pixels (int64), float64 keypoints (hw = 1):
  (a) host: per image the field formula of compute_vertex_hcoords (restated here with numpy) and
      torch.tensor(...).permute(2, 0, 1) as the loader does, then the batch stacked as the collate does, pinned and
      copied to the device; wall clock around a final synchronise, median of HOST_REPS batches;
  (b) vertex_targets on the device: time, and (field written + mask read) bytes over time against 3.35 TB/s;
  (c) seg_vertex_losses_from_keypoints against seg_vertex_losses on a materialised field (alone, and with the
      vertex_targets call that builds the field): time, compulsory bytes over time, and the peak of the memory
      allocated during one call.
Device times are CUDA events around INNER back-to-back calls, warmed, median of REPS.
    python benchmarks/vertex_targets.py > profiles/vertex_targets_<gpu>_<power>.json
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

from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402

B, H, W, K, C, NFG = 16, 480, 640, 9, 2, 20000
VD = 2 * K
REPS = int(os.environ.get("REPS", "30"))
INNER = int(os.environ.get("INNER", "10"))
HOST_REPS = int(os.environ.get("HOST_REPS", "7"))
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def host_field(mask, hcoords):
    """compute_vertex_hcoords' formula: [h,w,2K] float32."""
    h, w = mask.shape
    xy = np.argwhere(mask == 1)[:, [1, 0]]
    v = hcoords[None, :, :2] - xy[:, None, :] * hcoords[None, :, 2:]
    n = np.linalg.norm(v, axis=2, keepdims=True)
    n[n < 1e-3] += 1e-3
    v = v / n
    out = np.zeros([h, w, hcoords.shape[0], 2], np.float32)
    out[xy[:, 1], xy[:, 0]] = v
    return out.reshape(h, w, -1)


def host_batch_ms(masks, hcoords, dev):
    times = []
    for _ in range(HOST_REPS):
        t0 = time.perf_counter()
        vers = [torch.tensor(host_field(m, hc), dtype=torch.float32).permute(2, 0, 1) for m, hc in zip(masks, hcoords)]
        batch = torch.stack(vers).pin_memory().to(dev, non_blocking=True)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        del batch
    times.sort()
    return times[len(times) // 2]


def device_ms(fn, args):
    for _ in range(5):
        fn(*args)
    times = []
    for _ in range(REPS):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(INNER):
            fn(*args)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / INNER)
    times.sort()
    return times[len(times) // 2]


def peak_mb(fn, args):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn(*args)
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def main():
    if not torch.cuda.is_available():
        raise SystemExit("vertex_targets.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    rng = np.random.default_rng(0)
    masks = [syn.disc_mask(NFG, center=(320 + int(rng.integers(-40, 41)), 240 + int(rng.integers(-40, 41))))
             for _ in range(B)]
    hc = np.concatenate([rng.uniform([0, 0], [W, H], (B, K, 2)), np.ones((B, K, 1))], 2)
    mask = torch.from_numpy(np.stack(masks)).to(dev)
    hcoords = torch.from_numpy(hc).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    out = torch.randn(B, C + VD, H, W, device=dev, generator=g)
    seg, ver = out[:, :C], out[:, C:]
    weights = mask[:, None].float()
    name, power, clock = gpu_info()

    host_ms = host_batch_ms(masks, hc, dev)
    with torch.no_grad():
        field = nu.vertex_targets(mask, hcoords)
        host = torch.stack([torch.tensor(host_field(m, h)).permute(2, 0, 1) for m, h in zip(masks, hc)]).to(dev)
        field_equal = bool(torch.equal(field, host))
        del host
        kp_out = nu.seg_vertex_losses_from_keypoints(seg, ver, mask, hcoords, weights)
        mat_out = nu.seg_vertex_losses(seg, ver, mask, field, weights)
        losses_equal = all(a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() for a, b in zip(kp_out, mat_out))

        def materialised_end_to_end(seg, ver, mask, hcoords, weights):
            return nu.seg_vertex_losses(seg, ver, mask, nu.vertex_targets(mask, hcoords), weights)

        rows = {
            "vertex_targets": (nu.vertex_targets, (mask, hcoords)),
            "losses_from_keypoints": (nu.seg_vertex_losses_from_keypoints, (seg, ver, mask, hcoords, weights)),
            "losses_on_field": (nu.seg_vertex_losses, (seg, ver, mask, field, weights)),
            "vertex_targets_then_losses_on_field": (materialised_end_to_end, (seg, ver, mask, hcoords, weights)),
        }
        res = {k: {"ms": device_ms(fn, args), "peak_mb": peak_mb(fn, args)} for k, (fn, args) in rows.items()}
    npix = B * H * W
    bytes_ = {
        "vertex_targets": npix * (4 * VD + mask.element_size()),
        "losses_from_keypoints": npix * (4 * C + 4 * VD + 4 + mask.element_size()),
        "losses_on_field": npix * (4 * C + 8 * VD + 4 + mask.element_size()),
    }
    for k, v in bytes_.items():
        res[k]["compulsory_bytes"] = v
        res[k]["tb_per_s"] = v / (res[k]["ms"] * 1e-3) / 1e12
        res[k]["fraction_of_hbm_3_35_tb_s"] = v / (res[k]["ms"] * 1e-3) / HBM_BYTES_PER_S
    print(json.dumps({
        "bench": "vertex_targets", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
        "batch": B, "h": H, "w": W, "keypoints": K, "foreground_pixels": NFG, "mask_dtype": str(mask.dtype),
        "hcoords_dtype": str(hcoords.dtype), "reps": REPS, "inner": INNER, "host_reps": HOST_REPS,
        "host_cpu_threads": torch.get_num_threads(), "host_batch_ms": host_ms,
        "host_field_equals_device": field_equal, "keypoint_losses_equal_field_losses": losses_equal,
        "speedup_device_vs_host": host_ms / res["vertex_targets"]["ms"],
        "speedup_keypoints_vs_field": res["losses_on_field"]["ms"] / res["losses_from_keypoints"]["ms"],
        "rows": res}))


if __name__ == "__main__":
    main()
