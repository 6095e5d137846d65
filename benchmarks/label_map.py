"""Label maps on the device (`pvnet_b200.render.render_label_map`, csrc/render.cu) by CUDA events: nine icospheres of
20 480 or 81 920 faces each at overlapping LINEMOD-like poses (tests/label_map_cases.py), 480x640, b = 1, 16, 64,
per-image K, some slots absent.  Next to it, the same maps as nine `render_mesh` calls plus a compositing pass in
torch (stack, divide, mask, argmin: the design that keeps one depth map per mesh), and the reference's path per
image -- `get_mask_of_all_objects`' loop over the `lib.utils.opengl_render_backend` drop-in, nine renders with a
mesh upload and a depth-map download each and numpy compositing -- by host clock, with `masks_of_all_objects` on the
same dataset object beside it.  Appends one JSON line per measurement to profiles/label_map_h100_<power>w.jsonl (or
--out), with the card name and power limit read in the same run.

Derived numbers: `key_bytes` (b x h x w x 8, the one-pass workspace) against `depth_map_bytes` (M x b x h x w x 4, the
nine depth maps the alternative keeps), and the peak device memory each call allocates."""
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

from pvnet_b200 import render as pr  # noqa: E402
from tests import label_map_cases as lc  # noqa: E402

H, W = 480, 640
NEAR, FAR, DIV, MAXD = 10.0, 10000.0, 1000.0, 10.0


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


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--ref-images", type=int, default=8)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(", ")
    card, power = q[0], float(q[1])
    out = args.out or os.path.join(ROOT, "profiles", f"label_map_h100_{int(round(power))}w.jsonl")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    dev = "cuda:0"
    recs = []

    def emit(r):
        r = {"card": card, "power_limit_w": power, "h": H, "w": W, "M": 9, **r}
        recs.append(r)
        print(json.dumps(r), flush=True)

    for subdiv in (5, 6):
        for b in (1, 16, 64):
            meshes, labels, P, K, present = lc.scene(b, np.random.default_rng(b), subdiv=subdiv)
            ms = pr.MeshSet(meshes, labels, device=dev)
            Pd, Kd = torch.from_numpy(P).to(dev), torch.from_numpy(np.ascontiguousarray(K)).to(dev)
            prd = torch.from_numpy(present).to(dev)
            vd = [torch.from_numpy(v).to(dev) for v, _ in meshes]
            fd = [torch.from_numpy(f).to(dev) for _, f in meshes]
            lab = torch.tensor(labels, dtype=torch.uint8, device=dev)
            absent = (prd == 0).T[:, :, None, None]

            def one_pass():
                return pr.render_label_map(ms, Pd, Kd, H, W, NEAR, FAR, present=prd, depth_divisor=DIV,
                                           max_depth=MAXD)

            def nine_calls():
                d = torch.stack([pr.render_mesh(vd[m], fd[m], Kd, Pd[:, m], H, W, NEAR, FAR) for m in range(9)])
                d = d / DIV
                d = torch.where((d == 0) | absent | (d >= MAXD), torch.inf, d)
                best, slot = d.min(0)                           # the first minimum: the lower slot
                return torch.where(torch.isinf(best), 0, lab[slot]), best

            label, _ = one_pass()
            agree = float((nine_calls()[0] == label).float().mean())
            t1 = device_ms(one_pass, args.iters)
            t9 = device_ms(nine_calls, args.iters)
            emit({"faces_per_mesh": len(meshes[0][1]), "b": b, "render_label_map_ms": t1,
                  "nine_render_mesh_plus_composite_ms": t9, "speedup": t9 / t1,
                  "render_label_map_peak_bytes": peak_bytes(one_pass),
                  "nine_render_mesh_plus_composite_peak_bytes": peak_bytes(nine_calls),
                  "key_bytes": b * H * W * 8, "depth_map_bytes": 9 * b * H * W * 4,
                  "labelled_fraction": float((label > 0).float().mean()), "composite_label_agreement": agree})
            del ms, vd, fd

    # the reference's loop per image on the drop-in, and the batched call on the same dataset object
    for subdiv in (5, 6):
        n = args.ref_images
        db = lc.fake_db(range(n), np.random.default_rng(1), subdiv=subdiv)
        lc.reference_loop(db, 0)
        pr.masks_of_all_objects(db, [0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        want = np.stack([lc.reference_loop(db, i) for i in range(n)])
        t_ref = (time.perf_counter() - t0) / n * 1e3
        t0 = time.perf_counter()
        got = pr.masks_of_all_objects(db, range(n))
        t_batch = (time.perf_counter() - t0) / n * 1e3
        t0 = time.perf_counter()
        for i in range(n):
            pr.get_mask_of_all_objects(db, i)
        t_single = (time.perf_counter() - t0) / n * 1e3
        emit({"faces_per_mesh": 20 * 4 ** subdiv, "images": n, "reference_loop_on_dropin_host_ms_per_image": t_ref,
              "masks_of_all_objects_host_ms_per_image": t_batch, "get_mask_of_all_objects_host_ms_per_image": t_single,
              "maps_equal": bool(np.array_equal(got, want))})

    with open(out, "a") as fh:
        for r in recs:
            fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
