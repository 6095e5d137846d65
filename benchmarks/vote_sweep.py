"""BASELINE config 3: voting-only sweep on one GPU -- foreground pixel count x hypotheses,
K=9, max_num=10**9 (no subsampling).  Times pvnet_ransac_voting_v3 (whole layer: compaction
+ gather + hypotheses + vote + refit), with CUDA events on the launch
stream; prints one JSON line per point.  Inputs are flushed from L2 between iterations by
writing a 256 MB buffer."""
import json
import sys
import os

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402


def main():
    dev = "cuda:0"
    K = 9
    b = int(os.environ.get("SWEEP_BATCH", "4"))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    props = torch.cuda.get_device_properties(dev)
    sm_clock = props.clock_rate * 1e3 if hasattr(props, "clock_rate") else 1.98e9     # maximum SM clock, Hz
    sms = props.multi_processor_count
    pts = os.environ.get("SWEEP_POINTS")          # e.g. "10000:512,150000:2048"
    want = None if not pts else {(int(a), int(b_)) for a, b_ in (p.split(":") for p in pts.split(","))}
    for n in (1000, 10000, 50000, 150000):
        if want is not None and not any(n == a for a, _ in want):
            continue
        mask_np = syn.disc_mask(n)
        field = syn.planted_field(mask_np, K, 3)[0]
        mask = torch.from_numpy(np.stack([mask_np] * b)).to(dev)
        ver = torch.from_numpy(np.stack([field] * b)).to(dev)
        vertex = ver.permute(0, 2, 3, 1).view(b, 480, 640, K, 2)
        for hn in (128, 512, 2048):
            if want is not None and (n, hn) not in want:
                continue
            idxs = torch.from_numpy(np.stack([syn.draw_idxs(n, hn, K, seed=i) for i in range(b)])).to(dev)
            for _ in range(3):
                rv.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, max_num=10 ** 9, idxs=idxs)
            ts = []
            for _ in range(5):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                rv.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, max_num=10 ** 9, idxs=idxs)
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ms = float(np.median(ts))
            tests = (hn + 1) * K * n * b
            b_alg = b * (480 * 640 * 8 + n * K * 8 + hn * K * 8 + K * 24)
            print(json.dumps(dict(n_fg=n, hn=hn, batch=b, ms=round(ms, 4), images_per_s=round(b / ms * 1e3, 1),
                                  gtests_per_s=round(tests / ms / 1e6, 2),
                                  alg_GBps=round(b_alg / ms / 1e6, 2),
                                  issue_frac_at_8=round(tests * 8 / (sms * 128 * sm_clock) / (ms * 1e-3), 3))),
                  flush=True)


if __name__ == "__main__":
    main()
