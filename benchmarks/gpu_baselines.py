"""GPU-vs-GPU baselines on the same GPU (BASELINE.md section 4): what the REFERENCE's own CUDA path costs for
the work bench.py times, next to ours, same inputs, CUDA events / synchronize brackets.

 (i)  voting: oracle/ref_cuda.layer_v3 (+ layer_cov_with_mean) = the reference's kernels (compiled verbatim
      into oracle/_ref) driven by the reference's torch ops in the reference's order, host syncs included
      (they are part of what the reference costs), on config 2 / config 4 shapes; and on config 3's corner.
 (ii) network: Resnet18_8s._forward_torch (the reference graph: nn.Conv2d / BatchNorm2d / ... on cuDNN) at
      batch 16, TF32 on (torch default: cudnn.allow_tf32) and strict fp32, NCHW and channels_last.
Prints one JSON line per measurement plus a summary line with the ratios.  Test infrastructure only: the
reference side imports oracle/.
"""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from oracle import ref_cuda  # noqa: E402
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402

DEV = torch.device("cuda", 0)


def timed(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def vote_inputs(b, n_fg, k, seed):
    masks, fields = [], []
    for i in range(b):
        m = syn.disc_mask(n_fg, center=(320 + 3 * (i % 5), 240 - 2 * (i % 7)))
        masks.append(m)
        fields.append(syn.random_field(m, k, seed + i))
    mask = torch.from_numpy(np.stack(masks)).to(DEV)
    ver = torch.from_numpy(np.stack(fields)).to(DEV)
    return mask, ver.permute(0, 2, 3, 1).view(b, 480, 640, k, 2)


def main():
    out = []
    have_ref = ref_cuda.available()
    # ---------------------------------------------------------------- (ii) backbone
    net = bench.build_model(torch, DEV)
    x = torch.from_numpy(syn.backbone_input(16, 5)).to(DEV)
    with torch.no_grad():
        ours_ms = timed(lambda: net.forward_native(x), 20, warm=5)
        row = {"what": "Resnet18_8s forward, batch 16, 480x640", "ours_native_ms": round(ours_ms, 3)}
        old_c, old_m = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        try:
            for tf32 in (True, False):
                for cl in (False, True):
                    torch.backends.cudnn.allow_tf32 = tf32
                    torch.backends.cuda.matmul.allow_tf32 = tf32
                    torch.backends.cudnn.benchmark = True
                    m = net.to(memory_format=torch.channels_last) if cl else net.to(memory_format=torch.contiguous_format)
                    xx = x.contiguous(memory_format=torch.channels_last) if cl else x
                    ms = timed(lambda: m._forward_torch(xx), 10, warm=4)
                    row[f"cudnn_{'tf32' if tf32 else 'fp32'}_{'channels_last' if cl else 'nchw'}_ms"] = round(ms, 3)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old_c, old_m
            net.to(memory_format=torch.contiguous_format)
        best_tf32 = min(v for k_, v in row.items() if k_.startswith("cudnn_tf32"))
        row["speedup_vs_best_cudnn_tf32"] = round(best_tf32 / ours_ms, 2)
        row["speedup_vs_best_cudnn_fp32"] = round(min(v for k_, v in row.items() if k_.startswith("cudnn_fp32")) / ours_ms, 2)
    out.append(row)
    print(json.dumps(row), flush=True)

    # ---------------------------------------------------------------- (i) voting layers
    for name, b, n_fg, k, hn, cov, max_num in (("config2", 16, 20000, 9, 256, None, 30000),
                                               ("config4", 16, 20000, 9, 256, (256, 4096), 30000),
                                               # 1024 hyp: the reference's int32 index into its [hn,K,tn] u8 tensor
                                               # overflows at 2048 x 9 x 150000 = 2.76e9 (illegal address)
                                               ("config3_150k_x_1024", 1, 150000, 9, 1024, None, 10 ** 9)):
        mask, vertex = vote_inputs(b, n_fg, k, 7)

        def ours():
            return rv.ransac_voting_pipeline(mask, vertex, hn, 0.99, cov is not None, cov[0] if cov else 256,
                                             cov[1] if cov else 4096, 0.99, max_num=max_num, rng="device")

        def ours_reference_api():      # the drop-in functions with the reference's RNG replay (one host sync)
            kp = rv.ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh=0.99, max_num=max_num)
            if cov:
                rv.estimate_voting_distribution_with_mean(mask, vertex, kp, cov[0], cov[1], inlier_thresh=0.99,
                                                          max_num=max_num)

        row = {"what": "voting layer", "shape": name, "batch": b, "fg_px": n_fg, "K": k, "hyp": hn, "cov": cov,
               "ours_fused_ms": round(timed(ours, 10), 3), "ours_reference_api_ms": round(timed(ours_reference_api, 5), 3)}
        if have_ref:
            def ref():
                kp = ref_cuda.layer_v3(mask, vertex, hn, inlier_thresh=0.99, max_num=max_num)
                if cov:
                    ref_cuda.layer_cov_with_mean(mask, vertex, kp, cov[0], cov[1], inlier_thresh=0.99, max_num=max_num)
            row["reference_cuda_ms"] = round(timed(ref, 3, warm=1), 3)
            row["speedup_vs_reference_cuda"] = round(row["reference_cuda_ms"] / row["ours_fused_ms"], 1)
        out.append(row)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
