"""Experiment: does the voting layer of batch i (FP32-issue bound, CUDA cores) overlap with the backbone of batch
i+1 (tensor-core bound) when they run on two streams?  Config 4's per-GPU workload, 30 batches of 16.
Prints sequential vs two-stream throughput.  OVL_STEPS sets the number of timed steps, OVL_COV=0 drops the
covariance layer."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402


def main():
    dev = torch.device("cuda", 0)
    net = bench.build_model(torch, dev)
    xs = [torch.from_numpy(syn.backbone_input(bench.BATCH, 2000 + i)).to(dev) for i in range(3)]
    bench.calibrate_foreground(torch, net, xs[0])
    n = int(os.environ.get("OVL_STEPS", "30"))
    with_cov = os.environ.get("OVL_COV", "1") == "1"

    from pvnet_b200 import _native
    L = _native.lib()
    names = [L.pvnet_backbone_stage_name(i).decode() for i in range(L.pvnet_backbone_num_stages())]
    split = names.index("layer2.0.conv1 (s2)")           # stages before: packing, stem, pool, layer1 (column kernels, whole SM)
    tail = names.index("upsample 1/8->1/4")               # stages from here: decoder (column kernels again)

    def backbone(x):
        return net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, pixel_major=True)

    def new_out():
        return (torch.empty([bench.BATCH, 480, 640, 20], dtype=torch.float32, device=dev),
                torch.empty([bench.BATCH, 480, 640], dtype=torch.uint8, device=dev))

    def vote(out, mask):
        vertex = out[..., 2:].unflatten(3, (9, 2))
        return rv.ransac_voting_pipeline(mask, vertex, 256, 0.99, with_cov, 256, 4096, 0.99, rng="device")

    res = {}
    with torch.no_grad():
        # sequential, one stream
        for i in range(5):
            vote(*backbone(xs[i % 3]))
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(n):
            vote(*backbone(xs[i % 3]))
        e1.record()
        torch.cuda.synchronize()
        res["sequential_ms_per_step"] = round(e0.elapsed_time(e1) / n, 4)

        for prio_name, pa, pb in (("backbone_high", -1, 0), ("equal", 0, 0), ("vote_high", 0, -1)):
            A, B = torch.cuda.Stream(priority=pa), torch.cuda.Stream(priority=pb)
            keep = []

            def run(count):
                evs_b = []
                for i in range(count):
                    with torch.cuda.stream(A):
                        if i >= 2:
                            A.wait_event(evs_b[i - 2])            # at most two batches in flight
                        out, mask = backbone(xs[i % 3])
                        ea = torch.cuda.Event()
                        ea.record(A)
                    with torch.cuda.stream(B):
                        B.wait_event(ea)
                        out.record_stream(B)
                        mask.record_stream(B)
                        r = vote(out, mask)
                        eb = torch.cuda.Event()
                        eb.record(B)
                        evs_b.append(eb)
                    keep.append((out, mask, r))
                    if len(keep) > 4:
                        keep.pop(0)
            run(5)
            torch.cuda.synchronize()
            f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f0.record()
            A.wait_event(f0)
            B.wait_event(f0)
            run(n)
            torch.cuda.current_stream().wait_stream(A)
            torch.cuda.current_stream().wait_stream(B)
            f1.record()
            torch.cuda.synchronize()
            res[f"two_streams_{prio_name}_ms_per_step"] = round(f0.elapsed_time(f1) / n, 4)
        # ---- staged: the vote of batch i-1 starts when batch i reaches the per-tap (tensor-bound, smaller smem) phase
        for prio_name, pa, pb in (("backbone_high", -1, 0), ("equal", 0, 0)):
            A, B = torch.cuda.Stream(priority=pa), torch.cuda.Stream(priority=pb)
            keep = []

            def run2(count):
                prev = None
                evs_b = []
                for i in range(count + 1):
                    cur = None
                    if i < count:
                        with torch.cuda.stream(A):
                            if i >= 2:
                                A.wait_event(evs_b[i - 2])
                            out, mask = new_out()
                            net.run_stages(xs[i % 3], out, mask, 0, split, pixel_major=True)
                            e_mid = torch.cuda.Event()
                            e_mid.record(A)
                        cur = (out, mask)
                    if prev is not None:                          # vote of the previous batch, released at the stage boundary
                        with torch.cuda.stream(B):
                            B.wait_event(prev[2])                 # its backbone is complete
                            if i < count:
                                B.wait_event(e_mid)               # and the next batch is past its column-kernel prologue
                            prev[0].record_stream(B)
                            prev[1].record_stream(B)
                            r = vote(prev[0], prev[1])
                            eb = torch.cuda.Event()
                            eb.record(B)
                            evs_b.append(eb)
                            keep.append((prev, r))
                    if i < count:
                        with torch.cuda.stream(A):
                            net.run_stages(xs[i % 3], cur[0], cur[1], split, len(names), pixel_major=True)
                            e_done = torch.cuda.Event()
                            e_done.record(A)
                        prev = (cur[0], cur[1], e_done)
                    if len(keep) > 4:
                        keep.pop(0)
            run2(5)
            torch.cuda.synchronize()
            f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f0.record()
            A.wait_event(f0)
            B.wait_event(f0)
            run2(n)
            torch.cuda.current_stream().wait_stream(A)
            torch.cuda.current_stream().wait_stream(B)
            f1.record()
            torch.cuda.synchronize()
            res[f"staged_{prio_name}_ms_per_step"] = round(f0.elapsed_time(f1) / n, 4)
    res["env"] = {"OVL_COV": os.environ.get("OVL_COV")}
    res["images_per_s_best"] = round(bench.BATCH / min(v for k, v in res.items() if k.endswith("_ms_per_step")) * 1e3, 1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
