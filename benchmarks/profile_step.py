"""The bench step (backbone + vote, batch 16) for ncu: model build, calibration and one
warm-up step happen BEFORE cudaProfilerStart, so run ncu with `--profile-from-start off`:

  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none \
      --csv --log-file out/launches.csv python benchmarks/profile_step.py 2
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    dev = torch.device("cuda", 0)
    net = bench.build_model(torch, dev)
    x = torch.from_numpy(syn.backbone_input(bench.BATCH, 2000)).to(dev)
    fg = bench.calibrate_foreground(torch, net, x)
    step = bench.make_step(torch, net)
    with torch.no_grad():
        step(x)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        for _ in range(steps):
            step(x)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
    print(f"profiled {steps} steps, {fg:.0f} foreground px/image")


if __name__ == "__main__":
    main()
