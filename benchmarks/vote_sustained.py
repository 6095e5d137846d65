"""Is the vote kernel power-capped when it runs back to back?  The config-4 voting layer (16 images x ~20000 px,
K=9, 256 + 4096 hypotheses) repeated N times without pauses, nvidia-smi clocks and power sampled beside it;
then the same calls with a 20 ms idle gap after each.  One JSON line per mode."""
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvnet_b200 import ransac_voting_gpu as rv  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402


class Smi:
    def __init__(self):
        self.rows = []
        self.proc = subprocess.Popen(["nvidia-smi", "--id=0", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits",
                                      "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        threading.Thread(target=self._rd, daemon=True).start()

    def _rd(self):
        for line in self.proc.stdout:
            try:
                a, b = line.split(",")
                self.rows.append((time.time(), float(a), float(b)))
            except ValueError:
                pass

    def window(self, t0, t1):
        r = [x for x in self.rows if t0 <= x[0] <= t1]
        if not r:
            return None, None
        return float(np.median([x[1] for x in r])), float(np.median([x[2] for x in r]))


def main():
    dev = "cuda:0"
    K, b, n = 9, 16, 20000
    field_kind = os.environ.get("SUST_FIELD", "planted")
    mask_np = syn.disc_mask(n)
    if field_kind == "planted":
        field = syn.planted_field(mask_np, K, 3, sigma=0.05)[0]
    else:
        field = syn.random_field(mask_np, K, 5)
    mask = torch.from_numpy(np.stack([mask_np] * b)).to(dev).to(torch.uint8)
    ver = torch.from_numpy(np.stack([field] * b)).to(dev)
    vertex = ver.permute(0, 2, 3, 1).view(b, 480, 640, K, 2)
    smi = Smi()
    call = lambda: rv.ransac_voting_pipeline(mask, vertex, 256, 0.99, True, 256, 4096, 0.99, rng="device")
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    tests = b * n * K * (256 + 4096)
    modes = (("burst, 20 ms idle after each call", 0.02, 40), ("back to back", 0.0, 150))
    if os.environ.get("SUST_SKIP_BURST"):
        modes = modes[1:]
    for mode, gap, reps in modes:
        evs = []
        w0 = time.time()
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            evs.append((e0, e1))
            if gap:
                torch.cuda.synchronize()
                time.sleep(gap)
        torch.cuda.synchronize()
        w1 = time.time()
        ms = np.array([a.elapsed_time(c) for a, c in evs])
        clk, pw = smi.window(w0 + 0.3 * (w1 - w0), w1)
        print(json.dumps(dict(mode=mode, field=field_kind,
                              ms_first5=round(float(np.median(ms[:5])), 4), ms_last_half=round(float(np.median(ms[reps // 2:])), 4),
                              gtests_per_s_last_half=round(tests / float(np.median(ms[reps // 2:])) / 1e6, 1),
                              sm_mhz=clk, power_w=pw, wall_s=round(w1 - w0, 2))), flush=True)
    smi.proc.terminate()


if __name__ == "__main__":
    main()
