"""A training step from the loader's batch in its two forms; one JSON line.

Every step copies its batch from the host, then runs forward_train, the keypoint training losses
(seg_vertex_training_losses_from_keypoints, K = 9), backward() and Adam.  Three forms, each on its own copy of one
seeded network:
  (a) loader    the reference loader's tensors, pageable: the float32 [b,3,H,W] image after ToTensor + Normalize, the
                int64 mask, the float32 [b,1,H,W] vertex weights, sent with `.cuda()` as train() does
                (tools/train_linemod.py:143); forward_train(image), losses with those weights;
  (b) compact   the uint8 [b,H,W,3] image and a uint8 mask, pageable, `.cuda()`; forward_train(u8, mean, std),
                losses with vertex_weights=None (the weights are the mask's values);
  (c) pinned    (b) from pinned host tensors with `.cuda(non_blocking=True)`.
The keypoints (float64 [b,9,3]) go with every form.  The vertex field is sent by none: the keypoint losses build it.
Per configuration: the host bytes copied per step; the median step time over STEPS steps with the forms alternated
step by step, each step timed by the host clock from its first copy to a device synchronise; the copies alone, timed
the same way; and a back-to-back loop of STEPS steps per form without a synchronise between steps (time per step).
The first step of (a) and (b) starts from the same weights: `first_step_equal` says whether their outputs and losses
agree bit for bit (the loader normalises on the CPU, (b) on the device).
    python benchmarks/train_input.py > profiles/train_input_<gpu>_<power>.json
"""
import copy
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402
from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402
from pvnet_b200.pipeline import IMAGENET_MEAN, IMAGENET_STD  # noqa: E402
from train_step import gpu_info  # noqa: E402

K = 9
CONFIGS = [tuple(int(v) for v in c.split("x")) for c in
           os.environ.get("CONFIGS", "16x480x640,32x480x640,32x256x320").split(",")]
STEPS = int(os.environ.get("STEPS", "10"))
WARM = int(os.environ.get("WARM", "2"))
FORMS = ("loader", "compact", "pinned")


def host_batch(b, H, W, seed=0):
    """The loader's batch on the host in both forms (the same pixels): uint8 image and mask, and the float forms
    derived from them on the CPU as the loader derives them."""
    rng = np.random.default_rng(seed)
    img = torch.from_numpy(rng.integers(0, 256, (b, H, W, 3), dtype=np.uint8))
    nfg = max(H * W // 15, 64)
    masks = [syn.disc_mask(nfg, center=(W // 2 + int(rng.integers(-W // 16, W // 16 + 1)),
                                        H // 2 + int(rng.integers(-H // 16, H // 16 + 1))), h=H, w=W)
             for _ in range(b)]
    mask8 = torch.from_numpy(np.stack(masks).astype(np.uint8))
    hc = torch.from_numpy(np.concatenate([rng.uniform([0, 0], [W, H], (b, K, 2)), np.ones((b, K, 1))], 2))
    mean = torch.tensor(IMAGENET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
    x = img.permute(0, 3, 1, 2).float().div(255).sub(mean).div(std).contiguous()     # ToTensor + Normalize
    mask64 = mask8.long()
    return {"loader": (x, mask64, mask64[:, None].float(), hc),
            "compact": (img, mask8, hc),
            "pinned": (img.pin_memory(), mask8.pin_memory(), hc.pin_memory())}


def make_step(form, net, opt, data):
    def copies():
        if form == "pinned":
            return [d.cuda(non_blocking=True) for d in data]
        return [d.cuda() for d in data]

    def step():
        d = copies()
        if form == "loader":
            x, mask, wgt, hc = d
            seg, ver = net.forward_train(x)
        else:
            x, mask, hc = d
            wgt = None
            seg, ver = net.forward_train(x, mean=IMAGENET_MEAN, std=IMAGENET_STD)
        ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
        opt.zero_grad(set_to_none=True)
        (ls.mean() + lv.mean()).backward()
        opt.step()
        return seg, ver, ls, lv
    return step, copies


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def first_step_equal(base, host, dev):
    outs = []
    for form in ("loader", "compact"):
        net = copy.deepcopy(base).to(dev)
        step, _ = make_step(form, net, torch.optim.Adam(net.parameters(), lr=1e-3), host[form])
        outs.append([t.detach() for t in step()])
    return all(torch.equal(u, v) for u, v in zip(*outs))


def config_row(b, H, W, dev):
    host = host_batch(b, H, W, seed=b + H)
    torch.manual_seed(0)
    base = Resnet18_8s(ver_dim=2 * K, seg_dim=2).train()
    same = first_step_equal(base, host, dev)
    steps, copies = {}, {}
    for form in FORMS:
        net = copy.deepcopy(base).to(dev)
        steps[form], copies[form] = make_step(form, net, torch.optim.Adam(net.parameters(), lr=1e-3), host[form])
    for _ in range(WARM):
        for form in FORMS:
            steps[form]()
    st = {f: [] for f in FORMS}
    h2d = {f: [] for f in FORMS}
    for _ in range(STEPS):
        for form in FORMS:
            st[form].append(host_ms(steps[form]))
        for form in FORMS:
            h2d[form].append(host_ms(copies[form]))
    loop = {}
    for form in FORMS:
        def run(form=form):
            for _ in range(STEPS):
                steps[form]()
        loop[form] = host_ms(run) / STEPS
    med = lambda v: float(np.median(v))  # noqa: E731
    return {"b": b, "H": H, "W": W, "first_step_equal": same,
            "forms": {f: {"bytes_per_step": int(sum(t.numel() * t.element_size() for t in host[f])),
                          "step_ms": med(st[f]), "step_ms_min": float(min(st[f])), "step_ms_max": float(max(st[f])),
                          "h2d_ms": med(h2d[f]),
                          "loop_ms_per_step": loop[f]} for f in FORMS}}


def main():
    if not torch.cuda.is_available():
        raise SystemExit("train_input.py measures on a GPU; none is available")
    dev = torch.device("cuda:0")
    name, power, clock = gpu_info()
    rows = [config_row(b, H, W, dev) for b, H, W in CONFIGS]
    print(json.dumps({"bench": "train_input", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
                      "steps": STEPS, "warmup": WARM, "rows": rows}))


if __name__ == "__main__":
    main()
