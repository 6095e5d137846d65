"""The stem, max-pool and head of Resnet18_8s.forward_train on the native kernels against torch's; one JSON line.

Part one, per piece at batch 16 and 32, 480 x 640, on the same operands (channels_last for torch, as the torch graph
runs them): the native forward and backward against
  stem     cuDNN conv1 forward (F.conv2d, TF32) plus the copy of the image and its 5 zero channels into convraw.0's
           input, which the native stem writes in the same pass, and its weight gradient (aten.convolution_backward,
           weight only);
  max-pool F.max_pool2d (3, 2, 1) and its autograd backward;
  head     convraw.3 as F.conv2d(y, w, b).contiguous() and its autograd backward (input, weight and bias gradients).
CUDA events, WARM warm-up calls, REPS timed calls with the native and torch forms alternated, the median.  Shares
are computed from shapes: the stem's useful 2*64*147*Ho*Wo*b FLOPs against 495 TFLOP/s dense TF32, the max-pool's and
the head's compulsory bytes against 3.35 TB/s (H100 SXM data sheet).

Part two, a forward_train step (seg_vertex_training_losses_from_keypoints, backward(), Adam) at batch 16 and 32:
native against the same network with the three torch modules swapped back in for pc.stem_train / pc.maxpool_train /
pc.head_train, alternated step by step, with and without torch.use_deterministic_algorithms(True); median step time
and the peak memory allocated during a step.
    python benchmarks/stem_pool_head_train.py > profiles/stem_pool_head_train_<gpu>_<power>.json
"""
import copy
import json
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # deterministic cuBLAS, should a step use it

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))

from pvnet_b200 import conv as pc  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402
from bn_train import timed  # noqa: E402
from train_step import gpu_info, inputs, peak_mb  # noqa: E402

H, W, K = 480, 640, 9
BATCHES = tuple(int(b) for b in os.environ.get("BATCHES", "16,32").split(","))
REPS = int(os.environ.get("REPS", "20"))
WARM = int(os.environ.get("WARM", "3"))
STEPS = int(os.environ.get("STEPS", "10"))
HBM, TF32 = 3.35e12, 495e12
CL = torch.channels_last


def torch_stem(x, w, img, co, mean=None, std=None):
    """pc.stem_train of a float image in torch: cuDNN's conv1, and the image and 5 zero channels written into
    channels [co, co+8) of convraw.0's input img."""
    img[:, co:co + 3].copy_(x)
    img[:, co + 3:co + 8].zero_()
    return F.conv2d(x.contiguous(memory_format=CL), w, stride=2, padding=3)


def torch_maxpool(x):
    return F.max_pool2d(x, 3, 2, 1)


def torch_head(y, w, b):
    return F.conv2d(y, w, b).contiguous()


def piece_rows(b, dev):
    g = torch.Generator(device=dev).manual_seed(b)
    rows = []
    # stem
    x = torch.randn(b, 3, H, W, device=dev, generator=g)
    xc = x.contiguous(memory_format=CL)
    w = (0.1 * torch.randn(64, 3, 7, 7, device=dev, generator=g)).requires_grad_()
    dy = torch.randn(b, 64, H // 2, W // 2, device=dev, generator=g).contiguous(memory_format=CL)
    img = torch.empty(b, 8, H, W, device=dev, memory_format=CL)
    st = {"y": pc.stem_train(x, w, img, 0)}

    def stem_fwd():
        with torch.no_grad():
            pc.stem_train(x, w, img, 0)

    def cudnn_fwd():
        with torch.no_grad():
            torch_stem(xc, w, img, 0)

    def stem_wgrad():
        torch.autograd.grad(st["y"], w, dy, retain_graph=True)

    def cudnn_wgrad():
        torch.ops.aten.convolution_backward(dy, xc, w.detach(), None, [2, 2], [3, 3], [1, 1], False, [0, 0], 1,
                                            [False, True, False])

    for fn in (stem_fwd, cudnn_fwd, stem_wgrad, cudnn_wgrad):
        for _ in range(WARM):
            fn()
    t = timed({"native_fwd": stem_fwd, "torch_fwd": cudnn_fwd}, REPS)
    t.update(timed({"native_bwd": stem_wgrad, "torch_bwd": cudnn_wgrad}, REPS))
    flops = 2.0 * 64 * 147 * b * (H // 2) * (W // 2)
    row = {"piece": "stem conv1", "flops": flops, **{k + "_ms": v for k, v in t.items()}}
    for part in ("fwd", "bwd"):
        row[f"native_{part}_TFLOPs"] = flops / (row[f"native_{part}_ms"] * 1e-3) / 1e12
        row[f"native_{part}_fraction_of_tf32_peak"] = row[f"native_{part}_TFLOPs"] * 1e12 / TF32
    rows.append(row)
    del st, x, xc, dy, img
    torch.cuda.empty_cache()

    # max-pool
    C, h, w2 = 64, H // 2, W // 2
    xp = torch.relu(torch.randn(b, C, h, w2, device=dev, generator=g)).contiguous(memory_format=CL).requires_grad_()
    gp = torch.randn(b, C, h // 2, w2 // 2, device=dev, generator=g).contiguous(memory_format=CL)
    st = {"n": pc.maxpool_train(xp), "t": torch_maxpool(xp)}
    fns = {"native_fwd": lambda: pc.maxpool_train(xp), "torch_fwd": lambda: torch_maxpool(xp)}
    bws = {"native_bwd": lambda: torch.autograd.grad(st["n"], xp, gp, retain_graph=True),
           "torch_bwd": lambda: torch.autograd.grad(st["t"], xp, gp, retain_graph=True)}
    for fn in (*fns.values(), *bws.values()):
        for _ in range(WARM):
            fn()
    t = timed(fns, REPS)
    t.update(timed(bws, REPS))
    n_in, n_out = b * C * h * w2, b * C * (h // 2) * (w2 // 2)
    row = {"piece": "max-pool", "fwd_bytes": 4 * n_in + 5 * n_out, "bwd_bytes": 5 * n_out + 4 * n_in,
           **{k + "_ms": v for k, v in t.items()}}
    for part in ("fwd", "bwd"):
        row[f"native_{part}_fraction_of_hbm_peak"] = row[f"{part}_bytes"] / (row[f"native_{part}_ms"] * 1e-3) / HBM
    rows.append(row)
    del st, xp, gp
    torch.cuda.empty_cache()

    # head
    cin, cout = 32, 2 + 2 * K
    y = torch.randn(b, cin, H, W, device=dev, generator=g).contiguous(memory_format=CL).requires_grad_()
    wh = (0.2 * torch.randn(cout, cin, 1, 1, device=dev, generator=g)).requires_grad_()
    bh = torch.randn(cout, device=dev, generator=g).requires_grad_()
    gh = torch.randn(b, cout, H, W, device=dev, generator=g)
    st = {"n": pc.head_train(y, wh, bh), "t": torch_head(y, wh, bh)}
    fns = {"native_fwd": lambda: pc.head_train(y, wh, bh), "torch_fwd": lambda: torch_head(y, wh, bh)}
    bws = {"native_bwd": lambda: torch.autograd.grad(st["n"], (y, wh, bh), gh, retain_graph=True),
           "torch_bwd": lambda: torch.autograd.grad(st["t"], (y, wh, bh), gh, retain_graph=True)}
    for fn in (*fns.values(), *bws.values()):
        for _ in range(WARM):
            fn()
    t = timed(fns, REPS)
    t.update(timed(bws, REPS))
    P = b * H * W
    row = {"piece": "head convraw.3", "fwd_bytes": 4 * P * (cin + cout), "bwd_bytes": 4 * P * (2 * cin + cout),
           **{k + "_ms": v for k, v in t.items()}}
    for part in ("fwd", "bwd"):
        row[f"native_{part}_fraction_of_hbm_peak"] = row[f"{part}_bytes"] / (row[f"native_{part}_ms"] * 1e-3) / HBM
    rows.append(row)
    del st, y, gh
    torch.cuda.empty_cache()
    return rows


def step_rows(b, dev, deterministic):
    x, mask, hc, wgt = inputs(b, dev, seed=1)
    torch.manual_seed(0)
    base = Resnet18_8s(ver_dim=2 * K, seg_dim=2).to(dev).train()
    nets = {"native": base, "torch_modules": copy.deepcopy(base)}
    opts = {k: torch.optim.Adam(m.parameters(), lr=1e-3) for k, m in nets.items()}
    orig = pc.stem_train, pc.maxpool_train, pc.head_train

    def make(k):
        def step():
            if k == "torch_modules":
                pc.stem_train, pc.maxpool_train, pc.head_train = torch_stem, torch_maxpool, torch_head
            try:
                seg, ver = nets[k].forward_train(x)
            finally:
                pc.stem_train, pc.maxpool_train, pc.head_train = orig
            ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
            opts[k].zero_grad(set_to_none=True)
            (torch.mean(ls) + torch.mean(lv)).backward()
            opts[k].step()
        return step
    steps = {k: make(k) for k in nets}
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        for _ in range(WARM):
            for fn in steps.values():
                fn()
        t = timed(steps, STEPS)
        return {k: {"step_ms": t[k], "step_peak_mb": peak_mb(fn)} for k, fn in steps.items()}
    finally:
        torch.use_deterministic_algorithms(prev)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("stem_pool_head_train.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    name, power, clock = gpu_info()
    pieces, steps = {}, {}
    for b in BATCHES:
        pieces[str(b)] = piece_rows(b, dev)
    for b in BATCHES:
        for det in (False, True):
            steps[f"{b}{'_deterministic' if det else ''}"] = step_rows(b, dev, det)
            torch.cuda.empty_cache()
    print(json.dumps({"bench": "stem_pool_head_train", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
                      "h": H, "w": W, "reps": REPS, "warm": WARM, "steps": STEPS, "hbm_peak_Bps": HBM,
                      "tf32_peak_flops": TF32, "pieces": pieces, "forward_train_step": steps}))


if __name__ == "__main__":
    main()
