"""One Resnet18_8s training step three ways, and where its convolution time goes; one JSON line.

480 x 640, K = 9 (ver_dim 18), seg_dim 2, batch 16 and 32 (the reference config's train_batch_size).  A step is
forward, seg_vertex_training_losses_from_keypoints, mean(loss_seg) + mean(loss_vertex), backward() and an Adam step
(the reference's optimizer, lr 1e-3).  Three models with the same initial weights:
  torch_nchw          `net(x)` in train mode: today's PyTorch/cuDNN graph (TF32 convolutions, torch's default);
  torch_channels_last the same graph on a channels_last model and image (the fair layout baseline);
  forward_train       `net.forward_train(x)`: the 24 trunk/decoder convolutions on the native kernels.
The three alternate step by step in one run; each row is the median of STEPS steps after WARM warm-up rounds (CUDA
events around the step), and the peak of the memory allocated during one step above what was allocated before it.

Then, at the largest batch, per layer (the 24 convolutions of slots 1..24 at their 480 x 640 shapes, channels_last
operands): forward, data gradient and weight gradient, native (CUDA events around pvnet_conv2d_nhwc, zero insertion +
pvnet_conv2d_nhwc with the flipped pack, pvnet_conv2d_nhwc_wgrad + its reduction) against cuDNN (F.conv2d and
aten.convolution_backward on the channels_last input and weight, as the graph's ConvolutionBackward0 runs it, TF32), as ms and TFLOP/s of the layer's 2*Cout*Cin*k*k*Ho*Wo*b FLOPs
(the useful ones: zero insertion's extra multiplications by zero are not counted) against 495 TFLOP/s dense TF32
(H100 SXM data sheet).  And a torch.profiler run of one step of each model at that batch, its CUDA kernel time
grouped per layer into convolution forward / data gradient / weight gradient, and elementwise and other kernels.
    python benchmarks/train_step.py > profiles/train_step_<gpu>_<power>.json
"""
import copy
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from pvnet_b200 import conv as pc  # noqa: E402
from pvnet_b200 import net_utils as nu  # noqa: E402
from pvnet_b200 import synthetic as syn  # noqa: E402
from pvnet_b200.model_repository import _SLOTS, Resnet18_8s  # noqa: E402
from torch.profiler import ProfilerActivity, profile, record_function  # noqa: E402

H, W, K, C, NFG = 480, 640, 9, 2, 20000
VD = 2 * K
BATCHES = tuple(int(b) for b in os.environ.get("BATCHES", "16,32").split(","))
STEPS = int(os.environ.get("STEPS", "10"))
WARM = int(os.environ.get("WARM", "2"))
REPS = int(os.environ.get("REPS", "10"))
TF32_PEAK = 495e12


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return name, power, float(clock.split()[0])
    except Exception:
        return torch.cuda.get_device_name(0), "unknown", float("nan")


def inputs(b, dev, seed=0):
    rng = np.random.default_rng(seed)
    masks = [syn.disc_mask(NFG, center=(320 + int(rng.integers(-40, 41)), 240 + int(rng.integers(-40, 41))))
             for _ in range(b)]
    hc = np.concatenate([rng.uniform([0, 0], [W, H], (b, K, 2)), np.ones((b, K, 1))], 2)
    mask = torch.from_numpy(np.stack(masks)).to(dev)
    x = torch.randn(b, 3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
    return x, mask, torch.from_numpy(hc).to(dev), mask[:, None].float()


def models(dev):
    torch.manual_seed(0)
    base = Resnet18_8s(ver_dim=VD, seg_dim=C).to(dev).train()
    cl = copy.deepcopy(base).to(memory_format=torch.channels_last)
    nat = copy.deepcopy(base)
    forms = {"torch_nchw": (base, lambda m, x: m(x), lambda x: x),
             "torch_channels_last": (cl, lambda m, x: m(x), lambda x: x.contiguous(memory_format=torch.channels_last)),
             "forward_train": (nat, lambda m, x: m.forward_train(x), lambda x: x)}
    return {k: (m, fwd, prep, torch.optim.Adam(m.parameters(), lr=1e-3)) for k, (m, fwd, prep) in forms.items()}


def make_step(form, x, mask, hc, wgt):
    m, fwd, prep, opt = form
    xi = prep(x)

    def step():
        seg, ver = fwd(m, xi)
        ls, lv, _, _ = nu.seg_vertex_training_losses_from_keypoints(seg, ver, mask, hc, wgt)
        loss = torch.mean(ls) + torch.mean(lv)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return step


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def step_rows(b, dev):
    forms = models(dev)
    x, mask, hc, wgt = inputs(b, dev, seed=1)
    steps = {k: make_step(f, x, mask, hc, wgt) for k, f in forms.items()}
    for _ in range(WARM):
        for fn in steps.values():
            fn()
    times = {k: [] for k in steps}
    for _ in range(STEPS):
        for name, fn in steps.items():
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            e.record()
            e.synchronize()
            times[name].append(a.elapsed_time(e))
    res = {}
    for name, fn in steps.items():
        t = sorted(times[name])
        res[name] = {"step_ms": t[len(t) // 2], "step_ms_min": t[0], "step_ms_max": t[-1], "step_peak_mb": peak_mb(fn)}
    return res, steps, forms


CONV_KERNEL_KEYS = ("fprop", "dgrad", "wgrad", "k_conv_", "k_zero_insert", "implicit_convolve", "implicit_gemm",
                    "convolve", "conv2d")


def is_conv_kernel(name):
    return any(k in name.lower() for k in CONV_KERNEL_KEYS)


def layer_names(net):
    """conv module -> its state-dict name, for all 26 convolutions (stem and head included)."""
    return {m: n for n, m in net.named_modules() if isinstance(m, torch.nn.Conv2d)}


def profile_rows(steps, forms):
    """One profiled step of each form.  Every convolution runs inside a `layer::<name>` range (module hooks for the
    torch graphs, a wrapper of conv2d_train for forward_train); its autograd node carries the forward op's sequence
    number, which attributes the backward's kernels to the same layer.  Kernels are grouped per layer into fwd /
    dgrad / wgrad (by kernel name for cuDNN, by forward or backward range for the native kernels, whose data gradient
    is a forward-convolution kernel) and, outside the convolutions, into elementwise (BatchNorm, activations, pool,
    upsampling, cat, losses, optimizer, layout conversions)."""
    out = {}
    for name, fn in steps.items():
        net = forms[name][0]
        names = layer_names(net)
        by_weight = {id(m.weight): n for m, n in names.items()}
        open_ranges, hooks = {}, []

        def pre(m, _inp):
            r = record_function(f"layer::{names[m]}")
            r.__enter__()
            open_ranges[m] = r

        def post(m, _inp, _out):
            open_ranges.pop(m).__exit__(None, None, None)
        for m in names:
            hooks += [m.register_forward_pre_hook(pre), m.register_forward_hook(post)]
        orig = pc.conv2d_train

        def wrapped(x, weight, *a, **k):
            with record_function(f"layer::{by_weight[id(weight)]}"):
                return orig(x, weight, *a, **k)
        pc.conv2d_train = wrapped
        try:
            fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
        finally:
            pc.conv2d_train = orig
            for h in hooks:
                h.remove()
        events = prof.events()

        def ancestors(e):
            while e is not None:
                yield e
                e = e.cpu_parent
        seq_layer = {}
        for e in events:
            if e.sequence_nr >= 0:
                for a in ancestors(e):
                    if a.name.startswith("layer::"):
                        seq_layer[e.sequence_nr] = a.name[len("layer::"):]
                        break
        layers, kinds = {}, {}
        for e in events:
            for kern in getattr(e, "kernels", []):
                ms = kern.duration / 1e3
                layer, bwd = None, False
                for a in ancestors(e):
                    if a.name.startswith("layer::"):
                        layer = a.name[len("layer::"):]
                        break
                    if "Backward" in a.name and a.sequence_nr in seq_layer:
                        layer, bwd = seq_layer[a.sequence_nr], True
                        break
                kname = kern.name.lower()
                if layer is None or not is_conv_kernel(kname):
                    k = "elementwise_and_other"
                elif "wgrad" in kname:
                    k = "wgrad"
                elif "dgrad" in kname or bwd:
                    k = "dgrad"
                else:
                    k = "fwd"
                kinds[k] = kinds.get(k, 0.0) + ms
                if k != "elementwise_and_other":
                    row = layers.setdefault(layer, {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0})
                    row[k] += ms
        # cross-check: every CUDA kernel of the step, however launched, by the profiler's own averages
        total = sum(ev.self_device_time_total for ev in prof.key_averages()) / 1e3
        out[name] = {"ms_by_kind": kinds, "ms_by_layer": layers, "kernel_ms_total": total}
    return out


def events_ms(fn, reps=REPS):
    fn()
    fn()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(a.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def conv_table(dev):
    """(name, Cin, Cout, k, stride, dilation, output (H, W), buffer channels, data-gradient channels) of slots 1..24,
    read from the modules and from one batch-1 480 x 640 pass of the torch graph."""
    net = Resnet18_8s(ver_dim=VD, seg_dim=C).to(dev)
    mods = dict(net.named_modules())
    shapes, hooks = {}, []
    for conv_name, _ in _SLOTS[1:25]:
        hooks.append(mods[conv_name].register_forward_hook(
            lambda m, i, o, n=conv_name: shapes.__setitem__(n, tuple(o.shape[2:]))))
    with torch.no_grad():
        net._forward_torch(torch.zeros(1, 3, H, W, device=dev))
    for h in hooks:
        h.remove()
    rows = []
    for conv_name, _ in _SLOTS[1:25]:
        m = mods[conv_name]
        cin = m.in_channels
        # convraw.0 reads cat[fm, image, 5 zeros] and gives only fm a data gradient (Resnet18_8s.forward_train)
        cbuf, n = (cin + 5, cin - 3) if conv_name == "convraw.0" else (cin, cin)
        rows.append((conv_name.replace("resnet18_8s.", ""), cin, m.out_channels, m.kernel_size[0], m.stride[0],
                     m.dilation[0], shapes[conv_name], cbuf, n))
    return rows


def layer_rows(b, dev):
    rows = []
    g = torch.Generator(device=dev).manual_seed(2)
    cl = torch.channels_last
    for name, cin, cout, k, stride, dil, (ho, wo), cbuf, n in conv_table(dev):
        pad = dil * (k - 1) // 2
        x = torch.randn(b, cbuf, ho * stride, wo * stride, device=dev, generator=g).contiguous(memory_format=cl)
        dy = torch.randn(b, cout, ho, wo, device=dev, generator=g).contiguous(memory_format=cl)
        w = torch.randn(cout, cin, k, k, device=dev, generator=g) * 0.05
        # cuDNN's backward is timed as the channels_last graph's ConvolutionBackward0 calls it, with the real input
        # x: its layout is what selects channels_last (torch.nn.grad.conv2d_input passes a zero-stride stand-in
        # instead, which sends cuDNN to NCHW and converts dy)
        wbuf = F.pad(w, (0, 0, 0, 0, 0, cbuf - cin)).contiguous(memory_format=cl)
        xh, dyh = x.permute(0, 2, 3, 1), dy.permute(0, 2, 3, 1)
        wp, wd = pc.pack_weight(w, cin_pad=pc.cin_padded(cbuf)), pc.pack_dgrad_weight(w, n)
        zb, zn = torch.zeros(cout, device=dev), torch.zeros(n, device=dev)
        out = torch.empty(b, ho, wo, cout, device=dev)
        dxh = torch.empty(b, ho * stride, wo * stride, n, device=dev)

        def nat_fwd():
            pc.conv2d_nhwc(xh, 0, cbuf, wp, zb, out, 0, cout, k, stride, dil)

        def nat_dgrad():
            src = pc.zero_insert2x(dyh) if stride == 2 else dyh
            pc.conv2d_nhwc(src, 0, cout, wd, zn, dxh, 0, n, k, 1, dil)

        def nat_wgrad():
            src = pc.zero_insert2x(dyh) if stride == 2 else dyh
            pc.conv2d_nhwc_wgrad(xh, 0, cbuf, src, 0, cout, k, dil)

        def cud_fwd():
            return F.conv2d(x, wbuf, stride=stride, padding=pad, dilation=dil)

        def cud_backward(mask):
            return torch.ops.aten.convolution_backward(dy, x, wbuf, None, [stride] * 2, [pad] * 2, [dil] * 2, False,
                                                       [0, 0], 1, mask)

        def cud_dgrad():
            return cud_backward([True, False, False])[0]

        def cud_wgrad():
            return cud_backward([False, True, False])[1]

        assert cud_fwd().is_contiguous(memory_format=cl) or k == 1
        assert cud_dgrad().is_contiguous(memory_format=cl)
        flops = 2.0 * cout * cin * k * k * ho * wo * b
        row = {"layer": name, "cin": cin, "cout": cout, "k": k, "stride": stride, "dilation": dil, "out_hw": [ho, wo],
               "gflop": flops / 1e9}
        for label, fn in (("native_fwd", nat_fwd), ("native_dgrad", nat_dgrad), ("native_wgrad", nat_wgrad),
                          ("cudnn_fwd", cud_fwd), ("cudnn_dgrad", cud_dgrad), ("cudnn_wgrad", cud_wgrad)):
            ms = events_ms(fn)
            row[label + "_ms"] = ms
            row[label + "_tflops"] = flops / (ms * 1e-3) / 1e12
        for part in ("fwd", "dgrad", "wgrad"):
            row[f"native_{part}_fraction_of_tf32_peak"] = row[f"native_{part}_tflops"] * 1e12 / TF32_PEAK
        rows.append(row)
        del x, dy, out, dxh
    tot = {k: sum(r[k] for r in rows) for k in rows[0] if k.endswith("_ms")}
    return rows, tot


def main():
    if not torch.cuda.is_available():
        raise SystemExit("train_step.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    name, power, clock = gpu_info()
    steps, prof = {}, None
    for b in BATCHES:
        steps[str(b)], fns, forms = step_rows(b, dev)
        if b == BATCHES[-1]:
            prof = profile_rows(fns, forms)
        del fns, forms
        torch.cuda.empty_cache()
    layers, totals = layer_rows(BATCHES[-1], dev)
    print(json.dumps({
        "bench": "train_step", "gpu": name, "power_limit": power, "max_sm_clock_mhz": clock,
        "h": H, "w": W, "keypoints": K, "seg_dim": C, "optimizer": "Adam(lr=1e-3)",
        "cudnn_allow_tf32": torch.backends.cudnn.allow_tf32, "steps": STEPS, "warm": WARM, "reps": REPS,
        "step": steps, "profile_batch": BATCHES[-1], "profile": prof,
        "layers_batch": BATCHES[-1], "layers": layers, "layer_totals_ms": totals}))


if __name__ == "__main__":
    main()
