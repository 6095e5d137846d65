"""Regenerates tests/golden/conv_tap_store.json: sha256 digests of what the per-tap convolution stores.

Run on an H100:  python tests/golden/make_golden_conv_tap_store.py [out.json]

The cases, their seeded inputs and the launch are those of tests/test_gpu_conv_tap_store.py, which requires the
same digests: for every Cout (one per N tile width), every shape (partial tiles in both directions included), every
activation, with and without TF32 rounding of the output and with and without a residual, the bytes of the
destination's channel slice.  The committed file was recorded with the register -> global epilogue, before the
epilogue was moved to shared-memory staging and TMA stores; a change to how the tile is stored must leave every
byte where it was.  Each case is also checked against its fp64 restatement before its digest is recorded.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "conv_tap_store.json")
    import torch

    from pvnet_b200 import conv as pc
    from tests import test_gpu_conv_tap_store as t

    # the fp64 restatement of the smallest case runs anywhere; the kernel does not
    pre = t.reference_fp64(*[v.cpu() for v in _cpu_inputs(t, pc, torch)])
    print("fp64 restatement of cout 32, 8x16:", tuple(pre.shape), "max |v| %.3f" % pre.abs().max().item())
    if not torch.cuda.is_available():
        raise RuntimeError("make_golden_conv_tap_store.py needs a CUDA device: the digests are of the kernel's output")

    cases = {}
    for cout in t.COUTS:
        for shape in t.SHAPES:
            x, w, bias, res_buf = t.make_inputs(cout, shape)
            wp = pc.pack_weight(w)
            pre = t.reference_fp64(x, w, bias)
            for act, rnd, with_res in t.VARIANTS:
                key = t.case_key(cout, shape, act, rnd, with_res)
                flat = t.run_case(x, wp, bias, res_buf, cout, act, rnd, with_res)
                got = flat[:x.shape[0] * x.shape[1] * x.shape[2], t.PAD_C:t.PAD_C + cout].reshape(pre.shape)
                ref = t.finish_fp64(pre, res_buf, cout, act, with_res)
                scale = max(ref.abs().max().item(), 1.0)
                err = (got.double() - ref).abs().max().item()
                if err > 2e-5 * scale + 1e-5 + (scale * 2.0 ** -11 if rnd else 0.0):
                    raise RuntimeError(f"{key}: max err {err:.3e} against fp64, not recording it")
                cases[key] = t.digest(flat, cout)
                print(key, cases[key][:16])
    doc = dict(gpu=torch.cuda.get_device_name(0), sms=torch.cuda.get_device_properties(0).multi_processor_count,
               cases=cases)
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path, len(cases), "cases")


def _cpu_inputs(t, pc, torch):
    """x, w, bias of a one-tile case built on the CPU with the test's generator recipe (values only matter to the
    device-free rehearsal of the fp64 restatement)."""
    g = torch.Generator(device="cpu").manual_seed(1)
    x = torch.randn(1, 8, 16, t.CIN, generator=g)
    x = ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    w = torch.randn(32, t.CIN, t.KSIZE, t.KSIZE, generator=g) / 24.0
    return x, w, torch.randn(32, generator=g)


if __name__ == "__main__":
    main()
