"""Regenerates tests/golden/head_store.json: sha256 digests of what the native backbone's fused convraw.0 head writes.

Run on an H100:  python tests/golden/make_golden_head_store.py [out.json]

For every shape (partial tile rows and columns included), both output layouts (NCHW and pixel-major) and both
mask dtypes, `forward_native(x, with_mask=True)` runs on seeded weights and a seeded input, and the digests of
the output tensor's and the mask's bytes are recorded.  tests/test_gpu_head_store.py requires the same digests,
so a change to how the head's output is stored must leave every byte where it was.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pvnet_b200.model_repository import Resnet18_8s  # noqa: E402
from tests.helpers import seeded_state_dict  # noqa: E402

WEIGHT_SEED = 23
SHAPES = [(2, 480, 640), (1, 72, 104), (3, 16, 16), (1, 256, 264)]
MASK_DTYPES = {"uint8": torch.uint8, "int64": torch.int64}


def make_net(dev="cuda:0"):
    net = Resnet18_8s(18, 2)
    net.load_state_dict(seeded_state_dict(net, seed=WEIGHT_SEED))
    return net.to(dev).eval()


def make_input(shape, dev="cuda:0"):
    b, h, w = shape
    seed = b * 100003 + h * 1009 + w
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((b, 3, h, w), dtype=np.float32)).to(dev)


def digests(net, x, pixel_major, mask_dtype):
    """sha256 of forward_native's output and mask bytes"""
    with torch.no_grad():
        out, mask = net.forward_native(x, with_mask=True, mask_dtype=MASK_DTYPES[mask_dtype], pixel_major=pixel_major)
    torch.cuda.synchronize()
    return (hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest(),
            hashlib.sha256(mask.cpu().numpy().tobytes()).hexdigest())


def cases():
    for shape in SHAPES:
        for pixel_major in (False, True):
            for mask_dtype in MASK_DTYPES:
                yield shape, pixel_major, mask_dtype


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "head_store.json")
    net = make_net()
    rows = []
    for shape, pixel_major, mask_dtype in cases():
        out_sha, mask_sha = digests(net, make_input(shape), pixel_major, mask_dtype)
        rows.append(dict(shape=list(shape), pixel_major=pixel_major, mask_dtype=mask_dtype, out_sha256=out_sha,
                         mask_sha256=mask_sha))
        print(shape, "pixel-major" if pixel_major else "nchw", mask_dtype, out_sha[:16], mask_sha[:16])
    doc = dict(gpu=torch.cuda.get_device_name(0), weight_seed=WEIGHT_SEED, cases=rows)
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
