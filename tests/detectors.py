"""Shared pieces of the Resnet18_8s_detector / Resnet18_8s_detector_v2 tests: the golden outputs of the reference's
classes (tests/golden/make_golden_detectors.py), seeded networks, the detector plans' workspace layout, and the score
head restated in fp64."""
import json
import os

import numpy as np
import torch
import torch.nn.functional as F

from pvnet_b200 import model_repository as mr
from tests.deep_backbones import deep_backbone_input
from tests.helpers import GOLDEN, seeded_state_dict

DETECTOR_CLASSES = ("Resnet18_8s_detector", "Resnet18_8s_detector_v2")


def detector(name, seed=1):
    """A seeded detector (v2 on a fresh base; the seed covers its whole state dict, the base's included)."""
    net = mr.Resnet18_8s_detector() if name == "Resnet18_8s_detector" else \
        mr.Resnet18_8s_detector_v2(mr.Resnet18_8s_detector())
    net.load_state_dict(seeded_state_dict(net, seed=seed))
    return net


def detector_golden(name):
    """(input, score map) of the reference's `name` with seeded_state_dict(seed=1)."""
    z = np.load(os.path.join(GOLDEN, "resnet18_8s_detectors_ref.npz"))
    return deep_backbone_input(), z["v1" if name == "Resnet18_8s_detector" else "v2"]


def detector_state_dict_shapes():
    with open(os.path.join(GOLDEN, "resnet18_8s_detectors_state_dicts.json")) as f:
        return json.load(f)


def detector_buffers(last_stage):
    """(level, channels) of the buffers pvnet_backbone_create_detector carves for the 2-2-2-2 BasicBlock trunk, in
    order: S, the stem's output, the max-pool's, then per stage A, (D,) B, E; the last is the score head's input."""
    bufs = [(1, 16), (1, 64), (2, 64)]
    for s in range(last_stage):
        c = 64 << s
        bufs += [(2 if s == 0 else 3, c)] * (3 if s == 0 else 4)
    return bufs


def buffer_offsets(bufs, b, h, w):
    """Byte offsets of the carved buffers (256-byte aligned, in order) and the total."""
    al = lambda n: (n + 255) // 256 * 256  # noqa: E731
    offs, off = [], 0
    for level, ch in bufs:
        offs.append(off)
        off = al(off + ((b * h * w) >> (2 * level)) * ch * 4)
    return offs, off


def head3x3_fp64(y_nchw, weight, bias):
    """The score head in fp64, and R = the same on absolute values plus |bias| (the scale of the fp32 chain's
    rounding error)."""
    y, wt, bt = y_nchw.double(), weight.detach().double(), bias.detach().double()
    return F.conv2d(y, wt, bt, padding=1), F.conv2d(y.abs(), wt.abs(), bt.abs(), padding=1)
