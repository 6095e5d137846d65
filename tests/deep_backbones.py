"""Shared pieces of the Resnet34_8s / Resnet50_8s tests: the golden outputs of the reference's classes
(tests/golden/make_golden_backbones.py) and their regenerated input."""
import os

import numpy as np

from tests.helpers import GOLDEN

DEEP_BACKBONE_CLASSES = ("Resnet34_8s", "Resnet50_8s")
DEEP_BACKBONE_SHAPE = (2, 3, 56, 80)                      # b, 3, H, W of tests/golden/resnet{34,50}_8s_ref.npz


def deep_backbone_input():
    """The input of tests/golden/make_golden_backbones.py (regenerated, not stored)."""
    return np.random.default_rng(11).standard_normal(DEEP_BACKBONE_SHAPE, dtype=np.float32)


def deep_backbone_golden(name):
    """(input, seg, ver) of the reference's `name` (Resnet34_8s / Resnet50_8s) with seeded_state_dict(seed=1)."""
    z = np.load(os.path.join(GOLDEN, f"{name.lower()}_ref.npz"))
    return deep_backbone_input(), z["seg"], z["ver"]
