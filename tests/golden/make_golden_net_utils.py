"""Regenerates tests/golden/ref_net_utils.npz by running the REFERENCE'S OWN smooth_l1_loss and
compute_precision_recall (lib/utils/net_utils.py:54-80, 329-348) on the CPU.

    PVNET_REFERENCE=<path> python tests/golden/make_golden_net_utils.py

The module is imported unmodified from the reference project.  Its module-level imports of tensorboardX, easydict
and torchvision (used only by its logging helpers) are satisfied by empty stand-ins in sys.modules.  The inputs are
rebuilt from seeds by tests/loss_cases.py, so the file holds only outputs: per case the elementwise loss of every
sigma (NaNs made canonical, as a sha256 digest: it is above 4 KB), the normalised per-image loss, precision and recall.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests.helpers import _pack, reference_root  # noqa: E402
from tests.loss_cases import CASES, canon_nan, case_inputs  # noqa: E402


def import_reference():
    ed = types.ModuleType("easydict")
    ed.EasyDict = dict
    tb = types.ModuleType("tensorboardX")
    tb.SummaryWriter = object
    tv = types.ModuleType("torchvision")
    tv.utils = types.ModuleType("torchvision.utils")
    sys.modules.update({"easydict": ed, "tensorboardX": tb, "torchvision": tv, "torchvision.utils": tv.utils})
    spec = importlib.util.spec_from_file_location("ref_net_utils",
                                                  os.path.join(reference_root(), "lib", "utils", "net_utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = import_reference()
    out = {}
    for name in CASES:
        seg, mask, pred, vertex, weights, sigma = case_inputs(name)
        p, t, w = (torch.from_numpy(a) for a in (pred, vertex, weights))
        el = ref.smooth_l1_loss(p, t, w, sigma=sigma, normalize=False, reduce=False)
        norm = ref.smooth_l1_loss(p, t, w, sigma=sigma, normalize=True, reduce=True)
        prec, rec = ref.compute_precision_recall(torch.from_numpy(seg), torch.from_numpy(mask))
        out[f"{name}/elem"] = _pack(canon_nan(el))
        out[f"{name}/norm"] = norm.numpy()
        out[f"{name}/precision"] = prec.numpy()
        out[f"{name}/recall"] = rec.numpy()
        print(name, norm.numpy(), prec.numpy(), rec.numpy())
    np.savez_compressed(os.path.join(HERE, "ref_net_utils.npz"), **out)
    print("wrote ref_net_utils.npz", len(out), "arrays")


if __name__ == "__main__":
    main()
