"""Regenerates tests/golden/resnet18_8s_ref_{k9,k17}.npz from a checkout of the reference project:
    PVNET_REFERENCE=<path of the zju3dv/pvnet tree> python tests/golden/make_golden_backbone.py

Imports the REFERENCE network classes from <reference>/lib/networks/{resnet,
model_repository}.py (by file path, with `lib.utils.config` stubbed and the ImageNet
download at resnet.py:231 switched off), loads the deterministic weights of
tests/helpers.seeded_state_dict, runs Resnet18_8s(18,2).eval() on a seeded input on the
CPU (true fp32) and stores input + outputs.  The tests rebuild the same weights and check
that our module reproduces these outputs: the graph (dilation rules, decoder wiring,
align_corners upsampling, channel order of the concatenations) is pinned to the reference's.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.helpers import reference_root  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(reference_root(), "lib", "networks")


def load_reference_classes():
    saved = {k: sys.modules.get(k) for k in ("lib", "lib.utils", "lib.utils.config", "lib.networks",
                                             "lib.networks.resnet", "lib.networks.model_repository")}
    lib = types.ModuleType("lib"); lib.__path__ = []
    utils = types.ModuleType("lib.utils"); utils.__path__ = []
    cfgm = types.ModuleType("lib.utils.config"); cfgm.cfg = types.SimpleNamespace(MODEL_DIR="/tmp")
    nets = types.ModuleType("lib.networks"); nets.__path__ = []
    sys.modules.update({"lib": lib, "lib.utils": utils, "lib.utils.config": cfgm, "lib.networks": nets})

    def load(name, path):
        spec = importlib.util.spec_from_file_location(name, path)
        m = importlib.util.module_from_spec(spec)
        sys.modules[name] = m
        spec.loader.exec_module(m)
        return m

    r = load("lib.networks.resnet", os.path.join(REF, "resnet.py"))
    orig = r.resnet18
    r.resnet18 = lambda pretrained=False, **kw: orig(pretrained=False, **kw)   # no network here
    mr = load("lib.networks.model_repository", os.path.join(REF, "model_repository.py"))
    cls = mr.Resnet18_8s
    for k, v in saved.items():
        if v is None:
            sys.modules.pop(k, None)
        else:
            sys.modules[k] = v
    return cls


def main():
    cls = load_reference_classes()
    sys.path.insert(0, ROOT)
    from tests.helpers import BACKBONE_CASES, seeded_state_dict
    out = {}
    for tag, (ver, seg) in {"k9": (18, 2), "k17": (34, 2)}.items():
        h, w = BACKBONE_CASES[tag]
        net = cls(ver, seg)
        net.load_state_dict(seeded_state_dict(net, seed=1))
        net.eval()
        x = torch.from_numpy(np.random.default_rng(7).standard_normal((2, 3, h, w), dtype=np.float32))
        with torch.no_grad():
            s, v = net(x)
        # the input is not stored (tests.helpers.backbone_golden regenerates it): each file stays under 1 MB
        out[tag] = {"seg": s.numpy().copy(), "ver": v.numpy().copy()}
        np.savez_compressed(os.path.join(HERE, f"resnet18_8s_ref_{tag}.npz"), **out[tag])
    print({t: {k: v.shape for k, v in d.items()} for t, d in out.items()})


if __name__ == "__main__":
    main()
