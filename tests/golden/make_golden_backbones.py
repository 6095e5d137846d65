"""Regenerates tests/golden/{resnet34_8s,resnet50_8s}_ref.npz and resnet_8s_ref_state_dicts.json from a checkout of
the reference project:
    PVNET_REFERENCE=<path of the zju3dv/pvnet tree> python tests/golden/make_golden_backbones.py

Imports the REFERENCE network classes from <reference>/lib/networks/{resnet,model_repository}.py (by file path, with
`lib.utils.config` stubbed and the ImageNet downloads of resnet34 / resnet50 switched off), loads the deterministic
weights of tests/helpers.seeded_state_dict, runs Resnet34_8s(18,2).eval() and Resnet50_8s(18,2).eval() on a seeded
input on the CPU (true fp32) and stores the outputs; the tests regenerate the input (tests.deep_backbones.deep_backbone_input).
The JSON holds each class's state-dict keys, in order, with their shapes: the checkpoint format our classes must load.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.helpers import reference_root  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(reference_root(), "lib", "networks")


def load_reference_module():
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
    for name in ("resnet18", "resnet34", "resnet50"):           # no network here
        orig = getattr(r, name)
        setattr(r, name, lambda pretrained=False, _orig=orig, **kw: _orig(pretrained=False, **kw))
    mr = load("lib.networks.model_repository", os.path.join(REF, "model_repository.py"))
    for k, v in saved.items():
        if v is None:
            sys.modules.pop(k, None)
        else:
            sys.modules[k] = v
    return mr


def main():
    mr = load_reference_module()
    from tests.deep_backbones import DEEP_BACKBONE_CLASSES, deep_backbone_input
    from tests.helpers import seeded_state_dict
    keys = {}
    for name in DEEP_BACKBONE_CLASSES:
        net = getattr(mr, name)(18, 2)
        keys[name] = [[k, list(t.shape)] for k, t in net.state_dict().items()]
        net.load_state_dict(seeded_state_dict(net, seed=1))
        net.eval()
        with torch.no_grad():
            s, v = net(torch.from_numpy(deep_backbone_input()))
        path = os.path.join(HERE, f"{name.lower()}_ref.npz")
        np.savez_compressed(path, seg=s.numpy(), ver=v.numpy())
        print(name, s.shape, v.shape, os.path.getsize(path), "bytes")
    with open(os.path.join(HERE, "resnet_8s_ref_state_dicts.json"), "w") as f:
        json.dump(keys, f, indent=0)


if __name__ == "__main__":
    main()
