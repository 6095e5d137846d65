"""Regenerates tests/golden/resnet18_8s_detectors_ref.npz and resnet18_8s_detectors_state_dicts.json from a checkout
of the reference project:
    PVNET_REFERENCE=<path of the zju3dv/pvnet tree> python tests/golden/make_golden_detectors.py

Loads the REFERENCE Resnet18_8s_detector and Resnet18_8s_detector_v2 from <reference>/lib/networks/model_repository.py
the way make_golden_backbones.py does (`lib.utils.config` stubbed, no ImageNet download), loads the deterministic
weights of tests/helpers.seeded_state_dict(seed=1) (for v2: its whole state dict, the base detector's included), runs
both in eval mode on the CPU (true fp32) on tests.deep_backbones.deep_backbone_input() and stores the score maps.
The JSON holds each class's state-dict keys, in order, with their shapes: the checkpoint format our classes must load.
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.golden.make_golden_backbones import HERE, load_reference_module  # noqa: E402


def main():
    mr = load_reference_module()
    from tests.deep_backbones import deep_backbone_input
    from tests.helpers import seeded_state_dict
    x = torch.from_numpy(deep_backbone_input())
    v1 = mr.Resnet18_8s_detector()
    v2 = mr.Resnet18_8s_detector_v2(mr.Resnet18_8s_detector())
    keys, outs = {}, {}
    for name, net in (("Resnet18_8s_detector", v1), ("Resnet18_8s_detector_v2", v2)):
        keys[name] = [[k, list(t.shape)] for k, t in net.state_dict().items()]
        net.load_state_dict(seeded_state_dict(net, seed=1))
        net.eval()
        with torch.no_grad():
            outs[name] = net(x).numpy()
        print(name, outs[name].shape)
    path = os.path.join(HERE, "resnet18_8s_detectors_ref.npz")
    np.savez_compressed(path, v1=outs["Resnet18_8s_detector"], v2=outs["Resnet18_8s_detector_v2"])
    print(path, os.path.getsize(path), "bytes")
    with open(os.path.join(HERE, "resnet18_8s_detectors_state_dicts.json"), "w") as f:
        json.dump(keys, f, indent=0)


if __name__ == "__main__":
    main()
