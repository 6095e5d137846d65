"""Regenerates tests/golden/resnet50_8s_2o_ref.npz from a checkout of the reference project:
    PVNET_REFERENCE=<path of the zju3dv/pvnet tree> python tests/golden/make_golden_backbone_2o.py

Loads the REFERENCE Resnet50_8s_2o from <reference>/lib/networks/model_repository.py the way
make_golden_backbones.py does (`lib.utils.config` stubbed, no ImageNet download), loads the deterministic weights of
tests/helpers.seeded_state_dict(seed=1), runs Resnet50_8s_2o(18,2).eval() on the CPU (true fp32) on
tests.deep_backbones.deep_backbone_input() and stores seg, ver and the state-dict keys in order with their shapes
(the checkpoint format our class must load).
"""
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
    net = mr.Resnet50_8s_2o(18, 2)
    sd = net.state_dict()
    keys = np.array([k for k in sd])
    shapes = np.array([",".join(str(d) for d in t.shape) for t in sd.values()])
    net.load_state_dict(seeded_state_dict(net, seed=1))
    net.eval()
    with torch.no_grad():
        s, v = net(torch.from_numpy(deep_backbone_input()))
    path = os.path.join(HERE, "resnet50_8s_2o_ref.npz")
    np.savez_compressed(path, seg=s.numpy(), ver=v.numpy(), keys=keys, shapes=shapes)
    print("Resnet50_8s_2o", s.shape, v.shape, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
