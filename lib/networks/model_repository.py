"""`lib.networks.model_repository` as tools/demo.py:5 and tools/train_linemod.py:10 import it
(`from lib.networks.model_repository import *`), served by pvnet_b200.  Resnet50_8s_2o, Resnet18_8s_detector and
Resnet18_8s_detector_v2 are importable by name; `import *` yields the three networks the reference's tools use."""
from pvnet_b200.model_repository import (Resnet18_8s, Resnet18_8s_detector, Resnet18_8s_detector_v2,  # noqa: F401
                                         Resnet34_8s, Resnet50_8s, Resnet50_8s_2o)

__all__ = ["Resnet18_8s", "Resnet34_8s", "Resnet50_8s"]
