"""`lib.networks.model_repository` as tools/demo.py:5 and tools/train_linemod.py:10 import it
(`from lib.networks.model_repository import *`), served by pvnet_b200.  Resnet50_8s_2o is importable by name; `import *`
yields the three networks the reference's tools use."""
from pvnet_b200.model_repository import Resnet18_8s, Resnet34_8s, Resnet50_8s, Resnet50_8s_2o  # noqa: F401

__all__ = ["Resnet18_8s", "Resnet34_8s", "Resnet50_8s"]
