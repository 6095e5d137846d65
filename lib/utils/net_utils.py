"""`lib.utils.net_utils` as tools/demo.py:6 and tools/train_linemod.py:19 import it: `smooth_l1_loss` and
`compute_precision_recall` served by pvnet_b200's device kernel (pvnet_b200/net_utils.py), plus `vertex_targets` and
`seg_vertex_losses_from_keypoints`, which build the loader's vertex targets on the device; the checkpoint,
learning-rate and logging helpers on the host.  Unlike the reference module, importing it loads neither tensorboardX,
easydict nor torchvision; `Recorder(rec=True)` imports tensorboardX when it is built."""
from pvnet_b200.net_utils import (AverageMeter, NetWrapper, Recorder, adjust_learning_rate,  # noqa: F401
                                  compute_precision_recall, load_model, save_model, seg_vertex_losses,
                                  seg_vertex_losses_from_keypoints, set_learning_rate, smooth_l1_loss,
                                  vertex_targets)

__all__ = ["AverageMeter", "Recorder", "smooth_l1_loss", "load_model", "save_model", "adjust_learning_rate",
           "compute_precision_recall", "set_learning_rate", "seg_vertex_losses", "NetWrapper",
           "vertex_targets", "seg_vertex_losses_from_keypoints"]
