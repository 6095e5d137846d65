"""`lib.ransac_voting_gpu_layer.ransac_voting_gpu` as tools/demo.py:8,121 and
tools/train_linemod.py:8-9 import it, served by pvnet_b200."""
from pvnet_b200.ransac_voting_gpu import (  # noqa: F401
    estimate_voting_distribution,
    estimate_voting_distribution_with_mean,
    generate_hypothesis,
    ransac_motion_voting,
    ransac_voting_center,
    ransac_voting_hypothesis,
    ransac_voting_labels,
    ransac_voting_layer,
    ransac_voting_layer_v2,
    ransac_voting_layer_v3,
    ransac_voting_layer_v4,
    ransac_voting_layer_v5,
    ransac_voting_pipeline,
    ransac_voting_vanish_point_layer,
    refit_at_points,
)
