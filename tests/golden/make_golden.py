"""Regenerates tests/golden/*.npz.  Run with PVNET_REFERENCE naming a checkout of
the reference project:   PVNET_REFERENCE=<path> python tests/golden/make_golden.py

demo_cat.npz -- the reference's only usable known-answer fixture (SURVEY.md §4,
App. E).  From <reference>/data/demo (cat_mask.png, cat_points_3d.txt,
cat_pose.npy) and the LINEMOD intrinsics of lib/utils/base_utils.py:240-243 it
derives, exactly as tools/demo.py:58-71,74-88 (`compute_vertex`, `read_data`) do:
  fg_yx      [2289,2] int16   foreground pixel coordinates (row-major order)
  points_2d  [9,2]   float64  projected keypoints = the answer voting must return
The exact vector field is re-synthesised from these two in the tests (it is a
pure function of them), so the fixture stays a few KB.

oracle_cfg1.npz -- outputs of the oracle (oracle/pvnet_oracle.py) on BASELINE
config 1 (b=1, N=10000, K=9, hn=128, thresh 0.99, random and planted fields,
injected idxs), frozen so that a later change to the oracle or the generators is
noticed: counts [128,9] int32, keypoints [9,2], hypothesis checksum.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.helpers import reference_root  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def make_demo():
    import cv2
    demo = os.path.join(reference_root(), "data", "demo")
    mask = cv2.imread(os.path.join(demo, "cat_mask.png"))[..., 0]
    mask = (mask != 0)
    pts3d = np.loadtxt(os.path.join(demo, "cat_points_3d.txt"))
    pose = np.load(os.path.join(demo, "cat_pose.npy")).astype(np.float64)
    K = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])
    cam = pts3d @ pose[:, :3].T + pose[:, 3:].T
    img = cam @ K.T
    pts2d = img[:, :2] / img[:, 2:]
    fg = np.argwhere(mask).astype(np.int16)
    np.savez_compressed(os.path.join(HERE, "demo_cat.npz"), fg_yx=fg, points_2d=pts2d,
                        shape=np.array(mask.shape))
    print("demo_cat.npz:", fg.shape[0], "foreground px;", pts2d.round(4).tolist())


def make_cfg1():
    from oracle import pvnet_oracle as po
    from pvnet_b200 import synthetic as syn
    out = {}
    mask = syn.disc_mask(10000)
    for name, field in (("random", syn.random_field(mask, 9, 1000)),
                        ("planted", syn.planted_field(mask, 9, 1000)[0])):
        vertex = syn.as_reference_view(field[None])
        idxs = syn.draw_idxs(10000, 128, 9, seed=1000)
        kp, dbg = po.ransac_voting_layer_v3(mask[None], vertex, 128, inlier_thresh=0.99,
                                            idxs=[idxs], return_debug=True)
        out[name + "_counts"] = dbg[0]["counts"]
        out[name + "_kp"] = kp[0]
        out[name + "_hyp_sum"] = np.float64(dbg[0]["hyp"].astype(np.float64).sum())
        out[name + "_win_idx"] = dbg[0]["win_idx"]
    np.savez_compressed(os.path.join(HERE, "oracle_cfg1.npz"), **out)
    print("oracle_cfg1.npz written; planted kp:\n", out["planted_kp"])


if __name__ == "__main__":
    make_demo()
    make_cfg1()
