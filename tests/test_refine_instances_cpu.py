"""CPU: the two boundary rules of oracle/refine_instances_oracle.py (DESIGN.md §30) on hand-built label maps."""
import numpy as np

from oracle import refine_instances_oracle as rio
from oracle import refine_oracle as rfo


def _set(idx, w):
    return {divmod(int(p), w) for p in idx}


def test_shared_border_is_in_neither_contour():
    lab = np.zeros((6, 8), np.int32)
    lab[1:5, 1:4] = 1
    lab[1:5, 4:7] = 2
    c1, c2 = _set(rio.contour(lab, 0), 8), _set(rio.contour(lab, 1), 8)
    # the shared columns' inner rows touch only the other instance; their end rows touch the background
    assert not {(2, 3), (3, 3)} & c1 and not {(2, 4), (3, 4)} & c2 and (1, 3) in c1 and (4, 4) in c2
    assert (1, 1) in c1 and (4, 6) in c2 and (2, 1) in c1
    # one instance alone keeps the whole outline, as refine_oracle.boundary takes it
    one = (lab == 1).astype(np.int32)
    assert np.array_equal(rio.contour(one, 0), rfo.boundary(one != 0))


def test_label_above_L_counts_as_another_instance():
    lab = np.zeros((5, 7), np.int32)
    lab[1:4, 1:4] = 1
    lab[1:4, 4:6] = 40                                # above any L
    c = _set(rio.contour(lab, 0), 7)
    assert (2, 3) not in c and (2, 1) in c
    occ = rio.occluded(lab, 0)
    assert occ[2, 3] and not occ[2, 1]


def test_instance_on_the_image_edge():
    lab = np.zeros((4, 5), np.int64)
    lab[:, :2] = 1
    lab[:, 2:] = 2
    c = _set(rio.contour(lab, 0), 5)
    # column 0 lies on the border; column 1 only touches instance 2 and the top and bottom border
    assert {(r, 0) for r in range(4)} <= c and (1, 1) not in c and (0, 1) in c and (3, 1) in c


def test_silhouette_3x3_neighbourhood_just_touching():
    lab = np.zeros((7, 7), np.int32)
    lab[5, 5] = 2                                     # another instance diagonal to (4, 4) only
    depth = np.zeros((7, 7), np.float32)
    depth[1:5, 1:5] = 1.0
    s = _set(rio.silhouette(depth, lab, 0), 7)
    full = _set(rfo.boundary(depth > 0), 7)
    assert full - s == {(4, 4)}                      # (4, 4) has (5, 5) in its 3x3 neighbourhood; (4, 3) does not
    lab[5, 5] = 1                                     # the instance itself is not an occluder
    assert _set(rio.silhouette(depth, lab, 0), 7) == full


def test_num_zero_keeps_every_pose():
    lab = np.zeros((2, 6, 6), np.int32)
    lab[:, 1:4, 1:4] = 1
    poses = np.tile(np.eye(3, 4), (2, 3, 1, 1))
    poses[..., 2, 3] = 0.5
    out, info = rio.refine(lab, np.zeros(2, np.int32), poses, np.eye(3), np.zeros((0, 3), np.float32),
                           np.zeros((0, 3), np.int32), 0.05, 5.0)
    assert np.array_equal(out, poses) and (info["status"] == rio.NO_INSTANCE).all()
    assert (info["pairs"] == 0).all() and np.isnan(info["dist_before"]).all()
