"""CPU: `refine_instances` of tests/refine_depth_instance_cases.py (the contract of `pvnet_refine_poses_depth_instances`,
DESIGN.md §31) on hand-built 120x160 label maps: a pixel pairs only when it and its four 4-neighbours carry its own
label, labels above L are other instances, instances on the image edge and one pixel thick, absent rows, and L = 1
against `refine` on the mask.  Plus the entry point's refusals that come before any device work.  The device is held
to this helper in tests/test_gpu_refine_depth_instances.py."""
import numpy as np
import pytest
import torch

from oracle import refine_depth_oracle as rdo
from oracle import refine_oracle as rfo
from oracle import render_oracle as ro
from tests import refine_cases as rf
from tests import refine_depth_cases as rdc
from tests import refine_depth_instance_cases as ric
from tests import render_cases as rc

H, W = 120, 160
K = rc.camera_for(H, W, 300.0)
MESH = rf.tool_mesh()
FLAT = np.hstack([np.eye(3), np.zeros((3, 1))])


def flat(*_):
    """A render step that covers the whole frame at 0.5: with readings of 0.5 and the pose R = I, t = 0 every pixel's
    rendered and observed points coincide, so the pair set is the predicate alone."""
    return np.full((H, W), 0.5, np.float32)


def round0(labels, L, num=None, depth=None):
    """-> {j: first-round trace record} of every present row of the one-image map, and the info dict."""
    num = np.array([L if num is None else num])
    depth = np.full((1, H, W), 0.5, np.float32) if depth is None else depth
    traces = {}
    _, info = ric.refine_instances(labels[None], num, depth, np.tile(FLAT, (1, L, 1, 1)), K, *MESH, rf.NEAR, rf.FAR,
                                   rdc.GATE, rounds=0, render=flat, traces=traces)
    return {j: traces[(0, j)][0] for j in range(int(num[0]))}, info


def cells(idx):
    return {divmod(int(p), W) for p in idx}


def rect(r0, r1, c0, c1):
    return {(r, c) for r in range(r0, r1) for c in range(c0, c1)}


def test_a_pixel_next_to_another_instance_does_not_pair():
    lab = np.zeros((H, W), np.int32)
    lab[20:60, 20:80] = 1
    lab[20:60, 80:120] = 2
    tr, info = round0(lab, 2)
    # the interior of each rectangle: column 79's right neighbour and column 80's left one carry the other label
    assert cells(tr[0]["idx"]) == rect(21, 59, 21, 79)
    assert cells(tr[1]["idx"]) == rect(21, 59, 81, 119)
    assert (tr[0]["mask_pixels"], tr[1]["mask_pixels"]) == (40 * 60, 40 * 40)
    assert tr[0]["covered_pixels"] == H * W and (info["status"] == 0).all()
    # merged into one label, the border columns pair: the rule is what drops them
    merged = np.where(lab > 0, 1, 0)
    tm, _ = round0(merged, 1)
    assert {(r, c) for r in range(21, 59) for c in (79, 80)} <= cells(tm[0]["idx"])


def test_a_label_above_L_counts_as_another_instance():
    lab = np.zeros((H, W), np.int64)
    lab[30:70, 30:70] = 1
    lab[30:70, 70:90] = 40
    tr, _ = round0(lab, 2, num=1)
    assert cells(tr[0]["idx"]) == rect(31, 69, 31, 69)
    assert tr[0]["mask_pixels"] == 40 * 40


def test_an_instance_on_the_image_edge():
    lab = np.zeros((H, W), np.uint8)
    lab[:30, :40] = 1
    lab[H - 25:, W - 35:] = 2
    tr, _ = round0(lab, 2)
    # border pixels never pair; the row and column next to the border do, their outer neighbour being in the image
    assert cells(tr[0]["idx"]) == rect(1, 29, 1, 39)
    assert cells(tr[1]["idx"]) == rect(H - 24, H - 1, W - 34, W - 1)


@pytest.mark.parametrize("axis", [0, 1])
def test_an_instance_one_pixel_thick_has_no_pairs(axis):
    lab = np.zeros((H, W), np.int16)
    lab[40:80, 40:80] = 2
    if axis == 0:
        lab[50, 10:100] = 1                                   # a row, crossing instance 2
    else:
        lab[5:110, 60] = 1                                    # a column, crossing instance 2
    tr, info = round0(lab, 2)
    assert len(tr[0]["idx"]) == 0 and tr[0]["count"] == 0 and info["status"][0, 0] == rfo.FEW_PAIRS
    # instance 2 loses the pixels beside the crossing line, and the line itself
    cut = rect(41, 79, 41, 79) - ({(r, c) for r in (49, 50, 51) for c in range(W)} if axis == 0 else
                                  {(r, c) for r in range(H) for c in (59, 60, 61)})
    assert cells(tr[1]["idx"]) == cut and info["status"][0, 1] == 0


def test_num_zero_and_absent_rows_keep_their_pose():
    lab = np.zeros((2, H, W), np.int32)
    lab[:, 30:60, 30:60] = 1
    lab[:, 70:90, 90:130] = 2
    poses = np.tile(FLAT, (2, 3, 1, 1))
    poses[..., 2, 3] = np.arange(6).reshape(2, 3) + 0.25
    depth = np.full((2, H, W), 0.5, np.float32)
    out, info = ric.refine_instances(lab, np.array([0, 2]), depth, poses, K, *MESH, rf.NEAR, rf.FAR, rdc.GATE,
                                     rounds=0, render=flat)
    assert np.array_equal(out, poses)
    assert info["status"].tolist() == [[ric.NO_INSTANCE] * 3, [0, 0, ric.NO_INSTANCE]]
    absent = info["status"] == ric.NO_INSTANCE
    assert (info["pairs"][absent] == 0).all() and np.isnan(info["dist_before"][absent]).all()
    assert np.isnan(info["dist_after"][absent]).all() and (info["dist_before"][~absent] == 0).all()


def test_one_instance_equals_refine_on_the_mask():
    rng = np.random.default_rng(4)
    Pt = rf.true_poses(1, rng)[0]
    P0 = rf.perturb(Pt[None], rng)
    d = ro.render(*MESH, K, Pt.astype(np.float32)[None], H, W, rf.NEAR, rf.FAR)[0][0]
    obs = rdc.noisy(d, 1e-3, rng)[None]
    lab = (d > 0).astype(np.uint8)
    a, ia = rdo.refine(lab[None], obs, P0, K, *MESH, rf.NEAR, rf.FAR, rdc.GATE, rounds=3)
    b, ib = ric.refine_instances(lab[None], np.array([1]), obs, P0[:, None], K, *MESH, rf.NEAR, rf.FAR, rdc.GATE,
                                 rounds=3)
    assert np.array_equal(a, b[:, 0])
    for key in ia:
        assert np.array_equal(ia[key], ib[key][:, 0], equal_nan=True), key
    assert ib["pairs"][0, 0] > 100


def test_refine_poses_depth_instances_refuses_cpu_and_malformed_arguments():
    from pvnet_b200.refine import refine_poses_depth_instances
    v, f = (torch.from_numpy(x) for x in MESH)
    lab, num = torch.zeros(1, 8, 8, dtype=torch.uint8), torch.ones(1, dtype=torch.int32)
    depth, poses = torch.zeros(1, 8, 8), torch.zeros(1, 2, 3, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        refine_poses_depth_instances(lab, num, depth, poses, torch.eye(3), v, f, rf.NEAR, rf.FAR, gate=0.03)
    with pytest.raises(ValueError):                                                               # not a tensor
        refine_poses_depth_instances(lab.numpy(), num, depth, poses, torch.eye(3), v, f, rf.NEAR, rf.FAR, gate=0.03)
    with pytest.raises(TypeError):
        refine_poses_depth_instances(lab, num, depth, poses, torch.eye(3), v, f, rf.NEAR, rf.FAR)     # no gate
