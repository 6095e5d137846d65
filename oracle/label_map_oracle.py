"""numpy restatement of `pvnet_render_label_map` (csrc/render.cu, DESIGN.md §25): the label map of several meshes at
a batch of images, the reference's `OcclusionLineModDB.get_mask_of_all_objects` (lib/utils/data_utils.py:788-826).

The contract, which the kernel follows bit for bit:

* M meshes (1 <= M <= 255), each with its own fp32 vertices, int faces local to it, and a label in 1..255.  For each
  image, one [3,4] pose per slot and a `present` flag per slot (the reference leaves an object out when its pose
  is empty).  K is [3,3] or [b,3,3].
* A slot's depth at a pixel is `render_oracle.render`'s depth of its mesh alone (coverage, clip planes, pixel
  convention and fp64 geometry of DESIGN.md §24), divided by depth_divisor with one IEEE fp32 division: the
  reference's `render(...) / 1000.` on a float32 array.  near / depth_divisor must not underflow to 0, so a covered
  pixel's divided depth is positive.
* label: the label of the present slot with the smallest divided depth strictly below max_depth; ties go to the
  lower slot; 0 where there is none.  depth: that depth, max_depth where the label is 0.  This is the reference's
  update in slot order -- a covered pixel takes the object when its depth is below the map's -- on a depth map that
  starts at max_depth (10 in the reference).

The key is the divided depth, not Z: two fp32 depths one ulp apart can divide to the same value, and the earlier
slot then keeps the pixel.  CPU only; nothing here reads the reference.
"""
from __future__ import annotations

import numpy as np

from oracle import render_oracle as ro


def divide(depth, depth_divisor):
    """fp32 depth maps (0 where uncovered) / depth_divisor: one IEEE fp32 division per pixel."""
    return np.asarray(depth, np.float32) / np.float32(depth_divisor)


def composite(depths, labels, max_depth=np.inf):
    """depths fp32 [M,...] (already divided; 0 where the slot covers nothing or is absent), labels [M] -> label uint8
    [...], depth fp32 [...]: slot by slot, a covered pixel takes the slot's label when its depth is below the map's."""
    depths = np.asarray(depths, np.float32)
    label = np.zeros(depths.shape[1:], np.uint8)
    depth = np.full(depths.shape[1:], np.float32(max_depth), np.float32)
    for m in range(depths.shape[0]):
        take = (depths[m] != 0) & (depths[m] < depth)
        label[take] = labels[m]
        depth[take] = depths[m][take]
    return label, depth


def label_map(meshes, labels, poses, K, h, w, near, far, present=None, depth_divisor=1.0, max_depth=np.inf):
    """meshes [(verts [nv,3], faces [nf,3])] * M, labels [M], poses [b,M,3,4], K [3,3] or [b,3,3], present [b,M] or
    None -> label uint8 [b,h,w], depth fp32 [b,h,w]."""
    M = len(meshes)
    assert 1 <= M <= 255 and len(labels) == M and all(1 <= int(v) <= 255 for v in labels)
    poses = np.asarray(poses, np.float32).reshape(-1, M, 3, 4)
    b = poses.shape[0]
    K = np.asarray(K, np.float32)
    Ks = np.broadcast_to(K, (b, 3, 3)) if K.shape == (3, 3) else K.reshape(b, 3, 3)
    present = np.ones((b, M), bool) if present is None else np.asarray(present).reshape(b, M) != 0
    assert np.float32(near) / np.float32(depth_divisor) > 0
    label = np.zeros((b, h, w), np.uint8)
    depth = np.zeros((b, h, w), np.float32)
    for i in range(b):
        slots = np.zeros((M, h, w), np.float32)
        for m, (v, f) in enumerate(meshes):
            if present[i, m] and len(f):
                slots[m] = divide(ro.render(v, f, Ks[i], poses[i, m][None], h, w, near, far)[0][0], depth_divisor)
        label[i], depth[i] = composite(slots, labels, max_depth)
    return label, depth
