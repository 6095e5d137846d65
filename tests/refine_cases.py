"""Meshes, cameras, poses and masks for the silhouette-refinement tests (tests/test_refine_cpu.py,
tests/test_refine_edges_cpu.py, tests/test_gpu_refine.py, tests/test_gpu_refine_edges.py) and benchmarks/refine.py,
and `device_depth`, the oracle's render step on the device.  Lengths are in metres, so the perturbations read as
"3 degrees and 1 cm"."""
import numpy as np

from oracle import refine_oracle as rfo
from tests import render_cases as rc

NEAR, FAR = 0.05, 5.0


def lumpy_mesh(subdiv=2):
    """An asymmetric closed mesh about 10 cm across: an icosphere stretched to 12 x 8 x 6 cm with a bump on one side,
    so no rotation or mirror maps its silhouette onto itself."""
    v, f = rc.icosphere(subdiv, 1.0)
    v = v.astype(np.float64)
    bump = 1.0 + 0.5 * np.clip(v @ np.array([0.6, 0.7, 0.4]), 0, None) ** 3
    v = v * bump[:, None] * np.array([0.06, 0.04, 0.03])
    return v.astype(np.float32), f


def box(lo, hi):
    """An axis-aligned box as 12 triangles."""
    v, f = rc.cube(1.0)
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    return ((v + 1) / 2 * (hi - lo) + lo).astype(np.float32), f


def tool_mesh():
    """Three boxes that overlap into one asymmetric solid about 13 cm across (a handle, a head off to one side and a
    fin): its silhouette has corners, so a rotation or mirror image of it does not fit the same outline."""
    parts = [box((-0.07, -0.015, -0.01), (0.05, 0.015, 0.01)), box((0.03, -0.015, -0.01), (0.06, 0.05, 0.02)),
             box((-0.06, -0.01, 0.0), (-0.03, 0.01, 0.035))]
    verts, faces, off = [], [], 0
    for v, f in parts:
        verts.append(v)
        faces.append(f + off)
        off += len(v)
    return np.concatenate(verts), np.concatenate(faces).astype(np.int32)


def axis_angle(w):
    return rfo.so3_exp(np.asarray(w, np.float64))


def true_poses(b, rng, depth=(0.45, 0.6), shift=0.03):
    """b rotations in front of the camera, float64 [b,3,4]."""
    P = np.zeros((b, 3, 4))
    for i in range(b):
        P[i, :, :3] = rc.rotation(rng)
        P[i, :, 3] = (rng.normal(0, shift), rng.normal(0, shift), rng.uniform(*depth))
    return P


def perturb(P, rng, deg=3.0, dist=0.01):
    """Each pose turned by `deg` degrees about a random axis and moved by `dist` in a random direction."""
    out = np.array(P, np.float64, copy=True)
    for i in range(len(out)):
        a = rng.normal(size=3)
        d = rng.normal(size=3)
        out[i, :, :3] = axis_angle(a / np.linalg.norm(a) * np.deg2rad(deg)) @ out[i, :, :3]
        out[i, :, 3] += d / np.linalg.norm(d) * dist
    return out


def rotation_error_deg(Ra, Rb):
    c = (np.trace(Ra @ Rb.T) - 1) / 2
    return float(np.degrees(np.arccos(np.clip(c, -1, 1))))


def pose_error(Pa, Pb):
    """-> (rotation error in degrees, translation error in metres)."""
    Pa, Pb = np.asarray(Pa).reshape(3, 4), np.asarray(Pb).reshape(3, 4)
    return rotation_error_deg(Pa[:, :3], Pb[:, :3]), float(np.linalg.norm(Pa[:, 3] - Pb[:, 3]))


def comb_mesh(teeth=16, length=0.2, width=0.005, gap=0.01):
    """A spine with `teeth` thin bars hanging from it, facing +z: at 0.5 m and f = 572 px its silhouette has several
    thousand border pixels, more than one 4 096-point cap."""
    parts = [box((0.0, -0.01, 0.0), (teeth * (width + gap), 0.0, 0.01))]
    for k in range(teeth):
        x = k * (width + gap)
        parts.append(box((x, 0.0, 0.0), (x + width, length, 0.01)))
    verts, faces, off = [], [], 0
    for v, f in parts:
        verts.append(v)
        faces.append(f + off)
        off += len(v)
    return np.concatenate(verts), np.concatenate(faces).astype(np.int32)


def singular_scene():
    """Six one-pixel triangles whose silhouette points all lie on the line through the object's origin along the
    optical axis: mesh (verts, faces), a 40 x 40 K with fx = fy = 1 and (cx, cy) = (0.5, 0.5), the pose [3,4] and
    the mask (the same six pixels).  Pixel (k, k), k = 1, 2, 4, ..., 32, is covered at depth 4 / k, which
    back-projects to X_cam = (4, 4, 4 / k) exactly, so R^T (X_cam - t) = (0, 0, 4 / k) with t = (4, 4, 0): every
    rotation about the optical axis moves no point, the dw_z row and column of the normal equations are exactly
    zero, and so is A + 1e-3 diag(A)'s diagonal there."""
    h = w = 40
    K = np.array([[1, 0, 0.5], [0, 1, 0.5], [0, 0, 1]], np.float32)
    t = np.array([4.0, 4.0, 0.0])
    verts, faces = [], []
    for i, k in enumerate((1, 2, 4, 8, 16, 32)):
        Z = 4.0 / k
        for dx, dy in ((-0.3, -0.3), (0.3, -0.3), (0.0, 0.3)):      # a third of a pixel about the centre
            verts.append(np.array([4.0 + dx * Z, 4.0 + dy * Z, Z]) - t)
        faces.append([3 * i, 3 * i + 2, 3 * i + 1])
    pose = np.hstack([np.eye(3), t[:, None]])
    mask = np.zeros((h, w), bool)
    for k in (1, 2, 4, 8, 16, 32):
        mask[k, k] = True
    return (np.array(verts, np.float32), np.array(faces, np.int32)), K, pose, mask


# ---- masks with a chosen contour: the cases PVNet's argmax masks make (speckle, holes) at exact point counts ----

def _dilate4(on, k, outside=False):
    """Pixels within 4-neighbour distance k of an on pixel, or of the outside when `outside` is True."""
    out = on.copy()
    for _ in range(k):
        p = np.pad(out, 1, constant_values=outside)
        out = out | p[:-2, 1:-1] | p[2:, 1:-1] | p[1:-1, :-2] | p[1:-1, 2:]
    return out


def hole_sites(on):
    """Pixels of `on` at least two 4-steps from anything off (the outside included), on a 3-pixel grid: punching one
    out turns exactly its four neighbours into contour pixels, and no two sites share a neighbour."""
    h, w = on.shape
    r, c = np.mgrid[:h, :w]
    return np.flatnonzero(~_dilate4(~on, 2, outside=True) & (r % 3 == 0) & (c % 3 == 0))


def speckle_sites(on, region=None):
    """Off pixels whose 4-neighbours are all off, on a 2-pixel grid (inside `region` if given): setting one adds
    exactly one contour pixel, itself, and changes no other pixel's status."""
    h, w = on.shape
    r, c = np.mgrid[:h, :w]
    ok = ~_dilate4(on, 1) & (r % 2 == 0) & (c % 2 == 0)
    return np.flatnonzero(ok if region is None else ok & region)


def with_contour_count(on, n, holes=0, seed=0):
    """A copy of the mask `on` (bool [h,w]) with `holes` one-pixel holes punched inside it and isolated pixels
    scattered outside it, so that rfo.boundary finds exactly n points.  Both are drawn with `seed`."""
    on = np.asarray(on, bool)
    rng = np.random.default_rng(seed)
    out = on.copy().reshape(-1)
    hs = hole_sites(on)
    assert holes <= len(hs), (holes, len(hs))
    out[np.sort(rng.choice(hs, holes, replace=False))] = False
    extra = n - len(rfo.boundary(on)) - 4 * holes
    ss = speckle_sites(on)
    assert 0 <= extra <= len(ss), (n, extra, len(ss))
    out[np.sort(rng.choice(ss, extra, replace=False))] = True
    out = out.reshape(on.shape)
    assert len(rfo.boundary(out)) == n
    return out


def round0_d2(sil, depth, pose, K, con, w):
    """The first round's fp32 d2 [ns, nc] of every silhouette point against every contour pixel (rfo's steps)."""
    X = rfo.back_project(sil, depth, pose, K, w)
    u, v = rfo.project(X, pose, K)
    pu, pv = u.astype(np.float32), v.astype(np.float32)
    cu, cv = rfo.centres(con, w)
    dx, dy = cu[None, :] - pu[:, None], cv[None, :] - pv[:, None]
    return dx * dx + dy * dy


def straddling_tie(mask, depth, pose, K, gate=20.0, at=2047, margin=24):
    """Pad `mask` with isolated pixels in rows above the object, so that some silhouette point's nearest contour
    pixels are a tie between contour index `at` (the last point of the first 2 048-point tile) and a later index.

    The padding precedes every object contour pixel in row-major order and lies more than `margin` (> gate) rows
    above the object and its render, so it moves the object's contour indices up without being anyone's pair.
    -> (padded mask, silhouette index i, lower index, higher index) of the chosen tie, indices in the padded mask."""
    mask, h, w = np.asarray(mask, bool), *np.asarray(mask).shape
    assert margin > gate
    sil = rfo.boundary(depth > 0)
    con = rfo.boundary(mask)
    d = round0_d2(sil, depth, pose, K, con, w)
    best = d.min(1)
    ties = (d == best[:, None]).sum(1) >= 2
    a = d.argmin(1)
    cand = np.flatnonzero(ties & (best <= np.float32(gate) ** 2) & (a <= at))
    assert len(cand), "no tie to move"
    i = int(cand[0])
    lo, hi = np.flatnonzero(d[i] == best[i])[:2]
    top = min(np.nonzero(mask)[0].min(), np.nonzero(depth > 0)[0].min())
    rows = np.zeros((h, w), bool)
    rows[:max(0, top - margin)] = True
    sites = speckle_sites(mask, rows)
    pad = at - lo
    assert pad <= len(sites), (pad, len(sites))
    out = mask.copy().reshape(-1)
    out[sites[:pad]] = True
    out = out.reshape(h, w)
    assert np.array_equal(rfo.boundary(out)[pad:], con)
    return out, i, int(lo + pad), int(hi + pad)


def spur(on, length=15, half=3):
    """The mask `on` with a bar 2 half + 1 rows tall and `length` columns long stuck to its right edge at its middle
    row: a start at the truth then pairs most silhouette points at distance 0 and a few with the bar, and the least
    squares step towards the bar raises the mean pair distance, so the first round is undone."""
    out = np.asarray(on, bool).copy()
    rows, cols = np.nonzero(out)
    r0 = int(rows.mean())
    c1 = int(cols[rows == r0].max())
    out[max(0, r0 - half):r0 + half + 1, c1:c1 + length] = True
    return out


def device_depth(dev="cuda:0"):
    """Step 1 of oracle/refine_oracle.py on the device: `render=` for rfo.refine_image / rfo.refine that calls
    `pvnet_b200.render.render_mesh`, which tests/test_gpu_render.py pins bit for bit to render_oracle for the same
    fp32 pose and K.  The mesh is uploaded once per (verts, faces) pair."""
    import torch

    from pvnet_b200.render import render_mesh
    meshes = {}

    def render(verts, faces, K, pose32, h, w, near, far):
        key = (id(verts), id(faces))
        if key not in meshes:
            meshes[key] = (verts, faces, torch.as_tensor(np.ascontiguousarray(verts), device=dev),
                           torch.as_tensor(np.ascontiguousarray(faces), device=dev))
        v, f = meshes[key][2:]
        k = torch.as_tensor(np.asarray(K, np.float32), device=dev)
        p = torch.as_tensor(np.asarray(pose32, np.float32)[None], device=dev)
        return render_mesh(v, f, k, p, h, w, near, far)[0].cpu().numpy()

    return render
