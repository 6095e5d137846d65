"""Meshes, cameras and poses for the silhouette-refinement tests (tests/test_refine_cpu.py, tests/test_gpu_refine.py)
and benchmarks/refine.py.  Lengths are in metres, so the perturbations read as "3 degrees and 1 cm"."""
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
