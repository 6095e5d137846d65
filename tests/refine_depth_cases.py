"""Observed depth images for the depth-anchored refinement tests (tests/test_refine_depth_cpu.py,
tests/test_gpu_refine_depth.py) and benchmarks/refine_depth.py.  The mesh itself is the sensor: the observed depth is
its render at the true pose, then one of the variants below.  Lengths are in metres."""
import numpy as np

GATE = 0.03                                          # 3 cm: above a 1 cm / 3 degree start's largest point offset


def noisy(depth, sigma, rng):
    """Seeded Gaussian noise of `sigma` on every reading, float32; pixels without a reading keep 0."""
    d = np.asarray(depth, np.float32)
    out = d + rng.normal(0.0, sigma, d.shape).astype(np.float32)
    return np.where(d > 0, out, np.float32(0)).astype(np.float32)


def holed(depth, r0, c0, size):
    """A size x size block of zero readings (no reading) with its top-left corner at (r0, c0)."""
    out = np.array(depth, np.float32, copy=True)
    out[..., r0:r0 + size, c0:c0 + size] = 0
    return out


def occluded(depth, mask, r0, c0, size, gap=0.05):
    """An occluder: a size x size patch at (r0, c0) `gap` closer than the object's nearest reading in the image, and
    the mask cut out where it sits (the segmentation sees the occluder, not the object)."""
    d = np.array(depth, np.float32, copy=True)
    m = np.array(mask, copy=True)
    near = d[d > 0].min() if (d > 0).any() else 0.5
    d[r0:r0 + size, c0:c0 + size] = np.float32(near - gap)
    m[r0:r0 + size, c0:c0 + size] = 0
    return d, m


def as_u16_mm(depth):
    """uint16 millimetres (the LINEMOD PNG format), rounded to the nearest; read back with depth_scale = 1e-3."""
    return np.round(np.asarray(depth, np.float64) * 1000.0).clip(0, 65535).astype(np.uint16)


def along_axis(P, dist):
    """The poses P [b,3,4] moved by `dist` along the optical axis (t_z only)."""
    out = np.array(P, np.float64, copy=True)
    out[..., 2, 3] += dist
    return out
