"""Seeded EPnP problems, regenerated from their names (tests/golden/make_golden_epnp.py stores only cv2's poses for
them in tests/golden/epnp_cases.npz).  Built from tests/pnp_cases.py's regimes: object points, intrinsics and poses,
with isotropic Gaussian pixel noise of sigma 0, 1 or 3 px; object and image points are float32, the values cv2, the
oracle and the device all read.

Names: "<regime>/pn<count>/s<sigma>" (BATCH images each; the cat regime has 9 keypoints, so its counts stop at 9) and
"coplanar/pn<count>" (a random 0.2 m square of points with z = 0 exactly: status bit 1).
"""
import zlib

import numpy as np

from tests import pnp_cases as pc

POINT_COUNTS = (4, 5, 6, 9, 16, 32, 33, 100, 1024)
SIGMAS = (0, 1, 3)
BATCH = 8
COPLANAR_COUNTS = (6, 9, 32)


def names():
    out = []
    for regime in pc.REGIMES:
        for n in POINT_COUNTS:
            if regime == "cat" and n > 9:
                continue
            out += [f"{regime}/pn{n}/s{s}" for s in SIGMAS]
    return out + [f"coplanar/pn{n}" for n in COPLANAR_COUNTS]


def problem(name):
    """dict(P float32 [pn,3], K float64 [3,3], R [BATCH,3,3], t [BATCH,3], x float32 [BATCH,pn,2], unit)."""
    rng = np.random.default_rng(zlib.crc32(("epnp/" + name).encode()))
    parts = name.split("/")
    n = int(parts[1][2:])
    if parts[0] == "coplanar":
        regime, sigma = "cloud", 0.0
        P = np.concatenate([rng.uniform(-0.1, 0.1, (n, 2)), np.zeros((n, 1))], 1).astype(np.float32)
    else:
        regime, sigma = parts[0], float(parts[2][1:])
        P = pc.object_points(regime, n, rng)
    K = pc.camera(regime, rng if regime in ("cloud", "close", "mm") else None)
    R, t = pc.poses(regime, BATCH, rng)
    x = (pc.project(P, R, t, K) + rng.normal(0.0, 1.0, (BATCH, n, 2)) * sigma).astype(np.float32)
    return dict(P=P, K=K, R=R, t=t, x=x, unit=pc.unit(regime))


def key(name):
    return name.replace("/", "__")
