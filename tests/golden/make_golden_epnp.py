"""Writes tests/golden/epnp_cases.npz: OpenCV's EPnP pose for every problem of tests/epnp_cases.py, as the reference
computes it (lib/utils/evaluation_utils.py:19-52 with method=cv2.SOLVEPNP_EPNP: solvePnP, then Rodrigues), and the cv2
version.  The inputs are not stored; tests regenerate them from the names.  Needs cv2; run from the repository root:
    python tests/golden/make_golden_epnp.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import cv2  # noqa: E402

from tests import epnp_cases as ec  # noqa: E402


def cv2_epnp(P, x, K):
    _, rvec, tvec = cv2.solvePnP(P.astype(np.float64)[None], x.astype(np.float64)[None], K.astype(np.float64),
                                 np.zeros((8, 1)), flags=cv2.SOLVEPNP_EPNP)
    R, _ = cv2.Rodrigues(rvec)
    return np.concatenate([R, tvec], 1)


def main():
    out = {"cv2_version": np.array(cv2.__version__)}
    for name in ec.names():
        pr = ec.problem(name)
        out[ec.key(name)] = np.stack([cv2_epnp(pr["P"], x, pr["K"]) for x in pr["x"]])
    path = os.path.join(ROOT, "tests", "golden", "epnp_cases.npz")
    np.savez_compressed(path, **out)
    print(path, len(out) - 1, "problems")


if __name__ == "__main__":
    main()
