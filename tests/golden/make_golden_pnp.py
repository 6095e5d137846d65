"""Generates tests/golden/pnp_cases.npz (needs PVNET_REFERENCE = a checkout of the reference project, cv2, scipy).

Cases:
  demo        the reference's own fixture: data/demo/cat_points_3d.txt (+ centre) projected with
              cat_pose.npy and the linemod intrinsics of tools/demo.py:176-178 -> the pose must come back
              (known answer); identity weights and anisotropic weights (exact correspondences: the
              minimum is the same pose whatever the weights).
  noisy_*     the same object under random poses, keypoints perturbed by per-point anisotropic Gaussian
              noise with the matching covariances; expected pose = minimiser of the reference's cost
              (uncertainty_pnp.cpp:20-37) from the reference's initialisation (cv2 SOLVEPNP_P3P on the 4 most
              confident points, extend_utils.py:84-88) found by scipy LM at 1e-15 tolerances.  Also recorded:
              cv2.solvePnP(SOLVEPNP_ITERATIVE) for the isotropic cases (independent check of the optimiser).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests.helpers import reference_root  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import pnp_oracle as pn  # noqa: E402

REF = os.path.join(reference_root(), "data", "demo")


def main():
    import cv2
    pts = np.loadtxt(os.path.join(REF, "cat_points_3d.txt"))
    if pts.shape[0] == 8:                       # 8 FPS points + the centre, as tools/demo.py builds them
        bb8 = np.loadtxt(os.path.join(REF, "cat_bb8_3d.txt"))
        pts = np.concatenate([pts, ((bb8.max(0) + bb8.min(0)) / 2)[None]], 0)
    pose = np.load(os.path.join(REF, "cat_pose.npy"))
    K = np.array([[572.4114, 0., 325.2611], [0., 573.57043, 242.04899], [0., 0., 1.]])      # tools/demo.py:176-178
    rng = np.random.default_rng(2024)
    cases = {}

    def project(Rt):
        X = pts @ Rt[:, :3].T + Rt[:, 3]
        return np.stack([K[0, 0] * X[:, 0] / X[:, 2] + K[0, 2], K[1, 1] * X[:, 1] / X[:, 2] + K[1, 2]], 1)

    def add(name, kp, cov, expect):
        cases[name + "_kp"] = kp.astype(np.float32)
        cases[name + "_cov"] = cov.astype(np.float32)
        cases[name + "_pose"] = expect

    kp = project(pose)
    add("demo_iso", kp, np.tile(np.eye(2) * 4.0, (9, 1, 1)), pose)
    A = rng.normal(0, 1, (9, 2, 2))
    add("demo_aniso", kp, A @ A.transpose(0, 2, 1) + 0.5 * np.eye(2), pose)
    cv_iter = {}
    for i in range(12):
        r = rng.normal(0, 0.8, 3)
        t = np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.6, 1.2)])
        Rt = np.concatenate([pn.rodrigues(r), t[:, None]], 1)
        iso = i % 3 == 0
        if iso:
            cov = np.tile(np.eye(2) * rng.uniform(1, 9), (9, 1, 1))
        else:
            A = rng.normal(0, 1.5, (9, 2, 2))
            cov = A @ A.transpose(0, 2, 1) + 0.3 * np.eye(2)
        noise = np.stack([rng.multivariate_normal(np.zeros(2), c) for c in cov])
        kp32 = (project(Rt) + noise).astype(np.float32)
        cov32 = cov.astype(np.float32)
        w = pn.covariance_to_weights(cov32)
        expect = pn.uncertainty_pnp(kp32, w, pts, K, use_cv2_init=True)
        own = pn.uncertainty_pnp(kp32, w, pts, K, use_cv2_init=False)
        assert np.abs(expect - own).max() < 1e-12, "own P3P start reaches a different minimum than OpenCV's"
        g = pn.residuals(np.concatenate([pn.rotation_to_rvec(expect[:, :3]), expect[:, 3]]), kp32.astype(np.float64), w, pts, K)
        add(f"noisy_{i}", kp32, cov32, expect)
        if iso:
            ok, rv, tv = cv2.solvePnP(pts[None], kp32.astype(np.float64)[None], K, np.zeros((8, 1)), None, None, False,
                                      flags=cv2.SOLVEPNP_ITERATIVE)
            cv_iter[f"noisy_{i}"] = np.concatenate([pn.rodrigues(rv.ravel()), tv.reshape(3, 1)], 1)
            print(f"noisy_{i}: |scipy LM - cv2 ITERATIVE| = {np.abs(expect - cv_iter[f'noisy_{i}']).max():.2e}, cost {0.5 * g @ g:.4f}")
    for k, v in cv_iter.items():
        if v[2, 3] > 0:          # OpenCV's DLT start sometimes lands on the mirrored pose behind the camera: not a check
            cases[k + "_cv2iter"] = v
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pnp_cases.npz"), points_3d=pts, K=K, **cases)
    print("wrote", len(cases), "arrays")


if __name__ == "__main__":
    main()
