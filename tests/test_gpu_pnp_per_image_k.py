"""GPU: pvnet_uncertainty_pnp_per_image_k, the uncertainty PnP with one camera matrix per image (the truncated-LINEMOD
evaluation, where the loader returns a K per image).

- Every image of a per-image-K batch equals, bit for bit, pvnet_uncertainty_pnp called on that image alone with its
  K, and is within 1e-8 of the fp64 oracle (oracle/pnp_oracle.py) on the same float32 inputs.
- A batch whose cameras are all equal gives bit for bit the single-K call's poses and info.
- A K with a zero focal length marks its image (status 4, NaN pose) and leaves the others unchanged.
- Shape errors, no host synchronisation, one launch, and capture + replay in a CUDA graph with K changed between
  replays."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import pnp_oracle as pn
from pvnet_b200 import _native
from pvnet_b200 import extend_utils as eu
from tests import pnp_cases as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 64


def _cameras(rng, n):
    """float64 [n,3,3]: fx in [400, 1200], fy within 10 % of fx, and the principal point anywhere from far outside a
    640x480 image to its centre: cropping an image (the truncated set) shifts it by the crop's offset."""
    fx = rng.uniform(400, 1200, n)
    K = np.zeros((n, 3, 3))
    K[:, 0, 0], K[:, 1, 1] = fx, fx * rng.uniform(0.9, 1.1, n)
    K[:, 0, 2], K[:, 1, 2] = rng.uniform(-200, 840, n), rng.uniform(-150, 630, n)
    K[:, 2, 2] = 1.0
    K[0] = pc.K_LINEMOD                                     # LINEMOD's own camera, and its principal point
    K[1] = pc.K_LINEMOD                                     # moved by a 320x240 crop's offsets
    K[1, 0, 2] -= 160.0
    K[1, 1, 2] -= 120.0
    return K


def _problems(pn_, n=B, seed=0):
    """Noisy problems of one object, each image seen through its own camera.  Covariances are a quarter of
    pnp_cases.random_cov's (about 0.5 px of noise), so that Gauss-Newton ends quadratically and the solver's stopping
    rule leaves the pose within 1e-8 of the minimiser."""
    rng = np.random.default_rng(1000 + 17 * pn_ + seed)
    P = pc.object_points("cloud", pn_, rng)
    Ks = _cameras(rng, n)
    R, t = pc.poses("cloud", n, rng)
    cov = 0.25 * pc.random_cov(rng, (n, pn_))
    uv = np.stack([pc.project(P, R[i:i + 1], t[i:i + 1], Ks[i])[0] for i in range(n)])
    return P, Ks, pc.noisy(rng, uv, cov), cov.astype(np.float32)


def _weights32(cov):
    return pn.covariance_to_weights(cov.reshape(-1, 2, 2)).astype(np.float32).reshape(cov.shape[:-2] + (3,))


def _solve(kp, P, K, entry, cov):
    """One call of uncertainty_pnp_batched: K a host 3x3 (pvnet_uncertainty_pnp) or a CUDA tensor (the per-image
    entry).  entry: 'cov' hands the covariances to the kernel, 'weights_2d' the float32 weights."""
    extra = ({"cov": torch.from_numpy(np.ascontiguousarray(cov)).to(DEV)} if entry == "cov" else
             {"weights_2d": torch.from_numpy(_weights32(cov)).to(DEV)})
    poses, info = eu.uncertainty_pnp_batched(torch.from_numpy(np.ascontiguousarray(kp)).to(DEV), P, K,
                                             return_info=True, **extra)
    return poses.cpu().numpy(), info.cpu().numpy()


def _min_root_gap(kp, w, P, K):
    """Smallest distance between two roots of the Grunert quartic of the P3P start (as in test_gpu_pnp_edges.py)."""
    idxs = np.argsort(w[:, 0].astype(np.float64) + w[:, 1], kind="stable")[-4:]
    uv, Q = kp.astype(np.float64)[idxs], P.astype(np.float64)[idxs]
    f = np.stack([(uv[:, 0] - K[0, 2]) / K[0, 0], (uv[:, 1] - K[1, 2]) / K[1, 1], np.ones(4)], 1)
    f /= np.linalg.norm(f, axis=1, keepdims=True)
    a2, b2, c2 = ((Q[1] - Q[2]) ** 2).sum(), ((Q[0] - Q[2]) ** 2).sum(), ((Q[0] - Q[1]) ** 2).sum()
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    q, p = (a2 - c2) / b2, (a2 + c2) / b2
    coef = [(q - 1) ** 2 - 4 * c2 / b2 * ca * ca,
            4 * (q * (1 - q) * cb - (1 - p) * ca * cg + 2 * c2 / b2 * ca * ca * cb),
            2 * (q * q - 1 + 2 * q * q * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * p * ca * cb * cg
                 + 2 * (b2 - a2) / b2 * cg * cg),
            4 * (-q * (1 + q) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - p) * ca * cg),
            (1 + q) ** 2 - 4 * a2 / b2 * cg * cg]
    r = np.roots(coef)
    return min(abs(a - b) for j, a in enumerate(r) for b in r[j + 1:])


@pytest.mark.parametrize("entry", ["cov", "weights_2d"])
@pytest.mark.parametrize("pn_", [4, 9, 32])
def test_each_image_equals_its_own_single_k_solve_and_the_oracle(pn_, entry):
    """Bit for bit the existing entry on the image alone with its K; 1e-8 from the oracle.  With pn == 4 the answer is
    the P3P pose, and where the quartic has two roots closer than 2e-2 the pose follows the fp64 rounding of its
    coefficients, which device and oracle round differently (test_gpu_pnp_edges.py): those images are held to 1e-4."""
    P, Ks, kp, cov = _problems(pn_)
    poses, info = _solve(kp, P, torch.from_numpy(Ks).to(DEV), entry, cov)
    assert (info[:, 0] == 0).all(), info[info[:, 0] != 0]
    w = pn.covariance_to_weights(cov.reshape(-1, 2, 2)).reshape(B, pn_, 3)
    if entry == "weights_2d":
        w = _weights32(cov)
    P64 = P.astype(np.float64)
    bad = []
    for i in range(B):
        one, one_info = _solve(kp[i:i + 1], P, Ks[i], entry, cov[i:i + 1])
        assert np.array_equal(poses[i], one[0]) and np.array_equal(info[i], one_info[0]), i
        err = np.abs(poses[i] - pn.uncertainty_pnp(kp[i], w[i], P64, Ks[i])).max()
        bar = 1e-8 if pn_ > 4 or _min_root_gap(kp[i], w[i], P, Ks[i]) >= 2e-2 else 1e-4
        if not err <= bar:
            bad.append((i, err, int(info[i, 1])))
    assert not bad, bad


def test_equal_cameras_give_the_single_k_call():
    """All cameras equal, as a CUDA [b,3,3] and as a CUDA [3,3]: the host-K call's poses and info, bit for bit."""
    P, _, kp, cov = _problems(9, seed=1)
    K = pc.K_LINEMOD
    want = _solve(kp, P, K, "cov", cov)
    for k in (torch.from_numpy(np.broadcast_to(K, (B, 3, 3)).copy()).to(DEV), torch.from_numpy(K).to(DEV),
              torch.from_numpy(K).float().to(DEV).expand(B, 3, 3)):
        got = _solve(kp, P, k, "cov", cov)
        if k.dtype == torch.float32:                        # the float32 camera, widened: the same K as a host array
            want_k = _solve(kp, P, K.astype(np.float32).astype(np.float64), "cov", cov)
            assert np.array_equal(got[0], want_k[0]) and np.array_equal(got[1], want_k[1])
        else:
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    # the launch shape switches at 592 images: 1000 images of per-image K equal their own single-K calls in 2 halves
    P, Ks, kp, cov = _problems(9, n=1000, seed=2)
    big = _solve(kp, P, torch.from_numpy(Ks).to(DEV), "cov", cov)
    for s in (slice(0, 8), slice(590, 600), slice(992, 1000)):
        for i in range(s.start, s.stop):
            one = _solve(kp[i:i + 1], P, Ks[i], "cov", cov[i:i + 1])
            assert np.array_equal(big[0][i], one[0][0]) and np.array_equal(big[1][i], one[1][0]), i


def test_invalid_camera_affects_only_its_image():
    """fx == 0 or fy == 0 (what pvnet_uncertainty_pnp refuses for its host K): status 4, NaN pose, iterations 0.
    A NaN K is not refused by that rule: its image finds no P3P start (status 1) and stops.  Every other image keeps
    the pose and info of the all-valid batch."""
    P, Ks, kp, cov = _problems(9, n=16, seed=3)
    base = _solve(kp, P, torch.from_numpy(Ks).to(DEV), "cov", cov)
    bad_k = Ks.copy()
    bad_k[3, 0, 0] = 0.0
    bad_k[7, 1, 1] = 0.0
    bad_k[12] = 0.0
    bad_k[11] = np.nan
    poses, info = _solve(kp, P, torch.from_numpy(bad_k).to(DEV), "cov", cov)
    for i in (3, 7, 12):
        assert info[i, 0] == 4 and info[i, 1] == 0 and np.isnan(poses[i]).all(), (i, info[i])
    assert info[11, 0] & 1, info[11]
    keep = [i for i in range(16) if i not in (3, 7, 11, 12)]
    assert np.array_equal(poses[keep], base[0][keep]) and np.array_equal(info[keep], base[1][keep])


def test_shape_errors_and_null_cameras():
    P, Ks, kp, cov = _problems(9, n=4, seed=4)
    kp_d, cov_d = torch.from_numpy(kp).to(DEV), torch.from_numpy(cov).to(DEV)
    for shape in ((5, 3, 3), (3, 3, 3), (4, 3, 4), (4, 9), (9,), (1, 3, 3)):
        with pytest.raises(ValueError):
            eu.uncertainty_pnp_batched(kp_d, P, torch.ones(shape, dtype=torch.float64, device=DEV), cov=cov_d)
    L = _native.lib()
    out = torch.empty([4, 3, 4], dtype=torch.float64, device=DEV)
    p3 = torch.from_numpy(P).to(DEV)
    assert L.pvnet_uncertainty_pnp_per_image_k(kp_d.data_ptr(), cov_d.data_ptr(), None, p3.data_ptr(), None, 4, 9,
                                               out.data_ptr(), None, None) == -1
    assert b"null" in L.pvnet_last_error()
    k = torch.from_numpy(Ks).to(DEV)
    assert L.pvnet_uncertainty_pnp_per_image_k(kp_d.data_ptr(), cov_d.data_ptr(), None, p3.data_ptr(), k.data_ptr(),
                                               4, 33, out.data_ptr(), None, None) == -1
    torch.cuda.synchronize()


def test_no_host_synchronisation_and_one_launch():
    """CUDA keypoints, covariances, object points and float32 cameras [b,3,3]: no synchronising call (torch's sync
    debug mode raises on one), and one launch of the library for the whole batch."""
    P, Ks, kp, cov = _problems(9, seed=5)
    kp_d, cov_d, p3 = (torch.from_numpy(x).to(DEV) for x in (kp, cov, P))
    k32 = torch.from_numpy(Ks).float().to(DEV)
    for k in (k32, k32[0]):
        eu.uncertainty_pnp_batched(kp_d, p3, k, cov=cov_d)        # warm-up
        torch.cuda.synchronize()
        prev = torch.cuda.get_sync_debug_mode()
        torch.cuda.set_sync_debug_mode("error")
        _native.launch_count_reset()
        try:
            pose = eu.uncertainty_pnp_batched(kp_d, p3, k, cov=cov_d)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
        assert _native.launch_count() == 1
        torch.cuda.synchronize()
        assert torch.isfinite(pose).all()


def test_graph_capture_and_replay_with_changing_cameras():
    """The per-image call captured once into a CUDA graph with a static camera buffer: each replay after a new set of
    cameras is copied into that buffer equals the eager call with those cameras."""
    P, Ks, kp, cov = _problems(9, seed=6)
    rng = np.random.default_rng(6)
    cams = [Ks, _cameras(rng, B), _cameras(rng, B)]
    kp_d, cov_d, p3 = (torch.from_numpy(x).to(DEV) for x in (kp, cov, P))
    k_static = torch.from_numpy(cams[0]).to(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eu.uncertainty_pnp_batched(kp_d, p3, k_static, cov=cov_d, return_info=True)
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        g_pose, g_info = eu.uncertainty_pnp_batched(kp_d, p3, k_static, cov=cov_d, return_info=True)
    for K in cams + cams[:1]:
        k_static.copy_(torch.from_numpy(K).to(DEV))
        g.replay()
        want_pose, want_info = eu.uncertainty_pnp_batched(kp_d, p3, torch.from_numpy(K).to(DEV), cov=cov_d,
                                                          return_info=True)
        torch.cuda.synchronize()
        assert torch.equal(g_pose, want_pose) and torch.equal(g_info, want_info)
    assert not torch.equal(want_pose, eu.uncertainty_pnp_batched(kp_d, p3, torch.from_numpy(cams[1]).to(DEV),
                                                                  cov=cov_d))
