"""GPU: `pvnet_epnp` / `pvnet_epnp_per_image_k` (csrc/epnp.cu) behind `pnp(..., method=SOLVEPNP_EPNP)`.

- Against the fp64 oracle (oracle/epnp_oracle.py) on the same float32 inputs to 1e-10, and against OpenCV's poses in
  tests/golden/epnp_cases.npz to 1e-9, except images whose eigen-gap is below GAP_MIN (their number is pinned).
- info[:,1] is the oracle's N; R is a rotation to 1e-12; coplanar points get status 1.
- Point counts 4..4096 and batch sizes 1, 592 (one CTA per image) and past the four-warp switch.
- The per-image-K entry equals the single-K entry bit for bit; a zero focal length marks only its image; a NaN
  keypoint leaves the other images alone; argument errors; run-to-run identity; no host synchronisation; graph
  capture and replay; `pnp` through lib.utils.evaluation_utils, batched and numpy."""
import numpy as np
import pytest
import torch

from oracle import epnp_oracle as eo
from pvnet_b200 import _native
from pvnet_b200 import evaluation as ev
from tests import epnp_cases as ec
from tests import pnp_cases as pc
from tests.test_epnp_oracle_cpu import GAP_MIN, GOLDEN, pose_diff

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# images excluded from the device-vs-oracle and device-vs-cv2 pose bars: an eigen-gap below GAP_MIN (all have 5
# points); an N-selection tie only excuses a different N, the pose is still held to the bars
N_DEVICE_EXCLUDED = 120


def _solve(x, P, K, info=True):
    return ev._epnp_batched(torch.from_numpy(np.ascontiguousarray(x)).to(DEV), P, K, return_info=info)


def test_device_matches_oracle_and_cv2():
    excluded, bad = 0, []
    for name in ec.names():
        pr = ec.problem(name)
        poses, info = (t.cpu().numpy() for t in _solve(pr["x"], pr["P"], pr["K"]))
        for i in range(ec.BATCH):
            o = eo.epnp(pr["x"][i], pr["P"], pr["K"])
            R = poses[i, :, :3]
            assert np.abs(R @ R.T - np.eye(3)).max() < 1e-12, (name, i)
            assert info[i, 0] == o["status"], (name, i, info[i], o["status"])
            if name.startswith("coplanar"):
                assert info[i, 0] & 1
                continue
            if "/pn4/" in name:
                continue
            if o["gap"] < GAP_MIN:
                excluded += 1
                continue
            n_ok = info[i, 1] == o["N"] or eo.selection_tie(o["errors"])
            if not n_ok or not pose_diff(poses[i], o["pose"]) <= 1e-10 or \
                    not pose_diff(poses[i], GOLDEN[ec.key(name)][i]) <= 1e-9:
                bad.append((name, i, int(info[i, 1]), o["N"], pose_diff(poses[i], o["pose"])))
    assert not bad, bad
    assert excluded == N_DEVICE_EXCLUDED


@pytest.mark.parametrize("b", [1, 592, 593, 1500])
def test_batch_sizes_and_per_image_k(b):
    rng = np.random.default_rng(b)
    P = pc.object_points("cloud", 9, rng)
    Ks = np.stack([pc.camera("cloud", rng) for _ in range(b)])
    R, t = pc.poses("cloud", b, rng)
    x = np.stack([pc.project(P, R[i:i + 1], t[i:i + 1], Ks[i])[0] for i in range(b)])
    x = (x + rng.normal(0, 1.0, x.shape)).astype(np.float32)
    poses, info = _solve(x, P, torch.from_numpy(Ks).to(DEV))
    poses, info = poses.cpu().numpy(), info.cpu().numpy()
    for i in sorted({0, b // 2, b - 1, min(b - 1, 591), min(b - 1, 592)}):
        one, one_info = _solve(x[i:i + 1], P, Ks[i])
        assert np.array_equal(poses[i], one.cpu().numpy()[0]) and np.array_equal(info[i], one_info.cpu().numpy()[0])
        o = eo.epnp(x[i], P, Ks[i])
        assert pose_diff(poses[i], o["pose"]) <= 1e-10 or o["gap"] < GAP_MIN


@pytest.mark.parametrize("pn_", list(range(4, 41)) + [63, 64, 65, 255, 256, 1000, 4095, 4096])
def test_point_counts(pn_):
    rng = np.random.default_rng(100 + pn_)
    P = pc.object_points("cloud", pn_, rng)
    K = pc.camera("cloud", rng)
    R, t = pc.poses("cloud", 4, rng)
    x = (pc.project(P, R, t, K) + rng.normal(0, 1.0, (4, pn_, 2))).astype(np.float32)
    poses, info = (a.cpu().numpy() for a in _solve(x, P, K))
    for i in range(4):
        Rm = poses[i, :, :3]
        assert np.abs(Rm @ Rm.T - np.eye(3)).max() < 1e-12
        if pn_ > 4:
            o = eo.epnp(x[i], P, K)
            if not o["gap"] < GAP_MIN:
                assert pose_diff(poses[i], o["pose"]) <= 1e-10, (pn_, i)
                assert info[i, 1] == o["N"] or eo.selection_tie(o["errors"]), (pn_, i)


def test_bad_camera_and_nan_keypoint_affect_only_their_image():
    pr = ec.problem("cloud/pn9/s1")
    Ks = np.broadcast_to(pr["K"], (ec.BATCH, 3, 3)).copy()
    base = [a.cpu().numpy() for a in _solve(pr["x"], pr["P"], torch.from_numpy(Ks).to(DEV))]
    Ks[2, 0, 0] = 0.0
    Ks[5, 1, 1] = 0.0
    x = pr["x"].copy()
    x[6, 3, 0] = np.nan
    poses, info = (a.cpu().numpy() for a in _solve(x, pr["P"], torch.from_numpy(Ks).to(DEV)))
    for i in (2, 5):
        assert info[i, 0] == 4 and np.isnan(poses[i]).all()
    keep = [0, 1, 3, 4, 7]
    assert np.array_equal(poses[keep], base[0][keep]) and np.array_equal(info[keep], base[1][keep])
    with pytest.raises(RuntimeError):                       # a host K with a zero focal length is refused
        _solve(pr["x"], pr["P"], np.diag([0.0, 500.0, 1.0]))


def test_argument_errors():
    pr = ec.problem("cloud/pn9/s1")
    x = torch.from_numpy(pr["x"]).to(DEV)
    with pytest.raises(ValueError):
        ev.pnp(pr["P"][:3], x[:, :3], pr["K"], method=ev.SOLVEPNP_EPNP)
    for shape in ((5, 3, 3), (4, 9), (3, 4)):
        with pytest.raises(ValueError):
            ev.pnp(pr["P"], x, torch.ones(shape, dtype=torch.float64, device=DEV), method=ev.SOLVEPNP_EPNP)
    with pytest.raises(ValueError):
        ev.pnp(pr["P"], x, pr["K"], method=2)
    L = _native.lib()
    out = torch.empty([8, 3, 4], dtype=torch.float64, device=DEV)
    p3 = torch.from_numpy(pr["P"]).to(DEV)
    assert L.pvnet_epnp_per_image_k(x.data_ptr(), p3.data_ptr(), None, 8, 9, out.data_ptr(), None, None) == -1
    k = torch.from_numpy(np.broadcast_to(pr["K"], (8, 3, 3)).copy()).to(DEV)
    assert L.pvnet_epnp_per_image_k(x.data_ptr(), p3.data_ptr(), k.data_ptr(), 8, 4097, out.data_ptr(), None,
                                    None) == -1
    assert L.pvnet_epnp_per_image_k(x.data_ptr(), p3.data_ptr(), k.data_ptr(), 8, 3, out.data_ptr(), None, None) == -1
    torch.cuda.synchronize()


def test_run_to_run_identical_no_sync_and_graph_replay():
    pr = ec.problem("mm/pn100/s3")
    x, p3 = torch.from_numpy(pr["x"]).to(DEV), torch.from_numpy(pr["P"]).to(DEV)
    k = torch.from_numpy(np.broadcast_to(pr["K"], (ec.BATCH, 3, 3)).copy()).to(DEV)
    first = ev.pnp(p3, x, k, method=ev.SOLVEPNP_EPNP)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    _native.launch_count_reset()
    try:
        again = ev.pnp(p3, x, k, method=ev.SOLVEPNP_EPNP)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert _native.launch_count() == 1
    torch.cuda.synchronize()
    assert torch.equal(first, again)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ev.pnp(p3, x, k, method=ev.SOLVEPNP_EPNP)
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        g_pose = ev.pnp(p3, x, k, method=ev.SOLVEPNP_EPNP)
    other = ec.problem("mm/pn100/s1")["x"]
    for xs in (other, pr["x"]):
        x.copy_(torch.from_numpy(xs).to(DEV))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(g_pose, ev.pnp(p3, x, k, method=ev.SOLVEPNP_EPNP))


def test_through_the_reference_module():
    """`pnp` as the reference's module exports it: the batched CUDA form with method=1 gives the fixture's cv2 pose;
    the single-image numpy form keeps method 0 only and raises for method 1, as it did before EPnP existed."""
    from lib.utils.evaluation_utils import pnp
    pr = ec.problem("cat/pn9/s1")
    got = pnp(pr["P"], torch.from_numpy(pr["x"]).to(DEV), pr["K"], method=1)
    assert got.is_cuda and got.dtype == torch.float64 and tuple(got.shape) == (ec.BATCH, 3, 4)
    for i in range(ec.BATCH):
        assert pose_diff(got[i].cpu().numpy(), GOLDEN[ec.key("cat/pn9/s1")][i]) <= 1e-9
    with pytest.raises(ValueError):
        pnp(pr["P"], pr["x"][0], pr["K"], method=1)
