"""GPU: one pose per instance of one class (DESIGN.md §30).

- `pvnet_uncertainty_pnp_instances`: a present row (j < num[b]) is bit for bit what
  `pvnet_uncertainty_pnp_per_image_k` gives for that row with its image's K, in both weight forms, at L = 1, 3 and 32
  (b * L = 1024); an absent row is NaN with info (8, 0); num = 0 everywhere; host and device K agree; graph replay
  with num changed between replays.
- `PoseKeypointPipeline(max_instances=)`: eager and graph replays agree from the same device sampler state, per-batch
  cameras go through `run`, and on planted multi-instance scenes (apart, touching, noisy) the centre split + label
  vote + per-instance PnP finds every instance with its pose within the bounds below."""
import numpy as np
import pytest
import torch

from oracle import pnp_oracle as pn
from pvnet_b200 import extend_utils as eu
from pvnet_b200 import ransac_voting_gpu as rv
from pvnet_b200.pipeline import PoseKeypointPipeline
from tests import instance_pose_cases as ipc
from tests import pnp_cases as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _problems(b, L, pn_, seed):
    """[b,L] noisy problems of one object, image i seen through camera i; num[i] in 0..L with 0 and L both present."""
    rng = np.random.default_rng(seed)
    P = pc.object_points("cloud", pn_, rng)
    Ks = np.repeat(pc.K_LINEMOD[None], b, 0).copy()
    Ks[:, 0, 2] += rng.uniform(-150, 150, b)
    Ks[:, 0, 0] *= rng.uniform(0.9, 1.1, b)
    R, t = pc.poses("cloud", b * L, rng)
    cov = 0.25 * pc.random_cov(rng, (b * L, pn_))
    uv = np.stack([pc.project(P, R[i:i + 1], t[i:i + 1], Ks[i // L])[0] for i in range(b * L)])
    kp = pc.noisy(rng, uv, cov).astype(np.float32).reshape(b, L, pn_, 2)
    num = rng.integers(0, L + 1, b).astype(np.int32)
    num[0], num[-1] = 0, L
    return P, Ks, kp, cov.astype(np.float32).reshape(b, L, pn_, 2, 2), num


def _weights32(cov):
    return pn.covariance_to_weights(cov.reshape(-1, 2, 2)).astype(np.float32).reshape(cov.shape[:-2] + (3,))


@pytest.mark.parametrize("b,L,pn_", [(16, 1, 9), (16, 3, 9), (32, 32, 9), (5, 7, 4), (8, 8, 32)])
@pytest.mark.parametrize("form", ["cov", "weights_2d"])
def test_present_rows_bit_identical_absent_rows_nan(b, L, pn_, form):
    P, Ks, kp, cov, num = _problems(b, L, pn_, seed=100 * L + pn_)
    kp_d = torch.from_numpy(kp).to(DEV)
    arg = cov if form == "cov" else _weights32(cov)
    arg_d = torch.from_numpy(arg).to(DEV)
    num_d = torch.from_numpy(num).to(DEV)
    Kd = torch.from_numpy(Ks).to(DEV)
    pose, info = eu.uncertainty_pnp_instances(kp_d, num_d, P, Kd, **{form: arg_d}, return_info=True)
    # the same rows through the per-image-K entry: every row, with its image's camera repeated
    ref, ref_info = eu.uncertainty_pnp_batched(kp_d.flatten(0, 1), P, Kd.repeat_interleave(L, 0),
                                               **{form: arg_d.flatten(0, 1)}, return_info=True)
    pose, info = pose.cpu().numpy(), info.cpu().numpy()
    ref, ref_info = ref.view(b, L, 3, 4).cpu().numpy(), ref_info.view(b, L, 2).cpu().numpy()
    present = np.arange(L)[None, :] < num[:, None]
    assert present.any() and (~present).any() or L == 1
    assert np.array_equal(pose[present], ref[present])            # bit for bit, NaN-free rows
    assert np.array_equal(info[present], ref_info[present])
    assert np.isfinite(pose[present]).all()
    assert np.isnan(pose[~present]).all()
    assert (info[~present] == [8, 0]).all()


def test_num_zero_everywhere_and_num_above_L():
    b, L = 4, 5
    P, Ks, kp, cov, _ = _problems(b, L, 9, seed=7)
    kp_d, cov_d = torch.from_numpy(kp).to(DEV), torch.from_numpy(cov).to(DEV)
    pose, info = eu.uncertainty_pnp_instances(kp_d, torch.zeros(b, dtype=torch.int32, device=DEV), P, Ks[0],
                                              cov=cov_d, return_info=True)
    assert torch.isnan(pose).all() and (info.cpu() == torch.tensor([8, 0], dtype=torch.int32)).all()
    # num above L: every row is present; a host [3,3] K equals the device [b,3,3] copy of it
    full = torch.full((b,), L + 3, dtype=torch.int32, device=DEV)
    p_host, i_host = eu.uncertainty_pnp_instances(kp_d, full, P, Ks[0], cov=cov_d, return_info=True)
    p_dev, i_dev = eu.uncertainty_pnp_instances(kp_d, full, P, torch.from_numpy(Ks[0]).to(DEV).expand(b, 3, 3),
                                                cov=cov_d, return_info=True)
    assert torch.isfinite(p_host).all() and torch.equal(p_host, p_dev) and torch.equal(i_host, i_dev)
    assert ((i_host[..., 0].cpu() & 8) == 0).all()


def test_invalid_arguments_rejected():
    P, Ks, kp, cov, num = _problems(2, 3, 9, seed=3)
    kp_d, cov_d, num_d = (torch.from_numpy(a).to(DEV) for a in (kp, cov, num))
    with pytest.raises(ValueError):
        eu.uncertainty_pnp_instances(kp_d, num_d, P, Ks[0])                               # no weights
    with pytest.raises(ValueError):
        eu.uncertainty_pnp_instances(kp_d.flatten(0, 1), num_d, P, Ks[0], cov=cov_d)       # not [b,L,pn,2]
    with pytest.raises(ValueError):
        eu.uncertainty_pnp_instances(kp_d, num_d[:1], P, Ks[0], cov=cov_d)                 # num not [b]
    with pytest.raises(ValueError):
        eu.uncertainty_pnp_instances(kp_d, num_d, P, Ks[0], cov=cov_d[:, :2])              # cov not [b,L,pn,2,2]
    with pytest.raises(ValueError):
        eu.uncertainty_pnp_instances(kp_d, num_d, P, np.tile(Ks[0], (3, 1, 1)), cov=cov_d)  # 3 cameras for 2 images
    big = torch.zeros(33, 32, 9, 2, device=DEV)
    with pytest.raises(ValueError):                                                          # b * L > 1024
        eu.uncertainty_pnp_instances(big, torch.zeros(33, dtype=torch.int32, device=DEV), P, Ks[0],
                                     weights_2d=torch.zeros(33, 32, 9, 3, device=DEV))


def test_graph_replay_reads_num_on_the_device():
    b, L = 6, 4
    P, Ks, kp, cov, num = _problems(b, L, 9, seed=11)
    kp_d, cov_d, Kd = torch.from_numpy(kp).to(DEV), torch.from_numpy(cov).to(DEV), torch.from_numpy(Ks).to(DEV)
    num_d = torch.from_numpy(num).to(DEV)
    P_d = torch.from_numpy(P).to(DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eu.uncertainty_pnp_instances(kp_d, num_d, P_d, Kd, cov=cov_d)
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = eu.uncertainty_pnp_instances(kp_d, num_d, P_d, Kd, cov=cov_d)
    torch.cuda.current_stream().wait_stream(s)
    for n in (num, np.full(b, L, np.int32), np.zeros(b, np.int32)):
        num_d.copy_(torch.from_numpy(n))
        g.replay()
        torch.cuda.synchronize()
        want = eu.uncertainty_pnp_instances(kp_d, num_d, P_d, Kd, cov=cov_d)
        assert torch.equal(torch.nan_to_num(out), torch.nan_to_num(want))
        assert torch.isnan(out).all(-1).all(-1).cpu().numpy().tolist() == \
            (np.arange(L)[None] >= n[:, None]).tolist()


class _PlantedNet(torch.nn.Module):
    """Stands in for the backbone: forward_native returns the planted scenes' field and mask (pixel-major, seg_dim 2),
    so the instance step sees known instances."""
    seg_dim = 2

    def __init__(self, scenes):
        super().__init__()
        self.anchor = torch.nn.Parameter(torch.zeros(1, device=DEV))
        f = torch.from_numpy(np.stack([s["field"] for s in scenes])).to(DEV)
        b, h, w = f.shape[:3]
        self.out = torch.cat([torch.zeros(b, h, w, 2, device=DEV), f.flatten(3)], 3).contiguous()
        self.mask = torch.from_numpy(np.stack([s["mask"] for s in scenes])).to(DEV)

    def forward_native(self, x, **kw):
        return self.out, self.mask


def test_pipeline_graph_equals_eager_and_per_batch_cameras():
    """max_instances: on planted scenes (every instance found), eager and graph replays from the same device sampler
    state agree, with and without refinement; per-batch cameras reach the solve."""
    scenes = [ipc.pose_scene(3, 40, touching=True), ipc.pose_scene(2, 41)]
    net = _PlantedNet(scenes)
    pts3d = ipc.POINTS_3D
    hosts = [torch.zeros(2, 480, 640, 3, dtype=torch.uint8).pin_memory() for _ in range(3)]
    rng = np.random.default_rng(2)
    cams = [np.repeat(ipc.K_LINEMOD[None], 2, 0) * rng.uniform(0.95, 1.05, (2, 1, 1)) for _ in hosts]
    for c in cams:
        c[:, 2, 2] = 1.0
    mesh = (np.array([[-0.03, -0.03, 0.0], [0.03, -0.03, 0.0], [0.0, 0.04, 0.0], [0.0, 0.0, 0.03]], np.float32),
            np.array([[0, 1, 2], [0, 1, 3], [1, 2, 3], [0, 2, 3]], np.int32))

    def run(pipe, cameras=None):
        kp = [torch.full([2, 4, 9, 2], float("nan")).pin_memory() for _ in hosts]
        cov = [torch.full([2, 4, 9, 2, 2], float("nan")).pin_memory() for _ in hosts]
        pose = [torch.full([2, 4, 3, 4], float("nan"), dtype=torch.float64).pin_memory() for _ in hosts]
        got = []
        rv.reset_device_rng(DEV)
        pipe.run(hosts, out_host=kp, cov_host=cov, pose_host=pose, camera_matrices=cameras,
                 on_result=lambda i, r: got.append((r[0].clone(), r[1].clone())))
        return kp, cov, pose, got

    for refine in (None, dict(vertices=mesh[0], faces=mesh[1], near=0.05, far=5.0, rounds=2)):
        kw = dict(round_hyp_num=64, with_covariance=True, cov_round_hyp_num=64, cov_min_hyp_num=128,
                  points_3d=pts3d, camera_matrix=ipc.K_LINEMOD, max_instances=4, refine=refine)
        eager = PoseKeypointPipeline(net, **kw)
        graph = PoseKeypointPipeline(net, graph=True, **kw)
        for cameras in (None, cams):
            run(graph, cameras)                  # warm-up + capture
            e = run(eager, cameras)
            g = run(graph, cameras)
            for (la, na), (lb, nb) in zip(e[3], g[3]):
                assert torch.equal(la, lb) and torch.equal(na, nb)
                assert na.cpu().tolist() == [3, 2]   # every planted instance found: nothing below is vacuous
            for a, b in zip(e[:3], g[:3]):
                for x, y in zip(a, b):
                    assert torch.equal(torch.nan_to_num(x), torch.nan_to_num(y))
            assert torch.isfinite(e[2][-1][0, :3]).all() and torch.isfinite(e[2][-1][1, :2]).all()
            if refine is None and cameras is not None:
                kp, cov, pose, got = e
                want = eu.uncertainty_pnp_instances(kp[-1].to(DEV), got[-1][1], pts3d, cams[-1], cov=cov[-1].to(DEV))
                assert torch.equal(torch.nan_to_num(want.cpu()), torch.nan_to_num(pose[-1]))


# Measured on the seeds below (NVIDIA H100 80GB HBM3 at 700 W): worst case 0.87 deg and 3.5 mm (DESIGN.md §30).  The
# bounds leave headroom above it.
ROT_BOUND_DEG, T_BOUND_M = 1.5, 0.01


@pytest.mark.parametrize("n,touching,sigma,seed", [(1, False, 0.0, 1), (3, False, 0.0, 2), (2, True, 0.0, 3),
                                                   (4, True, 0.0, 4), (3, True, 0.03, 5), (5, False, 0.03, 6)])
def test_planted_scenes_every_instance_found_and_posed(n, touching, sigma, seed, record_property):
    s = ipc.pose_scene(n, seed, sigma=sigma, touching=touching)
    if touching:
        assert ipc.touching_pairs(s["gt"])
    I = 8
    mask = torch.from_numpy(s["mask"][None]).to(DEV)
    vertex = torch.from_numpy(s["field"][None]).to(DEV)
    rv.reset_device_rng(DEV)
    labels, num = rv.ransac_voting_center(mask, vertex[..., -1, :], 256, 0.99, max_instances=I)
    kp, cov = rv.ransac_voting_labels(labels, vertex, I, 256, 0.99, True)
    pose, info = eu.uncertainty_pnp_instances(kp, num, ipc.POINTS_3D, ipc.K_LINEMOD, cov=cov, return_info=True)
    assert int(num[0]) == n
    pose, lab = pose[0].cpu().numpy(), labels[0].cpu().numpy()
    assert np.isnan(pose[n:]).all() and (info[0, n:, 0].cpu() == 8).all()
    errs = []
    for j in range(n):
        # the ground-truth instance this label covers most of
        g = np.bincount(s["gt"][lab == j + 1], minlength=n + 1)[1:].argmax()
        errs.append(ipc.pose_errors(pose[j, :, :3], pose[j, :, 3], s["R"][g], s["t"][g]))
    errs = np.array(errs)
    record_property("rot_deg_max", float(errs[:, 0].max()))
    record_property("t_m_max", float(errs[:, 1].max()))
    print(f"instances={n} touching={touching} sigma={sigma}: rot deg mean {errs[:, 0].mean():.4f} max "
          f"{errs[:, 0].max():.4f}, t mm mean {1e3 * errs[:, 1].mean():.3f} max {1e3 * errs[:, 1].max():.3f}")
    assert errs[:, 0].max() < ROT_BOUND_DEG and errs[:, 1].max() < T_BOUND_M
