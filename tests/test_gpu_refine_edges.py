"""GPU: `pvnet_b200.refine.refine_poses` (csrc/refine.cu) against oracle/refine_oracle.py where the kernel's own
structure shows -- several 2 048-point contour tiles and a tie across two of them, one or many pair blocks per image,
the gate at a whole-number distance, speckled, holed and border-cut masks, odd image sizes, the accept / undo
decision at 480x640 with a 20 480-face mesh, the SINGULAR status, and mask dtypes.  The oracle renders with
`render_mesh` (tests/refine_cases.device_depth), which tests/test_gpu_render.py pins to its own renderer; the rest
of each round is the oracle's numpy.  First-round stages are compared bit for bit and the normal equations to
1e-12; over the rounds, each pose to 1e-9 and the status, pair count and mean distances bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import refine_oracle as rfo
from pvnet_b200 import _native, refine
from pvnet_b200.render import render_mesh
from tests import refine_cases as rf
from tests import render_cases as rc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RENDER = rf.device_depth(DEV)
TOOL = rf.tool_mesh()


def t(a, dtype=None):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def coverage(mesh, K, P, h, w):
    """bool [b,h,w] numpy: the mesh's coverage at poses P [b,3,4] by the device renderer."""
    return (render_mesh(t(mesh[0]), t(mesh[1]), t(K), t(P, torch.float32), h, w, rf.NEAR, rf.FAR) > 0).cpu().numpy()


def kof(K, i):
    return K if K.ndim == 2 else K[i]


def check_first_round(mesh, mask, P0, K, max_points=4096, gate=20.0, stale=None):
    """The first round's stages of every image against the oracle's -> the oracle's first-round records.  stale: an
    int32 to fill a freed block of the call's workspace size with first, so that the call's workspace (the caching
    allocator hands that block back) holds it wherever the kernels have not written."""
    h, w = mask.shape[1:]
    if stale is not None:
        need = ctypes.c_size_t()
        _native.check(_native.lib().pvnet_refine_workspace_bytes(len(P0), h, w, max_points, ctypes.byref(need)),
                      "pvnet_refine_workspace_bytes")
        torch.full((need.value // 4,), stale, dtype=torch.int32, device=DEV)
    _, _, tr = refine.refine_poses(t(mask, torch.uint8), t(P0), t(K), t(mesh[0]), t(mesh[1]), rf.NEAR, rf.FAR,
                                   rounds=1, gate=gate, max_points=max_points, return_info=True, trace=True)
    tr = {k: x.cpu().numpy() for k, x in tr.items()}
    recs = []
    for i in range(len(P0)):
        orec = []
        rfo.refine_image(mask[i], P0[i], kof(K, i), *mesh, rf.NEAR, rf.FAR, rounds=1, gate=gate,
                         max_points=max_points, trace=orec, render=RENDER)
        o = orec[0]
        ns, nc = tr["counts"][i]
        assert ns == len(o["sil"]) and nc == len(o["con"]), (i, ns, nc, len(o["sil"]), len(o["con"]))
        assert np.array_equal(tr["sil_idx"][i, :ns], o["sil"]), i
        assert np.array_equal(tr["con_idx"][i, :nc], o["con"]), i
        assert np.array_equal(tr["sil_obj"][i, :ns], o["X"]), i
        assert np.array_equal(tr["pair_idx"][i, :ns], o["pair"]), i
        if o["normal_eq"]:
            A, g = o["normal_eq"][0]
            ne = tr["normal_eq"][i]
            Ad = np.zeros((6, 6))
            Ad[np.triu_indices(6)] = ne[:21]
            Ad = Ad + np.triu(Ad, 1).T
            assert np.abs(Ad - A).max() <= 1e-12 * np.abs(A).max(), i
            assert np.abs(ne[21:] - g).max() <= 1e-12 * np.abs(g).max(), i
        recs.append(o)
    return recs


def same(a, b):
    return a == b or (np.isnan(a) and np.isnan(b))


def check_every_round(mesh, mask, P0, K, images=None, rounds=8, gate=20.0, max_points=4096):
    """For k = 0..rounds: the k-round call's poses of `images` to 1e-9, and status, pairs and mean distances bit for
    bit -> the oracle's (pose, info, trace) of the full call per image."""
    images = range(len(P0)) if images is None else images
    m, p, k, v, f = t(mask), t(P0), t(K), t(mesh[0]), t(mesh[1])
    full = {}
    for r in range(rounds + 1):
        out, info = refine.refine_poses(m, p, k, v, f, rf.NEAR, rf.FAR, rounds=r, gate=gate, max_points=max_points,
                                        return_info=True)
        out = out.cpu().numpy()
        info = {key: x.cpu().numpy() for key, x in info.items()}
        for i in images:
            tr = []
            P, oi = rfo.refine_image(mask[i], P0[i], kof(K, i), *mesh, rf.NEAR, rf.FAR, rounds=r, gate=gate,
                                     max_points=max_points, trace=tr, render=RENDER)
            assert np.abs(out[i] - P).max() <= 1e-9, (r, i)
            assert info["status"][i] == oi["status"] and info["pairs"][i] == oi["pairs"], (r, i, info["status"][i], oi)
            for key in ("dist_before", "dist_after"):
                assert same(float(info[key][i]), oi[key]), (r, i, key, float(info[key][i]), oi[key])
            if r == rounds:
                full[i] = (P, oi, tr)
    return full


# ---- first-round stages ----

H, W = 480, 640


def tool_scene(b, seed, h=H, w=W, K=rc.K_LINEMOD):
    rng = np.random.default_rng(seed)
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    return Pt, P0, coverage(TOOL, K, Pt, h, w)


@pytest.mark.parametrize("max_points", [4096, 10000])
def test_contour_counts_across_tiles(max_points):
    """Contours of 2 047 to 6 145 points, so the pair search walks one to four 2 048-point tiles, a last tile of one
    point, and the stride rule at 4 096."""
    counts = (2047, 2048, 2049, 4096, 4097, 6145)
    Pt, P0, on = tool_scene(len(counts), 101)
    mask = np.stack([rf.with_contour_count(on[i], n, holes=50 * i, seed=i) for i, n in enumerate(counts)])
    recs = check_first_round(TOOL, mask, P0, rc.K_LINEMOD, max_points=max_points)
    for n, o in zip(counts, recs):
        assert len(o["con"]) == -(-n // max(1, -(-n // max_points)))
    assert max(o["pair"].max() for o in recs) >= 2048                          # pairs found past the first tile


def test_contour_entries_past_the_count_are_never_read():
    """A contour of 2 049 points: the second tile holds one.  The workspace past it is filled with the index of a
    silhouette pixel that is not on the contour, so a pair search that read past the count would find it at d2 = 0."""
    Pt, P0, on = tool_scene(1, 104)
    mask = rf.with_contour_count(on[0], 2049, seed=1)[None]
    depth0 = render_mesh(t(TOOL[0]), t(TOOL[1]), t(rc.K_LINEMOD), t(P0, torch.float32), H, W, rf.NEAR,
                         rf.FAR).cpu().numpy()[0]
    off = np.setdiff1d(rfo.boundary(depth0 > 0), rfo.boundary(mask[0]))
    assert len(off)
    (o,) = check_first_round(TOOL, mask, P0, rc.K_LINEMOD, stale=int(off[0]))
    assert len(o["con"]) == 2049 and o["d2"][np.searchsorted(o["sil"], off[0])] > 0


def test_a_tie_across_two_tiles_keeps_the_lower_index():
    Pt, P0, on = tool_scene(2, 102)
    depth0 = render_mesh(t(TOOL[0]), t(TOOL[1]), t(rc.K_LINEMOD), t(P0, torch.float32), H, W, rf.NEAR,
                         rf.FAR).cpu().numpy()
    mask, ties = [], []
    for i in range(2):
        m, s, lo, hi = rf.straddling_tie(on[i], depth0[i], P0[i], rc.K_LINEMOD)
        assert lo == 2047 and hi >= 2048
        mask.append(m)
        ties.append((s, lo))
    recs = check_first_round(TOOL, np.stack(mask), P0, rc.K_LINEMOD)
    for o, (s, lo) in zip(recs, ties):
        assert o["pair"][s] == lo


def first_count(on, n):
    hit = [i for i, x in enumerate(on) if len(rfo.boundary(x)) == n]
    assert hit, n
    return hit[0]


def test_silhouettes_of_256_257_and_more_than_4096_points():
    """One pair block exactly full, one block plus one point, and (max_points 10 000) 17 or more blocks."""
    h, w = 96, 128
    K = rc.camera_for(h, w, 300.0)
    zs = np.linspace(0.43, 0.45, 201)                                          # the tool's silhouette: 266 .. 250 points
    P = np.zeros((len(zs), 3, 4))
    P[:, :, :3] = rf.axis_angle([0.3, -0.2, 0.1])
    P[:, 2, 3] = zs
    cov = coverage(TOOL, K, P, h, w)
    picks = [first_count(cov, 256), first_count(cov, 257)]
    P0 = P[picks]
    truth = rf.perturb(P0, np.random.default_rng(5), 2.0, 0.005)
    recs = check_first_round(TOOL, coverage(TOOL, K, truth, h, w), P0, K)
    assert [len(o["sil"]) for o in recs] == [256, 257]
    comb = rf.comb_mesh()
    P0 = np.zeros((2, 3, 4))
    P0[:, :, :3] = [rf.axis_angle([0.05, -0.04, 0.02]), rf.axis_angle([-0.03, 0.06, -0.05])]
    P0[:, :, 3] = [(-0.12, -0.09, 0.5), (-0.11, -0.1, 0.55)]
    truth = rf.perturb(P0, np.random.default_rng(6), 1.0, 0.003)
    recs = check_first_round(comb, coverage(comb, rc.K_LINEMOD, truth, H, W), P0, rc.K_LINEMOD, max_points=10000)
    assert all(len(o["sil"]) > 4096 for o in recs), [len(o["sil"]) for o in recs]


def test_gate_at_a_whole_number_distance():
    """In the first round each silhouette point projects back onto its own pixel centre, so d2 is a whole number:
    with gate 3, pairs at d2 == 9 are kept and pairs at d2 == 10 dropped."""
    h, w = 120, 160
    K = rc.camera_for(h, w, 300.0)
    P0 = rf.true_poses(2, np.random.default_rng(3))
    mask = np.roll(coverage(TOOL, K, P0, h, w), (1, 3), axis=(1, 2))          # one row down, three columns right
    recs = check_first_round(TOOL, mask, P0, K, gate=3.0)
    d2 = np.concatenate([o["d2"] for o in recs])
    pair = np.concatenate([o["pair"] for o in recs])
    assert (d2 == 9).any() and (pair[d2 == 9] >= 0).all()
    assert (d2 == 10).any() and (pair[d2 == 10] == -1).all()


# ---- every round ----

def test_batch_of_64_at_full_size_with_undone_and_degenerate_images():
    """480x640, per-image K about LINEMOD's, a 20 480-face mesh, b = 64.  Images 0-2 start at the truth with a bar
    stuck to the mask, so their first round is undone (REJECTED after one round); image 3's mask is a blob far from
    the render (FEW_PAIRS); images 4 and 5 are speckled and holed; the rest are the truth's coverage from starts
    3 degrees and 1 cm away."""
    b = 64
    rng = np.random.default_rng(2024)
    mesh = rf.lumpy_mesh(5)
    assert len(mesh[1]) == 20480
    Pt = rf.true_poses(b, rng)
    P0 = rf.perturb(Pt, rng)
    P0[:3] = Pt[:3]
    K = np.repeat(rc.K_LINEMOD[None], b, 0).astype(np.float64)
    K[:, 0, 0] *= rng.uniform(0.95, 1.05, b)
    K[:, 1, 1] *= rng.uniform(0.95, 1.05, b)
    K[:, :2, 2] += rng.normal(0, 3.0, (b, 2))
    K = K.astype(np.float32)
    mask = coverage(mesh, K, Pt, H, W)
    for i in range(3):
        mask[i] = rf.spur(mask[i])
    mask[3] = False
    mask[3, :6, :6] = True
    mask[4] = rf.with_contour_count(mask[4], 4097, holes=150, seed=4)
    mask[5] = rf.with_contour_count(mask[5], 6145, holes=300, seed=5)
    full = check_every_round(mesh, mask, P0, K, images=(0, 1, 2, 3, 4, 5, 17, 40, 63))
    undone = [i for i in (0, 1, 2) if full[i][1]["status"] == rfo.REJECTED and len(full[i][2]) == 2]
    assert undone, {i: (full[i][1], len(full[i][2])) for i in (0, 1, 2)}
    assert full[3][1]["status"] == rfo.FEW_PAIRS
    assert all(full[i][1]["status"] & ~rfo.REJECTED == 0 for i in (4, 5, 17, 40, 63))


def test_objects_cut_by_the_image_border():
    """A tool wider than the image (cut on the left and the right), and tools cut by the right, top and bottom-left
    borders: the boundary rules at r == 0, r == h - 1, c == 0 and c == w - 1 decide the cut pixels."""
    h, w = 120, 160
    K = rc.camera_for(h, w, 300.0)
    Pt = np.zeros((4, 3, 4))
    for i, wv in enumerate(([0.1, 0.05, 0.02], [0.2, -0.1, 0.3], [-0.15, 0.1, 0.05], [0.05, 0.2, -0.1])):
        Pt[i, :, :3] = rf.axis_angle(wv)
    Pt[:, :, 3] = [(0.0, 0.0, 0.2), (0.07, 0.0, 0.4), (0.0, -0.085, 0.4), (-0.065, 0.07, 0.35)]
    P0 = rf.perturb(Pt, np.random.default_rng(8), 2.0, 0.005)
    mask = coverage(TOOL, K, Pt, h, w)
    assert mask[0][:, 0].any() and mask[0][:, -1].any() and mask[1][:, -1].any() and mask[2][0].any()
    assert mask[3][-1].any() and mask[3][:, 0].any()
    check_first_round(TOOL, mask, P0, K)
    check_every_round(TOOL, mask, P0, K, rounds=5)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 37), (37, 1), (61, 47)])
def test_odd_image_sizes(h, w):
    K = rc.camera_for(h, w, 2.5 * max(h, w, 8))
    rng = np.random.default_rng(h * 100 + w)
    Pt = np.zeros((2, 3, 4))
    for i in range(2):
        Pt[i, :, :3] = rf.axis_angle(rng.normal(0, 0.2, 3))
    Pt[:, :, 3] = [(0.0, 0.0, 0.45), (0.01, -0.005, 0.5)]
    P0 = rf.perturb(Pt, rng, 2.0, 0.005)
    mask = coverage(TOOL, K, Pt, h, w)
    assert mask.any()
    check_every_round(TOOL, mask, P0, K, rounds=4)


def test_singular_normal_equations_keep_the_input_pose():
    """The scene whose normal equations have an exactly zero row (tests/refine_cases.singular_scene) next to an
    ordinary image: the kernel sets SINGULAR, keeps that image's input pose, and refines the other as the oracle does."""
    mesh, Ks, pose, m = rf.singular_scene()
    v, f = mesh
    out, info = refine.refine_poses(t(m[None], torch.uint8), t(pose[None]), t(Ks), t(v), t(f), 0.05, 5.0,
                                    return_info=True)
    P, oi = rfo.refine_image(m, pose, Ks, v, f, 0.05, 5.0, render=RENDER)
    assert oi["status"] == rfo.SINGULAR
    assert int(info["status"][0]) == refine.SINGULAR and int(info["pairs"][0]) == oi["pairs"] == 6
    assert np.array_equal(out[0].cpu().numpy(), pose)
    assert float(info["dist_before"][0]) == float(info["dist_after"][0]) == 0.0


# ---- mask dtypes ----

def test_nonzero_int64_and_strided_bool_masks_are_foreground():
    """The contract is "nonzero": an int64 mask of 256 (whose low byte is 0) and a non-contiguous bool view give the
    uint8 mask's result bit for bit."""
    h, w = 120, 160
    K = rc.camera_for(h, w, 300.0)
    Pt, P0, on = tool_scene(3, 103, h, w, K)
    on = np.stack([rf.with_contour_count(x, len(rfo.boundary(x)) + 200, holes=20, seed=i) for i, x in enumerate(on)])
    args = (t(P0), t(K), t(TOOL[0]), t(TOOL[1]), rf.NEAR, rf.FAR)
    ref, ri = refine.refine_poses(t(on, torch.uint8), *args, return_info=True)
    wide = torch.zeros((3, h, 2 * w), dtype=torch.bool, device=DEV)
    wide[:, :, ::2] = t(on)
    for m in (t(on, torch.int64) * 256, wide[:, :, ::2]):
        assert m.dtype == torch.bool or int(m.max()) == 256
        out, oi = refine.refine_poses(m, *args, return_info=True)
        assert torch.equal(out, ref) and all(torch.equal(oi[k], ri[k]) for k in ri)
    P, oinfo = rfo.refine(on, P0, K, *TOOL, rf.NEAR, rf.FAR, render=RENDER)
    assert np.abs(ref.cpu().numpy() - P).max() <= 1e-9
    assert np.array_equal(ri["status"].cpu().numpy(), oinfo["status"])
