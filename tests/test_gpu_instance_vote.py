"""GPU: `pvnet_ransac_voting_center` / `ransac_voting_center` (DESIGN.md section 29) against
oracle/instance_vote_oracle.py -- every round's counts, hypotheses, list lengths and winners bit for bit, the
label map bit for bit given the kernel's centres, the centres to the refit tolerance -- plus the edge cases,
the strided NCHW view, the device sampler and CUDA-graph replay."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import instance_vote_oracle as iv
from pvnet_b200 import _native
from pvnet_b200 import ransac_voting_gpu as rv
from tests.instance_vote_cases import draw_center_idxs, instance_scene, match_ids

pytestmark = pytest.mark.gpu

THRESH, MIN_NUM = 0.99, 100


def _run(mask, field, hn, I, idxs=None, min_num=MIN_NUM, rng="device"):
    lab, num, dbg = rv.ransac_voting_center(mask, field, hn, THRESH, min_num=min_num, max_instances=I,
                                            idxs=None if idxs is None else torch.as_tensor(idxs, device="cuda"),
                                            rng=rng, return_debug=True)
    torch.cuda.synchronize()
    return lab.cpu().numpy(), num.cpu().numpy(), {k: v.cpu().numpy() for k, v in dbg.items() if v is not None}


def _check(mask_np, field_np, idxs, lab, num, dbg, min_num=MIN_NUM):
    for bi in range(mask_np.shape[0]):
        o = iv.center_search(mask_np[bi], field_np[bi], idxs[bi], THRESH, min_num, centers_for_assign=dbg["centers"][bi])
        assert num[bi] == o["num"], bi
        np.testing.assert_array_equal(dbg["tn"][bi], o["tn"])
        np.testing.assert_array_equal(dbg["counts"][bi], o["counts"])
        np.testing.assert_array_equal(dbg["hyp"][bi], o["hyp"])
        np.testing.assert_array_equal(dbg["win_counts"][bi], o["win_counts"])
        np.testing.assert_allclose(dbg["centers"][bi], o["centers"], atol=1e-4, rtol=1e-5)
        assert np.all(dbg["centers"][bi, o["num"]:] == 0)
        np.testing.assert_array_equal(lab[bi], o["labels"])


def _scenes(specs, h=480, w=640):
    sc = [instance_scene(n, seed, h=h, w=w, sigma=sig, touching=t, radius=r) for n, seed, sig, t, r in specs]
    mask = np.stack([s["mask"] for s in sc])
    field = np.stack([s["field"][:, :, -1] for s in sc])
    return sc, mask, field


def test_oracle_parity_480x640():
    specs = [(1, 11, 0.0, False, (40, 70)), (3, 2, 0.0, False, (40, 70)), (5, 6, 0.03, True, (40, 70)),
             (4, 4, 0.0, True, (40, 70))]
    _, mask, field = _scenes(specs)
    idxs = draw_center_idxs(len(specs), 8, 256, 5)
    lab, num, dbg = _run(torch.from_numpy(mask).cuda(), torch.from_numpy(field).cuda(), 256, 8, idxs)
    _check(mask, field, idxs, lab, num, dbg)
    assert list(num) == [1, 3, 5, 4]


@pytest.mark.parametrize("dtype", ["uint8", "bool", "int64"])
def test_mask_dtypes_and_low_byte(dtype):
    _, mask, field = _scenes([(3, 2, 0.03, False, (40, 70))])
    idxs = draw_center_idxs(1, 4, 128, 1)
    m = torch.from_numpy(mask).cuda()
    if dtype == "bool":
        m = m.bool()
    elif dtype == "int64":
        m = m.long() * 3                    # low byte 3: foreground
        m[0, :40] = 256                     # low byte 0: background, as `.byte()` reads it
    ref_mask = m.cpu().numpy()
    lab, num, dbg = _run(m, torch.from_numpy(field).cuda(), 128, 4, idxs)
    _check(ref_mask, field, idxs, lab, num, dbg)


def test_strided_nchw_view_equals_contiguous():
    sc, mask, _ = _scenes([(3, 5, 0.03, False, (40, 70))])
    k = sc[0]["field"].shape[2]
    nchw = torch.from_numpy(np.ascontiguousarray(sc[0]["field"].reshape(480, 640, 2 * k).transpose(2, 0, 1)))[None]
    vertex = nchw.cuda().permute(0, 2, 3, 1).view(1, 480, 640, k, 2)       # the [b,h,w,k,2] view of the head
    view = vertex[..., -1, :]
    assert not view.is_contiguous()
    idxs = draw_center_idxs(1, 4, 256, 3)
    a = _run(torch.from_numpy(mask).cuda(), view, 256, 4, idxs)
    b = _run(torch.from_numpy(mask).cuda(), view.contiguous(), 256, 4, idxs)
    for x, y in zip(a[:2], b[:2]):
        np.testing.assert_array_equal(x, y)
    for key in a[2]:
        np.testing.assert_array_equal(a[2][key], b[2][key])
    _check(mask, sc[0]["field"][None, :, :, -1], idxs, *a)


def test_edge_cases():
    sc, mask, field = _scenes([(5, 3, 0.0, False, (40, 70))] * 5)
    mask[0] = 0                                                  # empty image
    mask[1] = 0
    mask[1, 100:105, 100:110] = 1                                # 50 < min_num foreground pixels
    idxs = draw_center_idxs(5, 3, 256, 9)                        # five objects, three instances at most
    lab, num, dbg = _run(torch.from_numpy(mask).cuda(), torch.from_numpy(field).cuda(), 256, 3, idxs)
    _check(mask, field, idxs, lab, num, dbg)
    assert num[0] == 0 and num[1] == 0 and np.all(lab[:2] == 0) and np.all(dbg["tn"][0] == 0)
    assert dbg["tn"][1, 0] == 50 and num[2] == 3
    # the winning count falling under min_num stops the search: choose min_num between two winners' counts
    w = dbg["win_counts"][2]
    mn = int(w[1]) + 1
    lab2, num2, dbg2 = _run(torch.from_numpy(mask).cuda(), torch.from_numpy(field).cuda(), 256, 3, idxs, min_num=mn)
    _check(mask, field, idxs, lab2, num2, dbg2, min_num=mn)
    assert num2[2] == 1 and dbg2["win_counts"][2, 1] == w[1]


@pytest.mark.parametrize("b", [1, 64])
def test_batch_sizes(b):
    specs = [(1 + i % 4, 100 + i, 0.03 * (i % 2), i % 3 == 0, (10, 18)) for i in range(b)]
    _, mask, field = _scenes(specs, h=96, w=128)
    idxs = draw_center_idxs(b, 6, 64, b)
    lab, num, dbg = _run(torch.from_numpy(mask).cuda(), torch.from_numpy(field).cuda(), 64, 6, idxs, min_num=20)
    _check(mask, field, idxs, lab, num, dbg, min_num=20)


def test_invalid_arguments_rejected():
    L = _native.lib()
    n = ctypes.c_size_t()
    assert L.pvnet_center_workspace_bytes(2, 48, 64, 64, ctypes.byref(n)) == 0
    m = torch.zeros(2, 48, 64, dtype=torch.uint8, device="cuda")
    f = torch.zeros(2, 48, 64, 2, device="cuda")
    out = torch.empty(2, 48, 64, dtype=torch.int32, device="cuda")
    num = torch.empty(2, dtype=torch.int32, device="cuda")
    cen = torch.empty(2, 33, 2, device="cuda")
    idxs = torch.zeros(2, 33, 64, 2, dtype=torch.int32, device="cuda")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    st = (ctypes.c_int64 * 4)(*f.stride())
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    for I, b in [(0, 2), (33, 2), (4, 1025)]:
        rc = L.pvnet_ransac_voting_center(p(m), 1, p(f), st, p(idxs), None, b, 48, 64, 64, 0.99, 100, I, p(out),
                                          p(num), p(cen), None, None, None, None, p(ws), n.value, None)
        assert rc == -1, (I, b)
    with pytest.raises(ValueError):
        rv.ransac_voting_center(m, f, 64, rng="batched")


def test_device_rng_graph_replay():
    sc, mask, field = _scenes([(3, 2, 0.0, False, (40, 70)), (1, 11, 0.0, False, (40, 70))])
    m, f = torch.from_numpy(mask).cuda(), torch.from_numpy(field).cuda()
    torch.manual_seed(77)
    rv.reset_device_rng()
    state = rv._rng_state(m.device)
    # one eager call: the device draws are the numpy Philox restatement's
    seed, off = (int(v) for v in state.cpu().tolist())
    lab, num, dbg = _run(m, f, 256, 4)
    idxs = iv.device_center_idxs(seed, off, 2, 4, 256)
    _check(mask, field, idxs, lab, num, dbg)
    assert int(state[1].item()) == off + 1
    # capture, then replay with fresh draws each time
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        rv.ransac_voting_center(m, f, 256, THRESH, min_num=MIN_NUM, max_instances=4)      # workspace warm
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        glab, gnum = rv.ransac_voting_center(m, f, 256, THRESH, min_num=MIN_NUM, max_instances=4)
    seen = set()
    for _ in range(3):
        seed, off = (int(v) for v in state.cpu().tolist())
        g.replay()
        torch.cuda.synchronize()
        assert off not in seen
        seen.add(off)
        o = iv.ransac_voting_center(mask, field, iv.device_center_idxs(seed, off, 2, 4, 256), THRESH, MIN_NUM)
        assert list(gnum.cpu().numpy()) == [r["num"] for r in o] == [3, 1]
        lab = glab.cpu().numpy()
        for bi in range(2):
            gt, cen = sc[bi]["gt"], o[bi]["centers"][:o[bi]["num"]]
            mat = match_ids(lab[bi], gt, cen, sc[bi]["centers"])
            assert (mat[gt > 0] == gt[gt > 0]).mean() >= (1.0 if bi == 1 else 0.99)
        assert np.abs(o[1]["centers"][0] - sc[1]["centers"][0]).max() < 1e-2


# ---------------------------------------------------------------- ransac_voting_labels
def _label_case(b, h, w, L, specs, seed):
    sc = [instance_scene(n, s_, h=h, w=w, sigma=0.03, radius=r) for n, s_, r in specs]
    labels = np.stack([s["gt"] for s in sc]).astype(np.int64)
    vertex = np.stack([s["field"] for s in sc])
    rng = np.random.default_rng(seed)
    sel = rng.random((b, h, w), dtype=np.float32)
    return sc, labels, vertex, sel


def _pipeline_parity(labels, vertex, sel, L, hn, with_cov, min_num, max_num, seed, pairs=None, ldtype=torch.int64):
    b, h, w, vn, _ = vertex.shape
    lab_t = torch.from_numpy(labels).cuda().to(ldtype)
    v = torch.from_numpy(vertex).cuda()
    s = torch.from_numpy(sel).cuda()
    hnt = 64 * 4
    g = np.random.default_rng(seed)
    idxs = torch.from_numpy(g.integers(0, 2 ** 31 - 1, (b, L, hn, vn, 2), dtype=np.int32)).cuda()
    cov_idxs = torch.from_numpy(g.integers(0, 2 ** 31 - 1, (b, L, hnt, vn, 2), dtype=np.int32)).cuda()
    kw = dict(with_covariance=with_cov, cov_round_hyp_num=64, cov_min_hyp_num=hnt, min_num=min_num, max_num=max_num,
              selection=s, return_debug=True)
    res = rv.ransac_voting_labels(lab_t, v, L, hn, 0.99, idxs=idxs, cov_idxs=cov_idxs if with_cov else None, **kw)
    kp, cov, dbg = res if with_cov else (res[0], None, res[1])
    pairs = [(bi, j) for bi in range(b) for j in range(L)] if pairs is None else pairs
    for bi, j in pairs:
        m = (lab_t[bi:bi + 1] == j + 1).byte()
        r = rv.ransac_voting_pipeline(m, v[bi:bi + 1], hn, 0.99, idxs=idxs[bi, j][None],
                                      cov_idxs=cov_idxs[bi, j][None] if with_cov else None,
                                      rng="device", **{**kw, "selection": s[bi:bi + 1]})
        rk, rc, rd = r if with_cov else (r[0], None, r[1])
        assert torch.equal(kp[bi, j], rk[0]), (bi, j)
        assert torch.equal(dbg["tn"][bi, j], rd["tn"][0]), (bi, j)
        assert torch.equal(dbg["counts"][bi, j], rd["counts"][0]), (bi, j)
        assert torch.equal(dbg["hyp"][bi, j], rd["hyp"][0]), (bi, j)
        if with_cov:
            assert torch.equal(cov[bi, j], rc[0]), (bi, j)
            assert torch.equal(dbg["cov_counts"][bi, j], rd["cov_counts"][0]), (bi, j)
    return dbg


@pytest.mark.parametrize("with_cov", [False, True])
def test_labels_bit_identical_to_pipeline(with_cov):
    # 6 labels: 1-5 present in some images, 6 never; max_num under the larger instances subsamples them, min_num
    # above the smallest drops it
    specs = [(5, 3, (20, 45)), (2, 1, (20, 45)), (4, 4, (15, 30))]
    _, labels, vertex, sel = _label_case(3, 240, 320, 6, specs, 1)
    sizes = [(labels == j).sum() for j in range(1, 6)]
    dbg = _pipeline_parity(labels, vertex, sel, 6, 128, with_cov, min_num=1400, max_num=3000, seed=2)
    tn = dbg["tn"].cpu().numpy()
    assert (tn[:, 5] == 0).all()
    fg = np.array([[(labels[bi] == j + 1).sum() for j in range(6)] for bi in range(3)])
    assert ((fg > 0) & (fg < 1400)).any() and (tn[(fg > 0) & (fg < 1400)] == 0).all()
    assert ((fg > 3000) & (tn < fg) & (tn > 0)).any(), sizes


@pytest.mark.parametrize("ldtype", [torch.uint8, torch.int32])
def test_labels_element_sizes(ldtype):
    specs = [(3, 2, (20, 45))]
    _, labels, vertex, sel = _label_case(1, 240, 320, 4, specs, 3)
    _pipeline_parity(labels, vertex, sel, 4, 64, True, min_num=5, max_num=30000, seed=4, ldtype=ldtype)


def test_labels_1024_virtual_images():
    b, L, h, w = 32, 32, 32, 48
    g = np.random.default_rng(5)
    labels = g.integers(0, 40, (b, h, w)).astype(np.int64)          # values 33..39 are not labels
    ys, xs = np.mgrid[0:h, 0:w]
    kp = g.uniform(0, 48, (b, 1, 1, 3, 2))
    d = kp - np.stack([xs, ys], -1)[None, :, :, None, :]
    vertex = (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)
    sel = g.random((b, h, w), dtype=np.float32)
    pairs = [(bi, j) for bi in range(0, b, 5) for j in range(L)] + [(b - 1, L - 1)]
    _pipeline_parity(labels, vertex, sel, L, 32, False, min_num=5, max_num=30, seed=6, pairs=pairs)


def test_labels_invalid_sizes_rejected():
    L_ = _native.lib()
    n = ctypes.c_size_t()
    assert L_.pvnet_labels_workspace_bytes(4, 48, 64, 9, 8, 256, ctypes.byref(n)) == 0
    for b, L in [(1, 0), (1, 33), (33, 32), (1025, 1)]:
        assert L_.pvnet_labels_workspace_bytes(b, 48, 64, 9, L, 256, ctypes.byref(n)) == -1, (b, L)
    lab = torch.zeros(2, 48, 64, dtype=torch.int64, device="cuda")
    v = torch.zeros(2, 48, 64, 9, 2, device="cuda")
    for L in (0, 33):
        with pytest.raises(RuntimeError):
            rv.ransac_voting_labels(lab, v, L, 64)
    lab = torch.zeros(33, 8, 8, dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError):
        rv.ransac_voting_labels(lab, torch.zeros(33, 8, 8, 9, 2, device="cuda"), 32, 64)


def test_center_and_labels_in_one_graph():
    sc = [instance_scene(3, 2), instance_scene(1, 11)]
    m = torch.from_numpy(np.stack([s["mask"] for s in sc])).cuda()
    vertex = torch.from_numpy(np.stack([s["field"] for s in sc])).cuda()
    I = 4

    def step():
        labels, num = rv.ransac_voting_center(m, vertex[..., -1, :], 256, THRESH, min_num=MIN_NUM, max_instances=I)
        kp, cov = rv.ransac_voting_labels(labels, vertex, I, 256, cov_round_hyp_num=256, cov_min_hyp_num=4096)
        return labels, num, kp, cov

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        labels, num, kp, cov = step()
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        assert num.cpu().tolist() == [3, 1]
        kpn, lab = kp.cpu().numpy(), labels.cpu().numpy()
        for bi, sce in enumerate(sc):
            for i in range(len(sce["centers"])):
                c = kpn[bi, i, -1]
                gi = int(np.argmin(np.hypot(*(sce["centers"] - c[None]).T)))
                err = np.abs(kpn[bi, i] - sce["keypoints"][gi]).max()
                # the one-instance image is split exactly; in the three-instance one about 0.2 % of the pixels take
                # a neighbour's label (DESIGN.md section 29), and their votes moved a keypoint by 0.011 px when measured
                assert err < (1e-2 if len(sce["centers"]) == 1 else 3e-2), (bi, i, err)
                fg = sce["gt"] == gi + 1
                assert (lab[bi][fg] == i + 1).mean() >= 0.99
        assert np.isfinite(cov.cpu().numpy()[:, :1]).all()
