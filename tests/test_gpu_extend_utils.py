"""GPU: farthest point sampling and binary mesh rasterisation on the device (pvnet_b200/extend_utils.py,
pvnet_b200/csrc/extend.cu), bit-identical to the reference's own compiled code (tests/golden/ref_extend.npz, made by
tests/golden/make_golden_ref_extend.py) and to the C oracle (oracle/extend_oracle.c):
  - FPS indices in both modes for pn from 1 to three times the on-chip capacity, sn up to pn + 3, lattice ties,
    duplicates, an all-duplicate cloud and NaN / inf / 1e30 coordinates; a batch of 13 equals 13 single calls;
    seeded clouds beyond the golden against the oracle;
  - masks for projected meshes of 10 k and 100 k triangles, full-frame, off-screen, partial, degenerate, shared-edge,
    sub-pixel and NaN triangles, bounds beyond 2^31 (oracle only) and odd sizes, with a canary margin around the
    mask that must stay untouched;
  - invalid arguments raise ValueError / RuntimeError."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import extend_oracle as eo
from pvnet_b200 import _native
from pvnet_b200 import extend_utils as eu
from tests import extend_cases as ec
from tests.helpers import GOLDEN, same_as_stored

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(GOLDEN, "ref_extend.npz")))


def _fps(pts, sn, start):
    got = eu.farthest_point_sampling(torch.from_numpy(pts).to(DEV), sn, start is None, start=start,
                                     return_indices=True)
    assert got.dtype == torch.int32 and tuple(got.shape) == (sn,)
    return got.cpu().numpy()


@pytest.mark.parametrize("name", ec.FPS_CASES)
def test_fps_bit_exact(golden, name):
    pts = ec.fps_cloud(name)
    pn = len(pts)
    for mode in ec.FPS_MODES:
        start = None if mode == "center" else ec.fps_start(pn)
        for sn in ec.fps_sample_counts(pn):
            got = _fps(pts, sn, start)
            assert same_as_stored(got, golden[f"fps/{name}/{mode}/{sn}"]), (name, mode, sn)
            assert np.array_equal(got, eo.farthest_point_sampling(pts, sn, start)), (name, mode, sn)


def test_fps_reference_call_shape(golden):
    pts = ec.fps_cloud("rand_1000").astype(np.float64)
    out = eu.farthest_point_sampling(pts, 8, True)
    idx = golden["fps/rand_1000/center/8"]
    assert isinstance(out, np.ndarray) and out.dtype == np.float32 and out.shape == (8, 3)
    assert np.array_equal(out, pts.astype(np.float32)[idx])
    assert eu.farthest_point_sampling(pts, 0, True).shape == (0, 3)


def test_fps_resident_capacity():
    L = _native.lib()
    n = ctypes.c_size_t()
    for pn, resident in ((ec.RESIDENT_CAPACITY, True), (ec.RESIDENT_CAPACITY + 1, False)):
        assert L.pvnet_farthest_point_sampling_workspace_bytes(2, pn, ctypes.byref(n)) == 0
        assert (n.value == 0) == resident, pn


def test_fps_batch_of_13_equals_single_calls():
    rng = np.random.default_rng(13)
    clouds = (rng.normal(size=(13, 2500, 3)) * rng.uniform(0.02, 0.2, (13, 1, 3))).astype(np.float32)
    starts = rng.integers(0, 2500, 13).astype(np.int32)
    dev = torch.from_numpy(clouds).to(DEV)
    for start in (None, starts):
        got = eu.farthest_point_sampling(dev, 64, start is None, start=start, return_indices=True).cpu().numpy()
        single = np.stack([_fps(clouds[i], 64, None if start is None else int(start[i])) for i in range(13)])
        assert np.array_equal(got, single)
        assert np.array_equal(got, eo.farthest_point_sampling(clouds, 64, start))
    pts = eu.farthest_point_sampling(dev, 8, True)
    assert tuple(pts.shape) == (13, 8, 3) and pts.is_cuda


@pytest.mark.parametrize("seed,pn,sn,b", [(1, 3000, 200, 2), (2, 20000, 64, 3), (3, 60000, 100, 2),
                                          (4, 200000, 40, 2), (5, 777, 900, 4)])
def test_fps_random_clouds_against_oracle(seed, pn, sn, b):
    rng = np.random.default_rng(seed)
    clouds = (rng.normal(size=(b, pn, 3)) * [0.1, 0.05, 0.07]).astype(np.float32)
    clouds[:, ::97] = np.round(clouds[:, ::97] * 64) / 64          # some coarse points: more equal distances
    starts = rng.integers(0, pn, b).astype(np.int32)
    dev = torch.from_numpy(clouds).to(DEV)
    for start in (None, starts):
        got = eu.farthest_point_sampling(dev, sn, start is None, start=start, return_indices=True).cpu().numpy()
        assert np.array_equal(got, eo.farthest_point_sampling(clouds, sn, start)), (seed, start is None)


def test_fps_drawn_start():
    pts = ec.fps_cloud("rand_1000")
    torch.manual_seed(3)
    got = eu.farthest_point_sampling(torch.from_numpy(pts).to(DEV), 16, return_indices=True).cpu().numpy()
    assert 0 <= got[0] < 1000
    assert np.array_equal(got, eo.farthest_point_sampling(pts, 16, int(got[0])))


def _raster_with_canary(t, h, w, margin=4096):
    """Runs the kernel on a mask inside a buffer whose margins hold 0xA5; returns the mask and checks the margins."""
    b = 1 if t.ndim == 3 else t.shape[0]
    tri = torch.from_numpy(np.ascontiguousarray(t, np.float32)).to(DEV)
    buf = torch.full((2 * margin + b * h * w,), 0xA5, dtype=torch.uint8, device=DEV)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _native.check(_native.lib().pvnet_mesh_binary_rasterization(
        tri.data_ptr() if tri.numel() else None, b, t.shape[-3], h, w, buf.data_ptr() + margin, stream),
        "pvnet_mesh_binary_rasterization")
    host = buf.cpu().numpy()
    assert (host[:margin] == 0xA5).all() and (host[margin + b * h * w:] == 0xA5).all(), "write outside the mask"
    return host[margin:margin + b * h * w].reshape((b, h, w) if t.ndim == 4 else (h, w))


@pytest.mark.parametrize("name", ec.RASTER_CASES + ec.RASTER_ORACLE_ONLY)
def test_raster_bit_exact(golden, name):
    t, h, w = ec.raster_case(name)
    want = eo.mesh_binary_rasterization(t, h, w)
    got = _raster_with_canary(t, h, w)
    assert np.array_equal(got, want), (name, int((got != want).sum()))
    if name in ec.RASTER_CASES:
        assert same_as_stored(got, golden[f"raster/{name}"]), name
        assert want.any() or name in ("offscreen",)
    # the reference call shape: numpy [tn,3,2] in, uint8 numpy [h,w] out
    out = eu.mesh_binary_rasterization(t, h, w)
    assert isinstance(out, np.ndarray) and out.dtype == np.uint8 and np.array_equal(out, want)


def test_raster_batch_of_16():
    rng = np.random.default_rng(16)
    base, h, w = ec.raster_case("sphere_10k")
    t = np.stack([base + rng.uniform(-200, 200, (1, 1, 2)).astype(np.float32) for _ in range(16)])
    want = eo.mesh_binary_rasterization(t, h, w)
    assert np.array_equal(_raster_with_canary(t, h, w), want)
    got = eu.mesh_binary_rasterization(torch.from_numpy(t).to(DEV), h, w)
    assert got.is_cuda and got.dtype == torch.uint8 and np.array_equal(got.cpu().numpy(), want)
    empty = _raster_with_canary(np.zeros((0, 3, 2), np.float32), 5, 7)
    assert not empty.any()


def test_invalid_arguments_raise():
    pts = torch.zeros(10, 3, device=DEV)
    with pytest.raises(ValueError):
        eu.farthest_point_sampling(pts, -1, True)
    with pytest.raises(ValueError):
        eu.farthest_point_sampling(torch.zeros(0, 3, device=DEV), 4, True)
    with pytest.raises(ValueError):
        eu.farthest_point_sampling(torch.zeros(10, 2, device=DEV), 4, True)
    with pytest.raises(ValueError):
        eu.farthest_point_sampling(pts, 4, start=[1, 2])
    with pytest.raises(RuntimeError, match="CUDA"):
        eu.farthest_point_sampling(torch.zeros(10, 3), 4, True)
    with pytest.raises(ValueError):
        eu.mesh_binary_rasterization(torch.zeros(4, 3, 2, device=DEV), 1, 10)
    with pytest.raises(ValueError):
        eu.mesh_binary_rasterization(torch.zeros(4, 2, 2, device=DEV), 10, 10)
    L = _native.lib()
    n = ctypes.c_size_t()
    idx = torch.zeros(8, dtype=torch.int32, device=DEV)
    m = torch.zeros(64, dtype=torch.uint8, device=DEV)
    tri = torch.zeros(1, 3, 2, device=DEV)
    bad = [L.pvnet_farthest_point_sampling(pts.data_ptr(), None, 1, 0, 4, idx.data_ptr(), None, 0, None),
           L.pvnet_farthest_point_sampling(pts.data_ptr(), None, 1, 10, -1, idx.data_ptr(), None, 0, None),
           L.pvnet_farthest_point_sampling(None, None, 1, 10, 4, idx.data_ptr(), None, 0, None),
           L.pvnet_farthest_point_sampling(pts.data_ptr(), None, 1, ec.RESIDENT_CAPACITY + 1, 4, idx.data_ptr(),
                                           None, 0, None),
           L.pvnet_farthest_point_sampling_workspace_bytes(1, 0, ctypes.byref(n)),
           L.pvnet_mesh_binary_rasterization(tri.data_ptr(), 1, 1, 1, 8, m.data_ptr(), None),
           L.pvnet_mesh_binary_rasterization(tri.data_ptr(), 1, 1, 8, 1, m.data_ptr(), None),
           L.pvnet_mesh_binary_rasterization(tri.data_ptr(), 1, -1, 8, 8, m.data_ptr(), None),
           L.pvnet_mesh_binary_rasterization(tri.data_ptr(), 1, 1, 8, 8, None, None)]
    assert bad == [-1] * len(bad)
    with pytest.raises(RuntimeError, match="below 2x2"):
        _native.check(L.pvnet_mesh_binary_rasterization(tri.data_ptr(), 1, 1, 1, 8, m.data_ptr(), None), "raster")
    torch.cuda.synchronize()
    assert eu.farthest_point_sampling(pts, 4, True, return_indices=True).cpu().tolist() == [0, 0, 0, 0]
