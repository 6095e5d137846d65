"""Inputs of the farthest-point-sampling and rasterisation cases, regenerated from their names.

Shared by tests/golden/make_golden_ref_extend.py (which records the reference's own code on them into
tests/golden/ref_extend.npz), tests/test_extend_oracle.py and tests/test_gpu_extend_utils.py."""
import io
import zipfile
import zlib

import numpy as np

from tests.helpers import _pack

RESIDENT_CAPACITY = 8 * 14336          # points of one cloud that stay on chip (csrc/extend.cu: 8 CTAs x FPS_SLICE)


def _rng(name):
    return np.random.default_rng(zlib.crc32(name.encode()))


# ------------------------------------------------------------------ farthest point sampling
FPS_SIZES = [1, 2, 7, 1000, RESIDENT_CAPACITY - 1, RESIDENT_CAPACITY, RESIDENT_CAPACITY + 1, 3 * RESIDENT_CAPACITY]
FPS_CASES = [f"rand_{n}" for n in FPS_SIZES] + ["lattice", "lattice_shuffled", "dups", "all_dup", "nan_inf"]
FPS_MODES = ["center", "start"]


def fps_cloud(name):
    """float32 [pn,3]."""
    rng = _rng(name)
    if name.startswith("rand_"):
        pn = int(name[5:])
        return (rng.normal(size=(pn, 3)) * [0.05, 0.08, 0.03]).astype(np.float32)
    if name.startswith("lattice"):
        g = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
        return g[rng.permutation(len(g))] if name.endswith("shuffled") else g
    if name == "dups":
        p = rng.normal(size=(600, 3)).astype(np.float32)
        return np.concatenate([p, p])[rng.permutation(1200)]
    if name == "all_dup":
        return np.tile(np.array([[0.25, -1.5, 3.0]], np.float32), (40, 1))
    if name == "nan_inf":
        p = rng.normal(size=(1000, 3)).astype(np.float32)
        k = rng.permutation(1000)
        p[k[:15], rng.integers(0, 3, 15)] = np.nan
        p[k[15:30], rng.integers(0, 3, 15)] = np.inf
        p[k[30:40], rng.integers(0, 3, 10)] = -np.inf
        p[k[40:50], rng.integers(0, 3, 10)] = 1e30
        p[k[50:55]] = -1e30
        return p
    raise KeyError(name)


def fps_sample_counts(pn):
    return [1, 8, 64] if pn > 2000 else sorted({1, 8, 64, pn, pn + 3})


def fps_start(pn):
    """The first index of the "start" mode: what the reference's rand() returns (taken modulo pn)."""
    return 3 * pn + (37 * pn) // 101


# ------------------------------------------------------------------ rasterisation
def _project(v, R, t, K):
    c = v @ R.T + t
    uv = c @ K.T
    return uv[:, :2] / uv[:, 2:3]


def _rot(rng):
    a = rng.normal(size=3)
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


_CAM = np.array([[572.4, 0.0, 325.3], [0.0, 573.6, 242.0], [0.0, 0.0, 1.0]])


def _sphere(n_lat, n_lon):
    th = np.linspace(0, np.pi, n_lat + 1)
    ph = np.linspace(0, 2 * np.pi, n_lon + 1)
    v = np.stack([np.sin(th)[:, None] * np.cos(ph)[None], np.sin(th)[:, None] * np.sin(ph)[None],
                  np.cos(th)[:, None] * np.ones_like(ph)[None]], -1).reshape(-1, 3)
    i = np.arange(n_lat)[:, None] * (n_lon + 1) + np.arange(n_lon)[None]
    i = i.ravel()
    f = np.concatenate([np.stack([i, i + n_lon + 1, i + 1], 1), np.stack([i + 1, i + n_lon + 1, i + n_lon + 2], 1)])
    return v, f


def _box(n):
    s = np.linspace(-1, 1, n + 1)
    u, w = np.meshgrid(s, s, indexing="ij")
    verts, faces = [], []
    for axis in range(3):
        for sign in (-1.0, 1.0):
            p = np.zeros((n + 1, n + 1, 3))
            p[..., axis] = sign
            p[..., (axis + 1) % 3] = u
            p[..., (axis + 2) % 3] = w
            base = sum(len(x) for x in verts)
            verts.append(p.reshape(-1, 3))
            i = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None]).ravel() + base
            faces += [np.stack([i, i + n + 1, i + 1], 1), np.stack([i + 1, i + n + 1, i + n + 2], 1)]
    return np.concatenate(verts) * [0.6, 0.9, 0.4], np.concatenate(faces)


def _mesh_tris(kind, rng, size):
    v, f = _sphere(*size) if kind == "sphere" else _box(size)
    v = v * 0.08
    t = np.array([rng.uniform(-0.05, 0.05), rng.uniform(-0.05, 0.05), rng.uniform(0.45, 0.7)])
    return _project(v, _rot(rng), t, _CAM)[f].astype(np.float32)


RASTER_CASES = ["sphere_10k", "box_10k", "sphere_100k", "box_100k", "full_frame", "full_frame_odd", "offscreen",
                "partial", "degenerate", "edges", "subpixel", "nan"]
RASTER_ORACLE_ONLY = ["huge"]    # bounds of 2^31 and beyond: the reference's int() is undefined there


def raster_case(name):
    """(triangles float32 [tn,3,2], h, w)."""
    rng = _rng(name)
    if name == "sphere_10k":
        return _mesh_tris("sphere", rng, (50, 100)), 480, 640
    if name == "sphere_100k":
        return _mesh_tris("sphere", rng, (224, 224)), 480, 640
    if name == "box_10k":
        return _mesh_tris("box", rng, 29), 480, 640
    if name == "box_100k":
        return _mesh_tris("box", rng, 92), 480, 640
    if name.startswith("full_frame"):
        h, w = (480, 640) if name == "full_frame" else (37, 53)
        t = np.array([[[-50, -40], [w + 60, -30], [-45, h + 70]], [[w + 60, -30], [w + 80, h + 90], [-45, h + 70]],
                      [[0, 0], [w - 1, 0], [0, h - 1]]], np.float32)
        return t, h, w
    if name == "offscreen":
        h, w = 61, 83
        left = rng.uniform([-500, -50], [-1.01, h + 50], (60, 3, 2))             # all x < -1
        right = rng.uniform([w + 0.01, -50], [900, h + 50], (60, 3, 2))          # all x > w
        above = rng.uniform([-50, -400], [w + 50, -1.01], (60, 3, 2))            # all y < -1
        near = rng.uniform([-1.99, -50], [-1.0, h + 50], (20, 3, 2))             # max x in [-2, -1]: column 0 tested
        return np.concatenate([left, right, above, near]).astype(np.float32), h, w
    if name == "partial":
        h, w = 120, 160
        return rng.uniform([-100, -80], [w + 100, h + 80], (300, 3, 2)).astype(np.float32), h, w
    if name == "degenerate":
        h, w = 63, 65
        p = rng.uniform(0, 60, (100, 1, 2)).astype(np.float32)
        zero = np.repeat(np.round(p[:50] * 2) / 2, 3, axis=1)                     # three equal vertices
        a, b = p[50:], rng.uniform(0, 60, (50, 1, 2)).astype(np.float32)
        s = rng.uniform(0, 1, (50, 1, 1)).astype(np.float32)
        line = np.concatenate([a, b, a + s * (b - a)], 1)                         # collinear, general direction
        ax = np.array([[[3, 7], [20, 7], [40, 7]], [[5, 2], [5, 30], [5, 50]], [[1, 1], [9, 9], [30, 30]],
                       [[2.5, 2.5], [10.5, 10.5], [20.5, 20.5]]], np.float32)    # axis-aligned and diagonal
        return np.concatenate([zero, line.astype(np.float32), ax]), h, w
    if name == "edges":
        h, w = 101, 131
        tris = []
        for y in range(-10, h + 10, 10):                                          # squares on integer vertices, two
            for x in range(-10, w + 10, 10):                                      # triangles sharing the diagonal
                tris += [[[x, y], [x + 10, y], [x, y + 10]], [[x + 10, y], [x + 10, y + 10], [x, y + 10]]]
        t = np.array(tris, np.float32)
        t = t[rng.random(len(t)) < 0.6]
        neg = rng.uniform(-1, 0, (40, 3, 2)).astype(np.float32)                   # vertices in (-1, 0)
        neg[:20, :, 1] += rng.integers(0, h, (20, 1)).astype(np.float32)
        neg[20:, :, 0] += rng.integers(0, w, (20, 1)).astype(np.float32)
        neg[::5, 2] += 0.999
        return np.concatenate([t, neg]), h, w
    if name == "subpixel":
        h, w = 45, 77
        c = rng.uniform([-1, -1], [w, h], (5000, 1, 2))
        return (c + rng.uniform(-1, 1, (5000, 3, 2))).astype(np.float32), h, w
    if name == "nan":
        h, w = 50, 70
        t = rng.uniform([-5, -5], [w + 5, h + 5], (120, 3, 2)).astype(np.float32)
        t[::3, rng.integers(0, 3), rng.integers(0, 2)] = np.nan
        t[1::7] = np.nan
        return t, h, w
    if name == "huge":
        h, w = 40, 50
        t = rng.uniform(0, 45, (60, 3, 2)).astype(np.float32)
        t[0:10, :, 0] = 3e9                                                       # min x >= 2^31
        t[10:20, :, 1] = np.inf
        t[20:30, :, 0] = -3e9                                                     # max x + 1 < -2^31
        t[30:40, 0, 0], t[30:40, 1, 0] = -3e9, 3e9                                # a box that spans the mask
        t[40:45, :, 1] = 2147483648.0
        return t, h, w
    raise KeyError(name)


# ------------------------------------------------------------------ the golden file
def golden_entries(fps, raster):
    """{key: array} of the golden file from fps(pts, sn, start) and raster(triangles, h, w); start is None for the
    init_center mode."""
    out = {}
    for name in FPS_CASES:
        pts = fps_cloud(name)
        pn = len(pts)
        for mode in FPS_MODES:
            for sn in fps_sample_counts(pn):
                out[f"fps/{name}/{mode}/{sn}"] = _pack(fps(pts, sn, None if mode == "center" else fps_start(pn)))
    for name in RASTER_CASES:
        t, h, w = raster_case(name)
        out[f"raster/{name}"] = _pack(raster(t, h, w))
    return out


def write_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps, so that the file is a function of its contents."""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
