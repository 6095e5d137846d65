"""Shared test helpers (CPU side)."""
import hashlib
import os
import re

import numpy as np

from pvnet_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def demo_fixture():
    """mask int64 [480,640], exact vector field NCHW [18,480,640] f32, points_2d [9,2].
    The field is rebuilt from the fixture with the recipe of the reference's
    tools/demo.py:58-71 (`compute_vertex`): (kp - xy)/norm, norm<1e-3 -> +1e-3."""
    z = np.load(os.path.join(GOLDEN, "demo_cat.npz"))
    h, w = (int(v) for v in z["shape"])
    fg = z["fg_yx"].astype(np.int64)
    pts = z["points_2d"]
    mask = np.zeros((h, w), np.int64)
    mask[fg[:, 0], fg[:, 1]] = 1
    xy = fg[:, [1, 0]].astype(np.float64)
    v = pts[None, :, :2] - xy[:, None, :]
    n = np.linalg.norm(v, axis=2, keepdims=True)
    n[n < 1e-3] += 1e-3
    v = v / n
    field = np.zeros((h, w, pts.shape[0], 2), np.float32)
    field[fg[:, 0], fg[:, 1]] = v
    nchw = np.ascontiguousarray(field.reshape(h, w, -1).transpose(2, 0, 1))
    return mask, nchw, pts


def cfg1_inputs(kind):
    mask = syn.disc_mask(10000)
    field = syn.random_field(mask, 9, 1000) if kind == "random" else syn.planted_field(mask, 9, 1000)[0]
    idxs = syn.draw_idxs(10000, 128, 9, seed=1000)
    return mask, field, idxs


def seeded_state_dict(model, seed=0):
    """Deterministic weights for a Resnet18_8s-shaped module, a pure function of
    (parameter name, shape, seed) -- so the golden generator (which builds the REFERENCE
    classes) and the tests (which build ours) get identical tensors without sharing a file.
    Conv weights ~ N(0, sqrt(2/fan_out)); BN gamma ~ U(0.5,1.5), beta ~ N(0,0.1),
    running_mean ~ N(0,0.1), running_var ~ U(0.5,1.5) so folding is exercised."""
    import hashlib

    import torch
    out = {}
    for name, t in model.state_dict().items():
        h = int(hashlib.sha256(f"{seed}:{name}".encode()).hexdigest()[:8], 16)
        g = torch.Generator().manual_seed(h)
        if name.endswith("num_batches_tracked"):
            out[name] = torch.zeros_like(t)
        elif name.endswith("running_var"):
            out[name] = torch.rand(t.shape, generator=g) + 0.5
        elif name.endswith("running_mean"):
            out[name] = torch.randn(t.shape, generator=g) * 0.1
        elif t.dim() == 4:
            fan = t.shape[0] * t.shape[2] * t.shape[3]
            out[name] = torch.randn(t.shape, generator=g) * (2.0 / fan) ** 0.5
        elif name.endswith(".weight"):          # BN gamma
            out[name] = torch.rand(t.shape, generator=g) + 0.5
        else:                                    # BN beta / conv bias
            out[name] = torch.randn(t.shape, generator=g) * 0.1
    return out


# ---------------------------------------------------------------- inputs of tests/golden/ref_variants.npz
VARIANT_HWK = (64, 80, 5)


def variant_inputs(seed, n_fg=900, classes=1):
    """mask [1,H,W] int64 with `classes` disc-shaped regions (values 1..classes), vertex
    [1,H,W,K,2] f32: unit vectors towards K planted keypoints, rotated by N(0, 0.05 rad) noise.
    Shared by tests/golden/make_golden_variants.py (which feeds them to the reference's own
    Python functions) and the tests that replay the recorded samples."""
    H, W, K = VARIANT_HWK
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    mask = np.zeros((H, W), np.int64)
    for c in range(classes):
        cx, cy = W * (c + 1) / (classes + 1), H / 2
        d2 = (xx - cx) ** 2 + (yy - cy) ** 2
        order = np.argsort(d2.ravel(), kind="stable")[:n_fg // classes]
        mask.ravel()[order] = c + 1
    kps = np.stack([W / 2 + 30 * np.cos(2 * np.pi * np.arange(K) / K), H / 2 + 20 * np.sin(2 * np.pi * np.arange(K) / K)], 1)
    d = kps[None, None] - np.stack([xx, yy], -1)[:, :, None, :].astype(np.float64)      # [H,W,K,2]
    ang = np.arctan2(d[..., 1], d[..., 0]) + rng.normal(0, 0.05, d.shape[:-1])
    vertex = np.stack([np.cos(ang), np.sin(ang)], -1).astype(np.float32)
    vertex[mask == 0] = 0
    return mask[None], vertex[None], kps


BACKBONE_CASES = {"k9": (64, 96), "k17": (48, 64)}       # tag -> input height, width (batch 2)


def backbone_golden():
    """Outputs of the reference network classes (tests/golden/resnet18_8s_ref_<tag>.npz, made by
    tests/golden/make_golden_backbone.py) with their inputs, which are regenerated from the same seed:
    {tag_x, tag_seg, tag_ver} for tag in BACKBONE_CASES."""
    out = {}
    for tag, (h, w) in BACKBONE_CASES.items():
        z = np.load(os.path.join(GOLDEN, f"resnet18_8s_ref_{tag}.npz"))
        out[tag + "_x"] = np.random.default_rng(7).standard_normal((2, 3, h, w), dtype=np.float32)
        out[tag + "_seg"], out[tag + "_ver"] = z["seg"], z["ver"]
    return out


def reference_root():
    """The reference project's checkout named by PVNET_REFERENCE (the golden generators need it)."""
    root = os.environ.get("PVNET_REFERENCE")
    if not root or not os.path.isdir(os.path.join(root, "lib")):
        raise SystemExit("set PVNET_REFERENCE to a checkout of the reference project (zju3dv/pvnet); got %r" % root)
    return root


# ------------------------------------------------------------------ stored outputs of the reference's CUDA kernels
RECORD_REF = os.environ.get("PVNET_RECORD_REF_GOLDEN") == "1"     # set by tests/golden/make_golden_ref.py
_DIGEST_ABOVE = 4096                                               # bytes: larger exact arrays are stored as sha256


def _np(a):
    if hasattr(a, "detach"):
        return a.detach().cpu().numpy()
    return np.asarray(a)


def _pack(a):
    """What a golden file holds for one exact array: the array, or a digest of dtype, shape and bytes."""
    a = np.ascontiguousarray(_np(a))
    if a.nbytes <= _DIGEST_ABOVE:
        return a
    return np.array(hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest())


def same_as_stored(got, stored):
    """Bit-exact equality of `got` with a stored array or digest."""
    got = _pack(got)
    if got.dtype.kind == "U" or stored.dtype.kind == "U":
        return str(got) == str(stored)
    return got.dtype == stored.dtype and got.shape == stored.shape and got.tobytes() == stored.tobytes()


def reference_kernels():
    """oracle.ref_cuda: the reference's own kernels; only needed while recording."""
    from oracle import ref_cuda
    assert ref_cuda.available(), "recording needs oracle/_ref/libpvnet_refcuda.so (build() with PVNET_REFERENCE set)"
    return ref_cuda


class RefGolden:
    """Outputs of the reference's kernels under a key, in tests/golden/<name>: computed by `fn` while recording
    (PVNET_RECORD_REF_GOLDEN=1, needs oracle/_ref), read from the file otherwise.  Names in `exact` are packed
    (_pack: compare with same_as_stored), the rest are stored whole."""

    def __init__(self, name):
        self.path = os.path.join(GOLDEN, name)
        self.data = None

    def get(self, key, fn, exact=()):
        if self.data is None:
            self.data = {} if RECORD_REF else dict(np.load(self.path))
        key = re.sub(r"\W+", "_", key)
        if RECORD_REF:
            for name, v in fn().items():
                self.data[f"{key}/{name}"] = _pack(v) if name in exact else np.asarray(_np(v))
        pre = key + "/"
        return {k[len(pre):]: v for k, v in self.data.items() if k.startswith(pre)}

    def save(self):
        if RECORD_REF and self.data:
            np.savez_compressed(self.path, **self.data)
