"""Pose evaluation on the device: the reference's lib/utils/evaluation_utils.py (`pnp`, `find_nearest_point_distance`,
`Evaluator`) and the nearest-point search of lib/utils/extend_utils/extend_utils.py:39-60, over the C ABI
(`pvnet_find_nearest_point_idx`, `pvnet_pose_metrics`, `pvnet_uncertainty_pnp` in include/pvnet_b200.h).

    find_nearest_point_idx(ref_pts, que_pts)          numpy [pn,dim] -> numpy int32 [pn2];  CUDA [b,pn,dim] -> [b,pn2]
    find_nearest_point_distance(pts1, pts2)           numpy -> numpy float64;  CUDA tensors stay on the device
    pose_metrics(pose_pred, pose_gt, model, K, symmetric=False, sym_proj=False)
                                                      -> float64 [b,4] = (add, proj, trans_cm, angle_deg) on the device
    pnp(points_3d, points_2d, camera_matrix, method=0)
    uncertainty_pnp_v2(points_2d, covars, points_3d, camera_matrix, type='single')
    Evaluator                                          the reference's recorder class, plus evaluate_batch() and
                                                       evaluate_keypoints_batch() (per-image cameras)

Numpy inputs keep the reference's return types (one host synchronisation per call, as the reference's host loop
has); batched CUDA tensors return CUDA tensors without synchronising.  No CPU path: without the library or a CUDA
device these functions raise.  Importing this module needs neither cv2, scipy nor plyfile.
"""
from __future__ import annotations

import ctypes
import importlib
import time

import numpy as np
import torch

from . import _native
from .extend_utils import covariance_to_weights, uncertainty_pnp, uncertainty_pnp_batched

SOLVEPNP_ITERATIVE = 0                  # cv2.SOLVEPNP_ITERATIVE
SYMMETRIC_CLASSES = ("eggbox", "glue")  # evaluation_utils.py:159,193,210


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _device(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("pvnet_b200: pose evaluation needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


def _on(x, dev, dtype):
    if isinstance(x, torch.Tensor):
        return x.to(device=dev, dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(x, dtype=torch.empty((), dtype=dtype).numpy().dtype), device=dev)


# ------------------------------------------------------------------------------------------ nearest-point search
def find_nearest_point_idx(ref_pts, que_pts):
    """For every point of que_pts the index of the nearest point of ref_pts (extend_utils.py:39-60), bit-identical to
    the reference kernel.  numpy [pn1,dim], [pn2,dim] -> numpy int32 [pn2]; CUDA tensors [pn,dim] or [b,pn,dim] ->
    int32 CUDA tensor [pn2] or [b,pn2], no synchronisation."""
    host = not isinstance(ref_pts, torch.Tensor)
    if host:
        assert ref_pts.shape[1] == que_pts.shape[1] and 1 < que_pts.shape[1] <= 3       # extend_utils.py:47
    dev = _device(ref_pts, que_pts)
    ref, que = _on(ref_pts, dev, torch.float32), _on(que_pts, dev, torch.float32)
    single = ref.dim() == 2
    if single:
        ref, que = ref[None], que[None]
    if ref.dim() != 3 or que.dim() != 3 or ref.shape[0] != que.shape[0] or ref.shape[2] != que.shape[2]:
        raise ValueError(f"ref_pts {tuple(ref.shape)} and que_pts {tuple(que.shape)} must be [b,pn,dim] alike")
    b, pn1, dim = ref.shape
    pn2 = que.shape[1]
    idxs = torch.empty([b, pn2], dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _native.check(_native.lib().pvnet_find_nearest_point_idx(ref.data_ptr(), que.data_ptr(), idxs.data_ptr(), b,
                                                                 pn1, pn2, dim, _stream(dev)),
                      "pvnet_find_nearest_point_idx")
    if single:
        idxs = idxs[0]
    return idxs.cpu().numpy() if host else idxs


def find_nearest_point_distance(pts1, pts2):
    """|pts1[nearest] - pts2| for every point of pts2 (evaluation_utils.py:54-62)."""
    idxs = find_nearest_point_idx(pts1, pts2)
    if isinstance(idxs, np.ndarray):
        return np.linalg.norm(pts1[idxs] - pts2, 2, 1)
    p1 = torch.as_tensor(pts1, device=idxs.device)
    p2 = torch.as_tensor(pts2, device=idxs.device)
    if p1.dim() == 2:
        return torch.linalg.norm(p1[idxs.long()] - p2, dim=-1)
    near = torch.gather(p1, 1, idxs.long()[..., None].expand(-1, -1, p1.shape[-1]))
    return torch.linalg.norm(near - p2, dim=-1)


# ------------------------------------------------------------------------------------------------ pose metrics
def pose_metrics(pose_pred, pose_gt, model, K, symmetric=False, sym_proj=False):
    """(add, proj, trans_cm, angle_deg) per image, float64 [b,4] on the device (evaluation_utils.py:75-141).

    pose_pred, pose_gt [b,3,4] (or [3,4]); model [n,3] mesh vertices; K a host [3,3] (numpy, list, CPU tensor) for
    every image, or a CUDA tensor [3,3] / [b,3,3] (per-image intrinsics).  symmetric: ADD-S instead of ADD;
    sym_proj: the nearest-point 2-D projection error of projection_2d_sym.  Thresholds are left to the caller:
    add < diameter*0.1, proj < 5, trans_cm < 5 and angle_deg < 5."""
    dev = _device(pose_pred, pose_gt, model, K)
    pp = _on(pose_pred, dev, torch.float64).reshape(-1, 3, 4).contiguous()
    pg = _on(pose_gt, dev, torch.float64).reshape(-1, 3, 4).contiguous()
    if pp.shape != pg.shape:
        raise ValueError(f"pose_pred {tuple(pp.shape)} and pose_gt {tuple(pg.shape)} differ")
    b = pp.shape[0]
    m = _on(model, dev, torch.float32)
    if m.dim() != 2 or m.shape[1] != 3:
        raise ValueError(f"model must be [n,3], got {tuple(m.shape)}")
    n = m.shape[0]
    k_host, k_dev = None, None
    if isinstance(K, torch.Tensor) and K.is_cuda:
        k_dev = K.to(dev, torch.float64).reshape(-1, 3, 3).expand(b, 3, 3).contiguous()
    else:
        k = np.asarray(K.detach().cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64).reshape(9)
        k_host = (ctypes.c_double * 9)(*k.tolist())
    L = _native.lib()
    nbytes = ctypes.c_size_t()
    _native.check(L.pvnet_pose_metrics_workspace_bytes(b, n, ctypes.byref(nbytes)), "pvnet_pose_metrics_workspace_bytes")
    ws = torch.empty([nbytes.value], dtype=torch.uint8, device=dev)
    out = torch.empty([b, 4], dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _native.check(L.pvnet_pose_metrics(pp.data_ptr(), pg.data_ptr(), m.data_ptr(), n, k_host,
                                           None if k_dev is None else k_dev.data_ptr(), b, int(bool(symmetric)),
                                           int(bool(sym_proj)), out.data_ptr(), ws.data_ptr(), nbytes.value,
                                           _stream(dev)),
                      "pvnet_pose_metrics")
    return out


# --------------------------------------------------------------------------------------------------------- PnP
def pnp(points_3d, points_2d, camera_matrix, method=SOLVEPNP_ITERATIVE):
    """evaluation_utils.py:19-52 with cv2.SOLVEPNP_ITERATIVE, on the device solver of `uncertainty_pnp` with unit
    weights (1, 0, 1): it then minimises the plain reprojection error, the objective of SOLVEPNP_ITERATIVE.  The
    start differs from OpenCV's (a DLT): with equal weights the solver's stable "four largest wxx + wxy" rule takes
    the LAST four points for its P3P start.  4 <= pn <= 32; with exactly 4 points the P3P pose is returned.
    numpy in -> numpy [3,4] float64; CUDA points_2d [b,pn,2] -> float64 CUDA [b,3,4] without synchronising."""
    if method != SOLVEPNP_ITERATIVE:
        raise ValueError(f"pnp: only method=0 (cv2.SOLVEPNP_ITERATIVE) is provided, got {method!r}")
    if isinstance(points_2d, torch.Tensor) and points_2d.is_cuda and points_2d.dim() == 3:
        b, pn, _ = points_2d.shape
        w = torch.zeros([b, pn, 3], dtype=torch.float32, device=points_2d.device)
        w[..., 0] = 1.0
        w[..., 2] = 1.0
        return uncertainty_pnp_batched(points_2d, points_3d, camera_matrix, weights_2d=w)
    p3, p2 = np.asarray(points_3d), np.asarray(points_2d)
    assert p3.shape[0] == p2.shape[0], 'points 3D and points 2D must have same number of vertices'
    w = np.tile(np.array([1.0, 0.0, 1.0], np.float32), (p2.shape[0], 1))
    return uncertainty_pnp(p2, w, p3, camera_matrix)


def uncertainty_pnp_v2_weights(covars: torch.Tensor) -> torch.Tensor:
    """extend_utils.py:131-139 on the device: 1 / (largest eigenvalue of the 2x2 cov), 0 where cov[0,0] < 1e-5,
    returned as the solver's weight triple (w, 0, w) float32 [...,3]."""
    c = covars.to(torch.float64)
    a, b_, c_, d = c[..., 0, 0], c[..., 0, 1], c[..., 1, 0], c[..., 1, 1]
    half = (a - d) * 0.5
    lam = (a + d) * 0.5 + torch.sqrt(half * half + b_ * c_)
    w = torch.where(a < 1e-5, torch.zeros_like(a), 1.0 / lam)
    return torch.stack([w, torch.zeros_like(w), w], -1).float()


def uncertainty_pnp_v2(points_2d, covars, points_3d, camera_matrix, type='single'):
    """extend_utils.py:116-177: the uncertainty PnP with the scalar weight 1/lambda_max(cov) per point, on the same
    device solver (weights (w, 0, w), so its selection key wxx + wxy = w is the reference's argsort(weights)[-4:]).
    numpy [pn,2], [pn,2,2], [pn,3], [3,3] -> numpy [3,4] float64; CUDA [b,pn,2], [b,pn,2,2] -> CUDA [b,3,4]."""
    if isinstance(points_2d, torch.Tensor) and points_2d.is_cuda and points_2d.dim() == 3:
        w = uncertainty_pnp_v2_weights(covars.to(points_2d.device))
        return uncertainty_pnp_batched(points_2d, points_3d, camera_matrix, weights_2d=w)
    pn = np.asarray(points_2d).shape[0]
    assert np.asarray(points_3d).shape[0] == pn and pn >= 4 and np.asarray(covars).shape[0] == pn   # :125
    dev = _device()
    w = uncertainty_pnp_v2_weights(torch.as_tensor(np.asarray(covars, np.float64), device=dev))
    p2 = torch.as_tensor(np.asarray(points_2d, np.float32), device=dev)[None]
    return uncertainty_pnp_batched(p2, np.asarray(points_3d, np.float32), camera_matrix,
                                   weights_2d=w[None])[0].cpu().numpy()


# --------------------------------------------------------------------------------------------------- Evaluator
class _RefName:
    """A class of the reference tree this module is installed into, imported on first use (so that importing
    this module does not need the dataset code, cv2 or plyfile)."""

    def __init__(self, module, name):
        self.module, self.name = module, name

    def get(self):
        return getattr(importlib.import_module(self.module), self.name)


_LineModModelDB = _RefName("lib.utils.data_utils", "LineModModelDB")
_Projector = _RefName("lib.utils.data_utils", "Projector")
_VotingType = _RefName("lib.datasets.linemod_dataset", "VotingType")


class _VotingTypeBB8:
    """The default `vote_type=VotingType.BB8`, resolved when a call uses it."""

    def __repr__(self):
        return "VotingType.BB8"


_BB8 = _VotingTypeBB8()


class Evaluator(object):
    """lib/utils/evaluation_utils.py:64-226 with the metrics computed by `pose_metrics` on the device.

    The per-image methods keep the reference's arguments and fill the same recorder lists.  `evaluate_batch` takes
    a batch of device poses and accumulates the pass counts and distance sums on the device; only
    `average_precision` reads them back (one synchronisation).  The dataset objects (LineModModelDB, Projector,
    VotingType) come from the reference tree on first use; `model_db=` / `projector=` supply them instead.
    average_precision does not write the reference's `tmp.npy` scratch file."""

    def __init__(self, *, model_db=None, projector=None):
        self.linemod_db = model_db if model_db is not None else _LineModModelDB.get()()
        self.projector = projector if projector is not None else _Projector.get()()
        self.projection_2d_recorder = []
        self.add_recorder = []
        self.cm_degree_5_recorder = []
        self.proj_mean_diffs = []
        self.add_dists = []
        self.uncertainty_pnp_cost = []
        # evaluate_batch totals (float64, device): images, proj passes, add passes, 5cm5deg passes, proj sum, add sum
        self.batch_totals = None
        self._points_dev = {}           # evaluate_keypoints_batch: (class, vote type, device) -> (keypoints, model)

    # ---- one image (numpy in, as the reference)
    @staticmethod
    def _metrics(pose_pred, pose_targets, model, K, symmetric=False, sym_proj=False):
        return pose_metrics(pose_pred, pose_targets, model, K, symmetric, sym_proj)[0].cpu().numpy()

    def _record_proj(self, proj_mean_diff, threshold=5):
        self.proj_mean_diffs.append(proj_mean_diff)
        self.projection_2d_recorder.append(proj_mean_diff < threshold)

    def _record_add(self, mean_dist, diameter, percentage=0.1):
        diameter = diameter * percentage
        self.add_recorder.append(mean_dist < diameter)
        self.add_dists.append(mean_dist)

    def _record_cm_degree_5(self, translation_distance, angular_distance):
        self.cm_degree_5_recorder.append(translation_distance < 5 and angular_distance < 5)

    def projection_2d(self, pose_pred, pose_targets, model, K, threshold=5):
        self._record_proj(self._metrics(pose_pred, pose_targets, model, K)[1], threshold)

    def projection_2d_sym(self, pose_pred, pose_targets, model, K, threshold=5):
        self._record_proj(self._metrics(pose_pred, pose_targets, model, K, sym_proj=True)[1], threshold)

    def add_metric(self, pose_pred, pose_targets, model, diameter, percentage=0.1):
        self._record_add(self._metrics(pose_pred, pose_targets, model, np.eye(3))[0], diameter, percentage)

    def add_metric_sym(self, pose_pred, pose_targets, model, diameter, percentage=0.1):
        self._record_add(self._metrics(pose_pred, pose_targets, model, np.eye(3), symmetric=True)[0], diameter,
                         percentage)

    def cm_degree_5_metric(self, pose_pred, pose_targets):
        m = self._metrics(pose_pred, pose_targets, np.zeros([1, 3], np.float32), np.eye(3))
        self._record_cm_degree_5(m[2], m[3])

    def _K(self, intri_type, intri_matrix=None):
        if intri_type == 'use_intrinsic' and intri_matrix is not None:
            return intri_matrix
        return self.projector.intrinsic_matrix[intri_type]

    def _all_metrics(self, pose_pred, pose_targets, class_type, K, sym_proj=False):
        model = self.linemod_db.get_ply_model(class_type)
        diameter = self.linemod_db.get_diameter(class_type)
        m = self._metrics(pose_pred, pose_targets, model, K, class_type in SYMMETRIC_CLASSES, sym_proj)
        self._record_add(m[0], diameter)
        self._record_proj(m[1])
        self._record_cm_degree_5(m[2], m[3])

    def evaluate(self, points_2d, pose_targets, class_type, intri_type='blender', vote_type=_BB8, intri_matrix=None):
        vt = _VotingType.get()
        points_3d = vt.get_pts_3d(vt.BB8 if vote_type is _BB8 else vote_type, class_type)
        K = self._K(intri_type, intri_matrix)
        pose_pred = pnp(points_3d, points_2d, K)
        self._all_metrics(pose_pred, pose_targets, class_type, K)
        return pose_pred

    def evaluate_uncertainty(self, mean_pts2d, covar, pose_targets, class_type,
                             intri_type='blender', vote_type=_BB8, intri_matrix=None):
        vt = _VotingType.get()
        points_3d = vt.get_pts_3d(vt.BB8 if vote_type is _BB8 else vote_type, class_type)
        begin = time.time()
        dev = _device()
        weights = covariance_to_weights(torch.as_tensor(np.asarray(covar, np.float32), device=dev)).cpu().numpy()
        K = self._K(intri_type, intri_matrix)
        pose_pred = uncertainty_pnp(mean_pts2d, weights, points_3d, K)
        self.uncertainty_pnp_cost.append(time.time() - begin)
        self._all_metrics(pose_pred, pose_targets, class_type, K)
        return pose_pred

    def evaluate_uncertainty_v2(self, mean_pts2d, covar, pose_targets, class_type,
                                intri_type='blender', vote_type=_BB8):
        vt = _VotingType.get()
        points_3d = vt.get_pts_3d(vt.BB8 if vote_type is _BB8 else vote_type, class_type)
        K = self.projector.intrinsic_matrix[intri_type]
        pose_pred = uncertainty_pnp_v2(mean_pts2d, covar, points_3d, K)
        # the symmetric classes use the nearest-point 2-D error here, unlike evaluate / evaluate_uncertainty
        self._all_metrics(pose_pred, pose_targets, class_type, K, sym_proj=class_type in SYMMETRIC_CLASSES)

    # ---- a batch on the device
    def _device_points(self, class_type, vote_type, dev):
        """The object's keypoints and mesh vertices as float32 device tensors, copied once per (class, vote type,
        device): a copy from pageable host memory would synchronise every batch."""
        key = (class_type, vote_type, dev)
        if key not in self._points_dev:
            vt = _VotingType.get()
            pts = vt.get_pts_3d(vt.BB8 if vote_type is _BB8 else vote_type, class_type)
            model = self.linemod_db.get_ply_model(class_type)
            self._points_dev[key] = (_on(pts, dev, torch.float32), _on(model, dev, torch.float32))
        return self._points_dev[key]

    def evaluate_keypoints_batch(self, points_2d, pose_targets, class_type, K, covar=None, vote_type=_BB8):
        """`evaluate` (covar None) or `evaluate_uncertainty` (covar [b,pn,2,2]) for a batch of images of one object
        on the device, with one camera per image: the truncated-LINEMOD branch of val() (tools/train_linemod.py:
        199-205) in one call per batch instead of one per image.  points_2d [b,pn,2] and pose_targets [b,3,4] CUDA
        tensors; K a CUDA [b,3,3] (or anything `uncertainty_pnp_batched` takes).  Poses, then `evaluate_batch` with
        the class's model, diameter and symmetry: the per-image methods' pose and metric values, bit for bit (the
        covariances become float32 weights first, as in evaluate_uncertainty).  Does not synchronise once the
        class's points are on the device.  Returns (pose_pred float64 [b,3,4], metrics float64 [b,4])."""
        dev = points_2d.device
        points_3d, model = self._device_points(class_type, vote_type, dev)
        if covar is None:
            pose_pred = pnp(points_3d, points_2d, K)
        else:
            weights = covariance_to_weights(covar.to(dev))
            pose_pred = uncertainty_pnp_batched(points_2d, points_3d, K, weights_2d=weights)
        m = self.evaluate_batch(pose_pred, pose_targets, model, self.linemod_db.get_diameter(class_type), K,
                                symmetric=class_type in SYMMETRIC_CLASSES)
        return pose_pred, m

    def evaluate_batch(self, pose_pred, pose_targets, model, diameter, K, symmetric=False, sym_proj=False):
        """Metrics of a batch of device poses [b,3,4] of one object; the pass counts and distance sums are added to
        `batch_totals` on the device (no synchronisation, CUDA-graph capturable).  Returns the [b,4] metrics."""
        m = pose_metrics(pose_pred, pose_targets, model, K, symmetric, sym_proj)
        add_ok = m[:, 0] < diameter * 0.1
        proj_ok = m[:, 1] < 5
        cm_ok = (m[:, 2] < 5) & (m[:, 3] < 5)
        upd = torch.stack([proj_ok.sum(dtype=torch.float64), add_ok.sum(dtype=torch.float64),
                           cm_ok.sum(dtype=torch.float64), m[:, 1].sum(), m[:, 0].sum()])
        if self.batch_totals is None:
            self.batch_totals = torch.zeros([6], dtype=torch.float64, device=m.device)
        self.batch_totals[0].add_(m.shape[0])
        self.batch_totals[1:].add_(upd)
        return m

    def average_precision(self, verbose=True):
        """Means of the three recorders (evaluation_utils.py:219-226), over the per-image calls and evaluate_batch."""
        n = len(self.projection_2d_recorder)
        sums = np.array([n, np.sum(self.projection_2d_recorder), np.sum(self.add_recorder),
                         np.sum(self.cm_degree_5_recorder)], np.float64)
        if self.batch_totals is not None:
            sums += self.batch_totals[:4].cpu().numpy()
        with np.errstate(invalid="ignore", divide="ignore"):
            proj, add, cm = sums[1] / sums[0], sums[2] / sums[0], sums[3] / sums[0]
        if verbose:
            print('2d projections metric: {}'.format(proj))
            print('ADD metric: {}'.format(add))
            print('5 cm 5 degree metric: {}'.format(cm))
        return proj, add, cm
