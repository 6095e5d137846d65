"""End-to-end inference from host memory: image batches in pinned host buffers -> keypoints
(and optionally covariances) back on the host, the way tools/train_linemod.py:190-205
(`[d.cuda() for d in data]` -> net -> EvalWrapper / UncertaintyEvalWrapper -> `.cpu()`) runs the
hot path, but with the host->device copy of batch i+1 overlapped with the compute of batch i
(two device input buffers, a side stream for copies, CUDA events for ordering; no host
synchronisation inside the loop; `run` synchronises once on the last device->host copy before it
returns, so the host buffers are valid when it does).

Per batch the device work is: `pvnet_backbone_forward` (fused argmax -> uint8 mask) and ONE
`pvnet_ransac_voting_pipeline` call (v3, plus estimate_voting_distribution_with_mean when
`with_covariance`), sampling on the device (rng="device": no torch RNG launches).

With `points_3d` + `camera_matrix` the uncertainty-driven PnP of `Evaluator.evaluate_uncertainty`
(lib/utils/evaluation_utils.py:165-201) runs on the device as well (`pvnet_uncertainty_pnp`), so POSES
[b,3,4] are what leaves the GPU (and what an 8-GPU job gathers).  Where every image has its own camera (the
truncated-LINEMOD loader's `Ks`, tools/train_linemod.py:186-205), build the pipeline with `points_3d` alone and
pass the cameras with the images: `step(x, camera_matrix=Ks)` with a CUDA [b,3,3], `run(host_batches,
camera_matrices=...)` with one host [b,3,3] per batch, copied on the same side stream as its image batch (into a
static device buffer per input buffer, so one captured graph serves every batch).  The solve is then
`pvnet_uncertainty_pnp_per_image_k`.

`graph=True`: the per-batch device work (31 backbone launches + the voting call's ~10 + PnP) is captured into one
CUDA graph per input buffer on first use and replayed afterwards -- 4 us of host time per batch instead of
0.4-5 ms of Python + launches (batch 1: 0.72 ms per image instead of 0.78; at batch 16 the GPU is the limit either
way, the host thread is what is freed).  The device-side sampler keeps drawing fresh samples across replays.

`refine=dict(vertices=, faces=, near=, far=, ...)`: the poses are then refined on the device before they are returned
(`refine.refine_poses` with the step's own fused-argmax mask, PnP poses, keypoints and covariances and its cameras,
the keypoint-anchored objective of DESIGN.md §27), inside the same captured graph when graph=True.  The mesh goes to
the device once.  With `refine=dict(..., depth=dict(gate=, rounds=8, max_points=4096, depth_scale=1.0))` the refined
poses are then refined again against each image's registered depth (`refine.refine_poses_depth`, DESIGN.md §28):
`step(x, depth=)` takes a CUDA [b,H,W] float32 or uint16, `run(..., depths=)` one host [b,H,W] per batch, copied on
the side stream into a static device buffer per input buffer like the cameras.  The mesh, clip planes and cameras are
refine's; depth-only refinement is `refine=dict(..., rounds=0, depth=...)`.

`max_instances=I` (DESIGN.md §30): several objects of one class per image.  The step then splits each image's
foreground into up to I instances with `ransac_voting_center` on the centre field (the last keypoint), votes every
instance's keypoints and covariances with `ransac_voting_labels`, and solves one pose per instance with
`extend_utils.uncertainty_pnp_instances`: `step` and `run` return (labels [b,H,W] int32, num [b] int32, keypoints
[b,I,K,2], covariances [b,I,K,2,2], poses [b,I,3,4] float64), where row j of image i is an instance when j < num[i]
(the other rows' poses are NaN).  It needs points_3d, a camera and with_covariance=True.  With `refine=` the instance
poses are refined on the label map by `refine.refine_poses_instances` with the step's keypoints and covariances;
`refine['depth']` is not available with max_instances.

Inputs may be float32 [b,3,H,W] (already normalised, what `ToTensor` + `Normalize` produce,
tools/demo.py:89-95) or uint8 [b,H,W,3] raw images: the latter are normalised on the device inside
the packing kernel (4x fewer host->device bytes).
"""
from __future__ import annotations

import numpy as np
import torch

from . import extend_utils as eu
from . import ransac_voting_gpu as rv
from . import refine as rfn

IMAGENET_MEAN = (0.485, 0.456, 0.406)      # tools/demo.py:91-94, lib/datasets/linemod_dataset.py:191-195
IMAGENET_STD = (0.229, 0.224, 0.225)


class PoseKeypointPipeline:
    def __init__(self, net, round_hyp_num=256, inlier_thresh=0.99, rng="device", with_covariance=False,
                 cov_round_hyp_num=256, cov_min_hyp_num=4096, max_num=30000, mean=IMAGENET_MEAN, std=IMAGENET_STD,
                 points_3d=None, camera_matrix=None, graph=False, refine=None, max_instances=None):
        self.net = net
        self.graph = bool(graph)
        self.hn = round_hyp_num
        self.thresh = inlier_thresh
        self.rng = rng
        self.with_cov = with_covariance
        self.cov_hn = cov_round_hyp_num
        self.cov_min = cov_min_hyp_num
        self.max_num = max_num
        self.mean, self.std = tuple(mean), tuple(std)
        self.with_pose = points_3d is not None and camera_matrix is not None
        if self.with_pose and not with_covariance:
            raise ValueError("poses need the covariances: with_covariance=True")
        if self.graph and rng != "device":
            raise ValueError("graph=True needs rng='device' (torch's generator cannot be replayed)")
        self.points_3d, self.camera_matrix = points_3d, camera_matrix
        self.max_instances = None
        if max_instances is not None:
            if isinstance(max_instances, bool) or int(max_instances) != max_instances or not 1 <= max_instances <= 32:
                raise ValueError(f"max_instances must be an integer in 1..32, got {max_instances!r}")
            if points_3d is None or not with_covariance:
                raise ValueError("max_instances needs points_3d and with_covariance=True")
            if rng != "device":
                raise ValueError("max_instances needs rng='device' (the instance split draws on the device)")
            if refine is not None and refine.get("depth") is not None:
                raise ValueError("refine['depth'] is not available with max_instances")
            self.max_instances = int(max_instances)
        self.refine = None
        if refine is not None:
            if points_3d is None or not with_covariance:
                raise ValueError("refine needs points_3d and with_covariance=True")
            cfg = dict(rounds=8, gate=20.0, max_points=4096, keypoint_weight=rfn.DEFAULT_KEYPOINT_WEIGHT, depth=None)
            unknown = set(refine) - {"vertices", "faces", "near", "far", *cfg}
            missing = {"vertices", "faces", "near", "far"} - set(refine)
            if unknown or missing:
                raise ValueError(f"refine: unknown keys {sorted(unknown)}, missing keys {sorted(missing)}")
            cfg.update(refine)
            if cfg["depth"] is not None:
                dcfg = dict(rounds=8, max_points=4096, depth_scale=1.0)
                unknown = set(cfg["depth"]) - {"gate", *dcfg}
                if unknown or "gate" not in cfg["depth"]:
                    raise ValueError(f"refine['depth']: unknown keys {sorted(unknown)}; gate is required")
                dcfg.update(cfg["depth"])
                cfg["depth"] = dcfg
            self.refine = cfg
        self._mesh_dev = None                       # (device, vertices, faces, constructor K or None)
        self._p3_dev = None
        # max_instances: the constructor's host camera is snapshotted here and goes to the device once
        host_k = camera_matrix is not None and not (isinstance(camera_matrix, torch.Tensor) and camera_matrix.is_cuda)
        self._k_host = torch.tensor(np.asarray(camera_matrix, np.float64)).reshape(3, 3) if host_k else None
        self._k_dev = None                          # the snapshot on the device
        self._bufs = None
        self._kbufs = None
        self._dbufs = None
        self._copy_stream = None

    @property
    def _with_depth(self):
        return self.refine is not None and self.refine["depth"] is not None

    def _setup(self, host_batch, dev, per_batch_k, host_depth=None):
        if (self._bufs is None or self._bufs[0].shape != host_batch.shape or self._bufs[0].dtype != host_batch.dtype
                or self._bufs[0].device != dev or (self._kbufs is not None) != per_batch_k
                or (self._dbufs is not None) != (host_depth is not None)
                or (host_depth is not None and (self._dbufs[0].shape != host_depth.shape
                                                or self._dbufs[0].dtype != host_depth.dtype))):
            self._bufs = [torch.empty(host_batch.shape, dtype=host_batch.dtype, device=dev) for _ in range(2)]
            # per input buffer: the batch's cameras, float64 [b,3,3] (static, so a captured graph reads each batch's)
            self._kbufs = ([torch.empty([host_batch.shape[0], 3, 3], dtype=torch.float64, device=dev) for _ in range(2)]
                           if per_batch_k else None)
            # per input buffer: the batch's registered depth (static, like the cameras)
            self._dbufs = ([torch.empty(host_depth.shape, dtype=host_depth.dtype, device=dev) for _ in range(2)]
                           if host_depth is not None else None)
            self._ready = [torch.cuda.Event() for _ in range(2)]      # H2D of buffer i finished
            self._free = [torch.cuda.Event() for _ in range(2)]       # compute no longer reads buffer i
            self._done = torch.cuda.Event()                           # last D2H of a run() finished
            self._copy_stream = torch.cuda.Stream(device=dev)
            self._graphs = [None, None]                               # per input buffer: (CUDAGraph, static result)
            for e in self._free:
                e.record(torch.cuda.current_stream(dev))

    def _step_graph(self, j):
        """Replay (capture on first use) the graph of `step(self._bufs[j], self._kbufs[j], self._dbufs[j])` on the
        current stream."""
        if self._graphs[j] is None:
            cur = torch.cuda.current_stream(self._bufs[j].device)
            side = torch.cuda.Stream(device=self._bufs[j].device)
            side.wait_stream(cur)
            k = None if self._kbufs is None else self._kbufs[j]
            d = None if self._dbufs is None else self._dbufs[j]
            with torch.cuda.stream(side):
                self.step(self._bufs[j], k, d)      # eager once on the capture stream: plans, workspaces, attributes
                side.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    res = self.step(self._bufs[j], k, d)
            cur.wait_stream(side)
            self._graphs[j] = (g, res)
        g, res = self._graphs[j]
        g.replay()
        return res

    def step(self, x, camera_matrix=None, depth=None):
        """x on the device: float32 [b,3,H,W] or uint8 [b,H,W,3] -> keypoints [b,K,2]
        (and covariances [b,K,2,2]) (and poses [b,3,4] float64).  camera_matrix: this batch's cameras, a CUDA
        tensor [b,3,3] (or [3,3]), in place of the constructor's; it needs `points_3d` and `with_covariance`.
        depth: this batch's registered depth, a CUDA [b,H,W] float32 or uint16; required exactly when
        refine['depth'] is set."""
        if camera_matrix is not None and (self.points_3d is None or not self.with_cov):
            raise ValueError("per-batch camera matrices need points_3d and with_covariance=True")
        if (depth is not None) != self._with_depth:
            raise ValueError("depth goes with refine['depth'], and refine['depth'] needs depth")
        # pixel-major head output: the vertex field is the contiguous [b,h,w,K,2] form of the permuted view of
        # tools/demo.py:48-50 (same values; the voting layer's gather then reads whole records, not sectors)
        if x.dtype == torch.uint8:
            out, mask = self.net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, mean=self.mean, std=self.std,
                                                pixel_major=True)
        else:
            out, mask = self.net.forward_native(x, with_mask=True, mask_dtype=torch.uint8, pixel_major=True)
        b, h, w, c = out.shape
        k = (c - self.net.seg_dim) // 2
        vertex = out[..., self.net.seg_dim:].unflatten(3, (k, 2))
        if self.max_instances is not None:
            return self._step_instances(mask, vertex, camera_matrix)
        # a 2-class argmax mask is binary: v3's `nonzero` and with_mean's `== 1` readings coincide
        if self.net.seg_dim == 2 or not self.with_cov:
            res = rv.ransac_voting_pipeline(mask, vertex, self.hn, self.thresh, self.with_cov, self.cov_hn, self.cov_min,
                                            self.thresh, max_num=self.max_num, rng=self.rng)
        else:
            kp = rv.ransac_voting_layer_v3(mask, vertex, self.hn, inlier_thresh=self.thresh, max_num=self.max_num,
                                           rng="batched")
            _, cov = rv.estimate_voting_distribution_with_mean(mask, vertex, kp, round_hyp_num=self.cov_hn,
                                                               min_hyp_num=self.cov_min, inlier_thresh=self.thresh,
                                                               max_num=self.max_num, rng="batched")
            res = (kp, cov)
        if self.with_pose or camera_matrix is not None:
            if self._p3_dev is None or self._p3_dev.device != x.device:     # the model points go to the device once
                self._p3_dev = torch.as_tensor(self.points_3d, dtype=torch.float32).to(x.device).contiguous()
            K = self.camera_matrix if camera_matrix is None else camera_matrix
            pose = eu.uncertainty_pnp_batched(res[0], self._p3_dev, K, cov=res[1])
            if self.refine is not None:
                pose = self._refine(mask, pose, K, res[0], res[1], depth)
            return res[0], res[1], pose
        return res

    def _step_instances(self, mask, vertex, camera_matrix):
        """The max_instances step after the backbone: instance split, per-instance vote, per-instance PnP."""
        I = self.max_instances
        labels, num = rv.ransac_voting_center(mask, vertex[..., -1, :], self.hn, self.thresh, max_instances=I)
        kp, cov = rv.ransac_voting_labels(labels, vertex, I, self.hn, self.thresh, True, self.cov_hn, self.cov_min,
                                          self.thresh, max_num=self.max_num)
        if self._p3_dev is None or self._p3_dev.device != mask.device:
            self._p3_dev = torch.as_tensor(self.points_3d, dtype=torch.float32).to(mask.device).contiguous()
        K = self.camera_matrix if camera_matrix is None else camera_matrix
        if K is None:
            raise ValueError("max_instances needs a camera: the constructor's camera_matrix or step's")
        if not (isinstance(K, torch.Tensor) and K.is_cuda):
            if camera_matrix is not None:
                raise ValueError("step's camera_matrix must be a CUDA tensor")
            if self._k_dev is None or self._k_dev.device != mask.device:
                self._k_dev = self._k_host.to(mask.device)
            K = self._k_dev
        pose = eu.uncertainty_pnp_instances(kp, num, self._p3_dev, K, cov=cov)
        if self.refine is not None:
            cfg = self.refine
            v, f = self._mesh(mask.device)
            pose = rfn.refine_poses_instances(labels, num, pose, K, v, f, cfg["near"], cfg["far"], rounds=cfg["rounds"],
                                              gate=cfg["gate"], max_points=cfg["max_points"], keypoints=kp,
                                              points_3d=self._p3_dev, cov=cov, keypoint_weight=cfg["keypoint_weight"])
        return labels, num, kp, cov, pose

    def _mesh(self, dev):
        """The refine mesh on the device, uploaded on first use -> (vertices f32, faces int32)."""
        if self._mesh_dev is None or self._mesh_dev[0] != dev:
            cfg = self.refine
            v = torch.as_tensor(cfg["vertices"], dtype=torch.float32).to(dev).contiguous()
            f = torch.as_tensor(cfg["faces"]).to(dev)
            f = f if f.dtype == torch.int32 else f.to(torch.int32)
            self._mesh_dev = (dev, v, f.contiguous(), None)
        return self._mesh_dev[1], self._mesh_dev[2]

    def _refine(self, mask, pose, K, kp, cov, depth):
        """refine_poses on the step's outputs, then refine_poses_depth on its poses when depth is given; the mesh (and
        a host camera) go to the device on first use."""
        dev = pose.device
        cfg = self.refine
        if self._mesh_dev is None or self._mesh_dev[0] != dev:
            v = torch.as_tensor(cfg["vertices"], dtype=torch.float32).to(dev).contiguous()
            f = torch.as_tensor(cfg["faces"]).to(dev)
            f = f if f.dtype == torch.int32 else f.to(torch.int32)
            k = None                                # the constructor's host camera, if any
            if self.camera_matrix is not None and not (isinstance(self.camera_matrix, torch.Tensor)
                                                       and self.camera_matrix.is_cuda):
                k = torch.as_tensor(self.camera_matrix, dtype=torch.float64).reshape(3, 3).to(dev)
            self._mesh_dev = (dev, v, f.contiguous(), k)
        _, v, f, k_host = self._mesh_dev
        if isinstance(K, torch.Tensor) and K.is_cuda:
            k = K
        elif K is self.camera_matrix and k_host is not None:
            k = k_host
        else:
            k = torch.as_tensor(K, dtype=torch.float64).reshape(3, 3).to(dev)
        pose = rfn.refine_poses(mask, pose, k, v, f, cfg["near"], cfg["far"], rounds=cfg["rounds"], gate=cfg["gate"],
                                max_points=cfg["max_points"], keypoints=kp, points_3d=self._p3_dev, cov=cov,
                                keypoint_weight=cfg["keypoint_weight"])
        if depth is not None:
            d = cfg["depth"]
            pose = rfn.refine_poses_depth(mask, depth, pose, k, v, f, cfg["near"], cfg["far"], gate=d["gate"],
                                          rounds=d["rounds"], max_points=d["max_points"],
                                          depth_scale=d["depth_scale"])
        return pose

    @torch.no_grad()
    def run(self, host_batches, out_host=None, cov_host=None, on_result=None, pose_host=None, camera_matrices=None,
            depths=None):
        """host_batches: sequence of pinned [b,3,H,W] float32 (or [b,H,W,3] uint8) tensors.  Results are
        copied device->host into out_host[i] (and cov_host[i]) -- pinned tensors -- when given; the call
        returns after the last of those copies has completed.  Returns the last device result (with graph=True a
        static tensor that the next replay on the same input buffer overwrites).
        camera_matrices: one host [b,3,3] (or [3,3]) per batch, numpy or CPU tensor (pinned float64 makes the copy as
        asynchronous as the images'): the cameras of that batch's images, used in place of the constructor's.
        depths: one host [b,H,W] float32 or uint16 tensor per batch (pinned, for an asynchronous copy), that batch's
        registered depth; required exactly when refine['depth'] is set."""
        dev = next(self.net.parameters()).device
        batches = list(host_batches)
        if not batches:
            return None
        cams = None
        if camera_matrices is not None:
            cams = [torch.as_tensor(k, dtype=torch.float64) for k in camera_matrices]
            if len(cams) != len(batches):
                raise ValueError(f"{len(cams)} camera batches for {len(batches)} image batches")
            for k in cams:
                eu.check_cameras(k.shape, batches[0].shape[0])
            if self.points_3d is None or not self.with_cov:
                raise ValueError("per-batch camera matrices need points_3d and with_covariance=True")
        if (depths is not None) != self._with_depth:
            raise ValueError("depths go with refine['depth'], and refine['depth'] needs depths")
        if depths is not None:
            depths = list(depths)
            if len(depths) != len(batches):
                raise ValueError(f"{len(depths)} depth batches for {len(batches)} image batches")
            if any(not isinstance(d, torch.Tensor) or d.shape != depths[0].shape or d.dtype != depths[0].dtype
                   for d in depths):
                raise ValueError("depths must be torch tensors of one shape and dtype")
        self._setup(batches[0], dev, cams is not None, None if depths is None else depths[0])
        main = torch.cuda.current_stream(dev)
        cs = self._copy_stream
        result = None

        def upload(i):
            j = i & 1
            cs.wait_event(self._free[j])
            with torch.cuda.stream(cs):
                self._bufs[j].copy_(batches[i], non_blocking=True)
                if cams is not None:
                    self._kbufs[j].copy_(cams[i], non_blocking=True)
                if depths is not None:
                    self._dbufs[j].copy_(depths[i], non_blocking=True)
                self._ready[j].record(cs)
        upload(0)
        for i in range(len(batches)):
            j = i & 1
            if i + 1 < len(batches):
                upload(i + 1)
            main.wait_event(self._ready[j])
            k = None if cams is None else self._kbufs[j]
            d = None if depths is None else self._dbufs[j]
            result = self._step_graph(j) if self.graph else self.step(self._bufs[j], k, d)
            self._free[j].record(main)
            # max_instances: (labels, num, keypoints, cov, poses); otherwise (keypoints, cov[, poses]) or keypoints
            res = result[2:] if self.max_instances is not None else result
            if out_host is not None:
                kp = res[0] if isinstance(res, tuple) else res
                out_host[i].copy_(kp, non_blocking=True)
            if cov_host is not None and isinstance(res, tuple):
                cov_host[i].copy_(res[1], non_blocking=True)
            if pose_host is not None and isinstance(res, tuple) and len(res) > 2:
                pose_host[i].copy_(res[2], non_blocking=True)
            if on_result is not None:
                on_result(i, result)
        if out_host is not None or cov_host is not None or pose_host is not None:
            self._done.record(main)
            self._done.synchronize()
        return result
