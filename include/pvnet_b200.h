/*
 * pvnet_b200.h -- C ABI of libpvnet_b200.so: the H100 (sm_90a) implementation of
 * PVNet's per-image inference hot path (voting layer + Resnet18_8s backbone).
 *
 * Boundary rules (SURVEY.md §8b):
 *   - plain C types only: device pointers, sizes, strides; no torch/ATen types;
 *   - the CALLER owns every buffer, including the workspace; the library allocates
 *     nothing on the hot path and launches only on the given stream (CUDA-graph
 *     capturable); it never synchronises and never calls exit();
 *   - every function returns 0 on success, a negative PVNET_E_* code on failure;
 *     pvnet_last_error() returns a thread-local message for the last failure;
 *   - all pointers are DEVICE pointers on the current CUDA device unless a
 *     parameter says "host".
 *
 * Reference interfaces these entry points stand in for (paths relative to the
 * zju3dv/pvnet tree):
 *   lib/ransac_voting_gpu_layer/src/ransac_voting.cpp:20-31,103   generate_hypothesis
 *   lib/ransac_voting_gpu_layer/src/ransac_voting.cpp:41-55,104   voting_for_hypothesis
 *   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:514-598      ransac_voting_layer_v3
 *   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:333-406      estimate_voting_distribution_with_mean
 *   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:763-858      ransac_voting_layer_v5
 *   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:983-1034     generate_hypothesis (python level)
 *   lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:99-216       ransac_voting_layer_v2 (refinement rounds)
 *   lib/ransac_voting_gpu_layer/src/ransac_voting.cpp:61-99       the vanishing-point kernel pair
 *   tools/train_linemod.py:119-130                                UncertaintyEvalWrapper.forward (v3 + with_mean)
 *   lib/utils/extend_utils/extend_utils.py:63-114                 uncertainty_pnp (+ evaluation_utils.py:165-201)
 *   lib/utils/extend_utils/src/nearest_neighborhood.cu:123-163    findNearestPointIdxLauncher
 *   lib/utils/evaluation_utils.py:75-141                          the pose metrics (ADD(-S), 2D projection, 5 cm 5 deg)
 *   lib/utils/extend_utils/src/farthest_point_sampling.cpp        farthest_point_sampling[_init_center]
 *   lib/utils/extend_utils/src/mesh_rasterization.cpp             mesh_binary_rasterization
 *   lib/utils/opengl_render_backend.py:306-419                    render (depth and flat RGB)
 *   lib/utils/data_utils.py:788-826                               get_mask_of_all_objects (label map)
 *   lib/utils/net_utils.py:54-80,329-348                          smooth_l1_loss, compute_precision_recall
 *   tools/train_linemod.py:83-91                                  NetWrapper's cross-entropy (nn.CrossEntropyLoss)
 *   lib/networks/model_repository.py:64-80                        Resnet18_8s.forward
 *   tools/train_linemod.py:260                                    optim.Adam's step
 * INTEGRATION.md shows the ctypes binding the reference's Python wrapper uses.
 */
#ifndef PVNET_B200_H_
#define PVNET_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define PVNET_API __attribute__((visibility("default")))
#else
#define PVNET_API
#endif

/* opaque: a cudaStream_t passed as void* (torch: torch.cuda.current_stream().cuda_stream) */
typedef void *pvnet_stream_t;

enum {
    PVNET_OK = 0,
    PVNET_E_INVALID = -1,   /* bad argument (shape, stride, null pointer, size) */
    PVNET_E_WORKSPACE = -2, /* workspace too small */
    PVNET_E_CUDA = -3,      /* a CUDA runtime / driver call failed */
    PVNET_E_STATE = -4      /* object used before it was initialised */
};

/* How a mask element becomes "foreground". */
enum {
    PVNET_MASK_NONZERO_BYTE = 0, /* v3: `.byte()` then nonzero  (ransac_voting_gpu.py:527) */
    PVNET_MASK_EQUALS_ONE = 1    /* with_mean: `mask == 1`      (ransac_voting_gpu.py:339) */
};

PVNET_API const char *pvnet_last_error(void);
/* ABI version.  2: backbone slot 0 holds the stem in its space-to-depth packing (was [7*7][3][64]) and the
 * backbone has 26 conv slots.  3: pvnet_backbone_create_trunk builds a backbone from a trunk description
 * (BasicBlock or Bottleneck, blocks per stage; Resnet34_8s, Resnet50_8s), whose conv-slot count and stage list are
 * per handle (pvnet_backbone_handle_num_convs / _num_stages / _stage_name); raw_dim may be 64 there; the
 * train-mode BatchNorm's block-tail forms (1, 2) take up to 2048 channels. */
PVNET_API int pvnet_version(void);

/* ------------------------------------------------------------------ voting layer */

/* Bytes of workspace the fused voting entry points need for a batch of `b` images
 * of h*w pixels, `vn` keypoints and `hn_total` hypotheses per keypoint. */
PVNET_API int pvnet_vote_workspace_bytes(int b, int h, int w, int vn, int hn_total, size_t *bytes);

/* Per-image foreground counts (before any subsampling): fg_out[b] int32.
 * mask: [b,h,w] contiguous, elements of mask_elem_size bytes (1,2,4,8; integer or bool).
 * The host reads fg_out to replay the reference's torch RNG calls in the reference's
 * order (ransac_voting_gpu.py:531-547); nothing else in the layer needs the host. */
PVNET_API int pvnet_mask_foreground_count(const void *mask, int mask_elem_size, int mask_mode,
                                          int b, int h, int w, int32_t *fg_out,
                                          void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* ransac_voting_layer_v3 (ransac_voting_gpu.py:514-598), whole batch, no host sync.
 *
 *   mask       [b,h,w] contiguous, foreground = low byte nonzero
 *   vertex     f32, logical shape [b,h,w,vn,2], addressed through vertex_strides[5]
 *              (in ELEMENTS).  The reference passes a permuted view of an NCHW tensor
 *              (tools/demo.py:48-50): strides {C*H*W, W, 1, 2*H*W, H*W}; it is read
 *              in place, never copied.
 *   idxs       int32 [b,hn,vn,2]: the pixel-pair samples (ransac_voting_gpu.py:547).
 *              Each value is reduced modulo the image's pixel count tn (identity for
 *              values already in [0,tn)).
 *   selection  f32 [b,h,w] or NULL: the uniform field of ransac_voting_gpu.py:538.
 *              Read only for images whose foreground count exceeds max_num; NULL means
 *              "never subsample" (all foreground pixels take part).
 *   out_pts    f32 [b,vn,2]  voted + least-squares-refitted keypoints (x,y);
 *              zeros for images with fewer than min_num foreground pixels (:531-534).
 *   out_counts int32 [b,hn,vn] or NULL: inlier count of every hypothesis (:561).
 *   out_hyp    f32 [b,hn,vn,2] or NULL: the hypotheses (:554).
 *   out_tn     int32 [b] or NULL: pixels that took part per image (after subsampling).
 *
 * The reference's `while True` (:552-576) re-scores the same idxs each round, so its
 * output does not depend on confidence/max_iter; one scoring pass is performed.
 */
PVNET_API int pvnet_ransac_voting_v3(const void *mask, int mask_elem_size,
                                     const float *vertex, const int64_t vertex_strides[5],
                                     const int32_t *idxs, const float *selection,
                                     int b, int h, int w, int vn, int hn,
                                     float inlier_thresh, int min_num, int max_num,
                                     float *out_pts, int32_t *out_counts, float *out_hyp, int32_t *out_tn,
                                     void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* One refinement round of ransac_voting_layer_v2 (ransac_voting_gpu.py:178-204) for a whole batch: the
 * pixels (mask low byte nonzero, subsampled like v3) that are inliers of points [b,vn,2] re-estimate
 * them as the least-squares intersection of their lines -> out_pts [b,vn,2].  The reference's
 * pinverse(A) b equals this normal-equation solution for full-rank A.  Workspace:
 * pvnet_vote_workspace_bytes(b, h, w, vn, 1). */
PVNET_API int pvnet_refit_at_points(const void *mask, int mask_elem_size,
                                    const float *vertex, const int64_t vertex_strides[5],
                                    const float *selection, const float *points,
                                    int b, int h, int w, int vn, float inlier_thresh, int min_num, int max_num,
                                    float *out_pts, void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* ransac_voting_layer_v5 (ransac_voting_gpu.py:763-858): v3 plus a per-keypoint confidence
 * out_conf [b,vn] = (inliers of the refitted point at conf_thresh, 0.999 in the reference :850)
 * / tn; zeros for skipped images (:788-793).  Same arguments as pvnet_ransac_voting_v3 otherwise. */
PVNET_API int pvnet_ransac_voting_v5(const void *mask, int mask_elem_size,
                                     const float *vertex, const int64_t vertex_strides[5],
                                     const int32_t *idxs, const float *selection,
                                     int b, int h, int w, int vn, int hn,
                                     float inlier_thresh, float conf_thresh, int min_num, int max_num,
                                     float *out_pts, float *out_conf, int32_t *out_counts, float *out_hyp,
                                     int32_t *out_tn, void *workspace, size_t workspace_bytes,
                                     pvnet_stream_t stream);

/* ransac_voting_layer_v4 (ransac_voting_gpu.py:669-760): v3 plus the residual variance of the
 * refit, out_var [b,vn] = sum over the winner's inliers of (n.p - n.c)^2 / #inliers with
 * n = (d_y,-d_x) and p the refitted point (:750-752; 0/0 = NaN as in torch); a skipped image
 * gives zeros and var = 1 (:685-689).  Same arguments as pvnet_ransac_voting_v3 otherwise. */
PVNET_API int pvnet_ransac_voting_v4(const void *mask, int mask_elem_size,
                                     const float *vertex, const int64_t vertex_strides[5],
                                     const int32_t *idxs, const float *selection,
                                     int b, int h, int w, int vn, int hn,
                                     float inlier_thresh, int min_num, int max_num,
                                     float *out_pts, float *out_var, int32_t *out_counts, float *out_hyp,
                                     int32_t *out_tn, void *workspace, size_t workspace_bytes,
                                     pvnet_stream_t stream);

/* ransac_motion_voting (ransac_voting_gpu.py:960-981; tools/train_linemod.py:117
 * `MotionEvalWrapper`): out_pts [b,vn,2] = mean over the foreground pixels (low byte nonzero, as
 * `.byte()`) of vertex + (x, y); zeros for an empty mask (:971-973).  Workspace:
 * pvnet_vote_workspace_bytes(b, h, w, vn, 1). */
PVNET_API int pvnet_ransac_motion_voting(const void *mask, int mask_elem_size,
                                         const float *vertex, const int64_t vertex_strides[5],
                                         int b, int h, int w, int vn, float *out_pts,
                                         void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* estimate_voting_distribution_with_mean (ransac_voting_gpu.py:333-406).
 *
 *   mask       foreground = element == 1
 *   idxs       int32 [b,rounds*hn,vn,2], rounds = ceil(min_hyp_num/hn) (fresh draw per
 *              round, :367; the rounds are simply concatenated, :381-384)
 *   mean       f32 [b,vn,2] (from v3)
 *   out_cov    f32 [b,vn,2,2]: sum_h w_h d_h d_h^T / (sum_h w_h + 1e-3), d_h = hyp_h - mean,
 *              w_h = count_h/tn, zeroed where below (max_h w_h - 0.1)   (:394-401)
 *   Images with fewer than min_num foreground pixels use min_hyp_num hypotheses at
 *   (0,0) with weight 1 (:343-348).
 */
PVNET_API int pvnet_vote_cov_with_mean(const void *mask, int mask_elem_size,
                                       const float *vertex, const int64_t vertex_strides[5],
                                       const int32_t *idxs, const float *selection, const float *mean,
                                       int b, int h, int w, int vn, int hn, int rounds, int min_hyp_num,
                                       float inlier_thresh, int min_num, int max_num,
                                       float *out_cov, int32_t *out_counts, float *out_hyp, int32_t *out_tn,
                                       void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* The uncertainty pipeline of tools/train_linemod.py:119-130 (`UncertaintyEvalWrapper.forward`):
 *     mean      = ransac_voting_layer_v3(mask, vertex, hn, inlier_thresh)            (ransac_voting_gpu.py:514-598)
 *     mean, cov = estimate_voting_distribution_with_mean(mask, vertex, mean, ...)     (ransac_voting_gpu.py:333-406)
 * as ONE launch sequence: the mask is compacted and the vector field gathered once for both
 * layers, and when both thresholds agree one kernel scores the v3 and the covariance hypotheses
 * together.  out_cov == NULL runs the v3 part alone.
 *
 *   mask_mode  how BOTH layers read the mask.  The reference's v3 takes nonzero (:527) and
 *              with_mean takes == 1 (:339); for the binary argmax mask of a 2-class network the
 *              two agree and either mode gives the reference's result.  (Callers with other
 *              masks use the two separate entry points.)
 *   idxs       int32 [b,hn,vn,2] or NULL; cov_idxs int32 [b,cov_rounds*cov_hn,vn,2] or NULL;
 *              selection f32 [b,h,w] or NULL (one field for both layers)
 *   rng_state  DEVICE pointer to {uint64 seed, uint64 offset} or NULL.  Whatever sample set is
 *              NULL is drawn on the device (Philox4x32-10; idxs = 32 random bits modulo tn like
 *              torch's random_, selection = 24 bits * 2^-24 like uniform_); the call then advances
 *              the offset, so a captured CUDA graph draws fresh samples on every replay.
 *              With rng_state == NULL a NULL selection means "never subsample".
 *   out_pts    f32 [b,vn,2]; out_cov f32 [b,vn,2,2] or NULL
 *   out_counts/out_hyp [b,hn,vn(,2)], out_cov_counts/out_cov_hyp [b,cov_rounds*cov_hn,vn(,2)],
 *   out_tn [b]: optional debug outputs.
 *   Workspace: pvnet_vote_workspace_bytes(b, h, w, vn, hn + cov_rounds*cov_hn). */
PVNET_API int pvnet_ransac_voting_pipeline(const void *mask, int mask_elem_size, int mask_mode,
                                           const float *vertex, const int64_t vertex_strides[5],
                                           const int32_t *idxs, const int32_t *cov_idxs, const float *selection,
                                           const unsigned long long *rng_state,
                                           int b, int h, int w, int vn, int hn, float inlier_thresh,
                                           int cov_hn, int cov_rounds, int cov_min_hyp_num, float cov_inlier_thresh,
                                           int min_num, int max_num, float *out_pts, float *out_cov,
                                           int32_t *out_counts, float *out_hyp,
                                           int32_t *out_cov_counts, float *out_cov_hyp, int32_t *out_tn,
                                           void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* 1:1 stand-ins for the reference extension's two functions, same layouts:
 * direct [tn,vn,2] f32, coords [tn,2] f32 (x,y), idxs [hn,vn,2] i32, hypo [hn,vn,2] f32.
 * pvnet_generate_hypothesis writes every element of hypo (degenerate pairs -> (0,0),
 * ransac_voting_kernel.cu:42-43,75).  pvnet_voting_for_hypothesis only SETS inliers
 * [hn,vn,tn] u8 to 1 where the test passes (caller zero-fills, ransac_voting_gpu.py:557).
 * pvnet_vote_counts returns sum_t inliers as int32 [hn,vn] without the u8 tensor. */
PVNET_API int pvnet_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs,
                                        float *hypo, int tn, int vn, int hn, pvnet_stream_t stream);
PVNET_API int pvnet_voting_for_hypothesis(const float *direct, const float *coords, const float *hypo,
                                          uint8_t *inliers, int tn, int vn, int hn, float inlier_thresh,
                                          pvnet_stream_t stream);
PVNET_API int pvnet_vote_counts(const float *direct, const float *coords, const float *hypo,
                                int32_t *counts, int tn, int vn, int hn, float inlier_thresh,
                                pvnet_stream_t stream);

/* ------------------------------------------------------------------ uncertainty-driven PnP
 * The consumer of the keypoints + covariances above (SURVEY.md section 8 f-1); reference, per image on the
 * host: lib/utils/evaluation_utils.py:165-201 (`Evaluator.evaluate_uncertainty`) ->
 * lib/utils/extend_utils/extend_utils.py:63-114 (`uncertainty_pnp`) ->
 * lib/utils/extend_utils/src/uncertainty_pnp.cpp:61-92 (Ceres LM over 2 pn residuals x 6 parameters).
 *
 * pvnet_covariance_to_weights: cov f32 [n,2,2] -> weights f32 [n,3] = (wxx, wxy, wyy) of inv(sqrtm(cov)),
 *   zeros where cov[0,0] < 1e-6 or any element is NaN (evaluation_utils.py:170-181) or the matrix is not
 *   positive definite (where scipy's sqrtm + inv would fail).
 * pvnet_uncertainty_pnp: batched form of extend_utils.py:63 `uncertainty_pnp(points_2d, weights_2d,
 *   points_3d, camera_matrix)`: points_2d f32 [b,pn,2]; EITHER weights_2d f32 [b,pn,3] OR cov f32
 *   [b,pn,2,2] (converted as above; pass NULL for the other); points_3d f32 [pn,3] (one object);
 *   camera_matrix: HOST array of 9 doubles (row-major K).  4 <= pn <= 32.  One warp per image, fp64:
 *   P3P (Grunert; quartic roots by Durand-Kerner, fp32 then fp64 on all four at once, real ones Newton-polished
 *   in fp64) on the first three of the four points with the largest wxx + wxy (extend_utils.py:84;
 *   the fourth disambiguates, as OpenCV's SOLVEPNP_P3P), then Levenberg-Marquardt on
 *   sum_i |W_i (proj(R X_i + t) - x_i)|^2 (uncertainty_pnp.cpp:20-37) to the stationary point: it stops after
 *   taking a step with max |delta| < 1e-9 (pn == 4 returns the P3P pose, :90-94).
 *   out_pose f64 [b,3,4] = (R | t) like the reference's return value; out_info int32 [b,2] or NULL =
 *   (status bits: 1 = P3P found no solution and the identity start was used, 2 = the 500-iteration cap was hit and
 *   the pose is not converged, 4 = see pvnet_uncertainty_pnp_per_image_k;
 *   LM iterations).  A zero fx or fy in camera_matrix is refused (PVNET_E_INVALID).
 * pvnet_uncertainty_pnp_per_image_k: the same solve with one camera per image, as the truncated-LINEMOD loader
 *   supplies them (lib/datasets/linemod_dataset.py:206-207, tools/train_linemod.py:199-205): every argument as
 *   above except camera_matrices, a DEVICE array of doubles [b,3,3] (row-major K per image, contiguous).  Image i
 *   is solved with its own K exactly as pvnet_uncertainty_pnp solves it with that K: same kernel, same launch, bit
 *   for bit the same pose and info.  Both entries read fx, cx, fy, cy (K[0], K[2], K[4], K[5]) and ignore the rest.
 *   An image whose K has fx == 0 or fy == 0 is not solved: its pose is NaN and its status is 4; the other images
 *   are unaffected.  The K are read on the device only: the call does not synchronise and is graph-capturable. */
PVNET_API int pvnet_covariance_to_weights(const float *cov, int n, float *weights, pvnet_stream_t stream);
PVNET_API int pvnet_uncertainty_pnp(const float *points_2d, const float *cov, const float *weights_2d,
                                    const float *points_3d, const double camera_matrix[9], int b, int pn,
                                    double *out_pose, int32_t *out_info, pvnet_stream_t stream);
PVNET_API int pvnet_uncertainty_pnp_per_image_k(const float *points_2d, const float *cov, const float *weights_2d,
                                                const float *points_3d, const double *camera_matrices, int b, int pn,
                                                double *out_pose, int32_t *out_info, pvnet_stream_t stream);

/* ------------------------------------------------------------------ EPnP
 * The reference's `pnp(points_3d, points_2d, camera_matrix, method=cv2.SOLVEPNP_EPNP)` (lib/utils/evaluation_utils.py:
 * 19-52, :26-28) for a batch: Lepetit, Moreno-Noguer and Fua's closed-form EPnP (IJCV 2009), one warp per image, fp64
 * (csrc/epnp.cu; oracle/epnp_oracle.py restates it in numpy).  Fixed work per image: no iteration count depends on
 * the data except the Jacobi eigen-solvers', which stop after at most 30 (3x3) and 20 (12x12) sweeps.
 * pvnet_epnp:
 *   points_2d      f32 [b,pn,2]  image points (pixels) of every image, device
 *   points_3d      f32 [pn,3]    object points, one object for the whole batch, device
 *   camera_matrix  HOST array of 9 doubles (row-major K); fx, cx, fy, cy (K[0], K[2], K[4], K[5]) are read; a zero
 *                  fx or fy is refused (PVNET_E_INVALID)
 *   b              >= 1 images
 *   pn             4 <= pn <= 4096 correspondences (cv2.solvePnP needs 4; every sum strides over the points)
 *   out_pose       f64 [b,3,4] = (R | t), the reference's return value, device
 *   out_info       int32 [b,2] or NULL = (status bits, the linearisation N in 1..3 whose pose was kept); status 1:
 *                  the object points' PCA is rank-deficient (coplanar or collinear: smallest eigenvalue <= 1e-10 of
 *                  the largest), the pose is still computed but is unreliable, as OpenCV's is there; 4: fx or fy is 0
 *                  (per-image entry only), the pose is NaN
 *   stream         CUDA stream; no workspace, no allocation, no host synchronisation: graph-capturable
 * pvnet_epnp_per_image_k: the same with camera_matrices, a DEVICE array of doubles [b,3,3] (one K per image).  Same
 *   kernel and launch: image i gets bit for bit the pose pvnet_epnp gives it with that K.  An image whose K has
 *   fx == 0 or fy == 0 gets status 4 and a NaN pose; the other images are unaffected. */
PVNET_API int pvnet_epnp(const float *points_2d, const float *points_3d, const double camera_matrix[9], int b, int pn,
                         double *out_pose, int32_t *out_info, pvnet_stream_t stream);
PVNET_API int pvnet_epnp_per_image_k(const float *points_2d, const float *points_3d, const double *camera_matrices,
                                     int b, int pn, double *out_pose, int32_t *out_info, pvnet_stream_t stream);

/* ------------------------------------------------------------------ pose evaluation
 * The metrics tools/train_linemod.py:177-229 (`val()`) reports, computed per image on the host there
 * (lib/utils/evaluation_utils.py:75-141).
 *
 * pvnet_find_nearest_point_idx: replaces findNearestPointIdxLauncher
 *   (lib/utils/extend_utils/src/nearest_neighborhood.cu:123-163, called by extend_utils.py:39-60).  For every
 *   query point the index of the nearest reference point of the same image: ref_pts f32 [b,pn1,dim], que_pts f32
 *   [b,pn2,dim], idxs int32 [b,pn2]; dim 2 or 3.  Bit-identical to the reference kernel: the same FP32 rounding
 *   sequence (DESIGN.md §2), a NaN distance never wins, ties keep the lowest index, and a query with no finite
 *   distance below FLT_MAX gets 0.  (The reference's exclude_self has no caller and is not provided.)
 *
 * pvnet_pose_metrics: evaluation_utils.py:75-141 for a batch of images of one object.
 *   pose_pred, pose_gt f64 [b,3,4] (R | t); model f32 [n,3] (the mesh vertices, get_ply_model);
 *   the camera is EITHER camera_matrix, a HOST array of 9 doubles (row-major K, one for all images), OR
 *   camera_dev, a device f64 [b,3,3] (per-image K, intri_type 'use_intrinsic'); pass NULL for the other.
 *   out f64 [b,4] = (add, proj, trans_cm, angle_deg):
 *     add       mean over vertices of |(R_p X + t_p) - (R_g X + t_g)|                      (:97-98,115)
 *               symmetric != 0: ADD-S, the distance from every gt-transformed vertex to the nearest
 *               pred-transformed vertex, searched as above on the fp32 roundings          (:125-128, :54-62)
 *     proj      mean pixel distance of the two projections (R X + t) K^T -> [:2] / z      (:76-78)
 *               sym_proj != 0: the nearest-point form of projection_2d_sym                (:83-86)
 *     trans_cm  100 |t_p - t_g|;  angle_deg = deg(acos((min(tr(R_p R_g^T), 3) - 1) / 2))    (:136-140)
 *   The fp64 operation order of the transform and the projection is fixed (eval.cu); the result is
 *   run-to-run deterministic.  Workspace: pvnet_pose_metrics_workspace_bytes(b, n). */
PVNET_API int pvnet_find_nearest_point_idx(const float *ref_pts, const float *que_pts, int32_t *idxs,
                                           int b, int pn1, int pn2, int dim, pvnet_stream_t stream);
PVNET_API int pvnet_pose_metrics_workspace_bytes(int b, int n, size_t *bytes);
PVNET_API int pvnet_pose_metrics(const double *pose_pred, const double *pose_gt, const float *model, int n,
                                 const double camera_matrix[9], const double *camera_dev, int b,
                                 int symmetric, int sym_proj, double *out,
                                 void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* ------------------------------------------------------------------ validation losses
 * The per-image figures the reference's NetWrapper.forward (tools/train_linemod.py:79-91, tools/demo.py:31-43)
 * computes from the full-resolution outputs and val() prints, in one pass over them (losses.cu, DESIGN.md §10):
 *   loss_seg     f32 [b]  nn.CrossEntropyLoss(reduce=False) then the mean over pixels  (train_linemod.py:83,87-88):
 *                         -log_softmax(seg)[t] in fp32 as torch computes it; t = -100 (ignore_index) adds 0 and still
 *                         counts; any other t outside [0,C) makes the image's value NaN (torch: a device-side assert)
 *   loss_vertex  normalize != 0: f32 [b] = sum(in) / (ver_dim * sum(w) + 1e-3) per image   (net_utils.py:73-74);
 *                normalize == 0: f32 [b,ver_dim,h,w] contiguous, the elementwise `in_loss` (net_utils.py:64-71),
 *                bit-identical to torch's chain of fp32 ops, with c1 = 1/sigma^2, c2 = sigma^2/2, c3 = 0.5/sigma^2
 *                derived in double from `sigma` and rounded to float.  (The reference's reduce=True computes a mean
 *                and discards it, :76-77; the value stays per image.)
 *   precision, recall  f32 [b]  compute_precision_recall (net_utils.py:329-348): argmax over the C channels (first
 *                maximum, a NaN wins), exact int64 counts tp, fp, fn, then (tp+1)/(tp+fp+1) and (tp+1)/(tp+fn+1) in
 *                fp32: bit-identical to torch's fp32 sums while those stay below 2^24; above that the counts are
 *                exact and rounded once, where torch's fp32 sums depend on its summation order.
 * A NULL output skips its part.  Inputs are read in place with ELEMENT strides (the stride along w must be 1):
 *   seg_pred f32 [b,C,h,w] (seg_strides[4]) and mask [b,h,w] (mask_strides[3], elements of mask_elem_size bytes:
 *   8 int64, 4 int32, 1 uint8 / bool) for loss_seg / precision / recall;
 *   vertex_pred, vertex f32 [b,ver_dim,h,w] and vertex_weights f32 [b,1,h,w] (strides[4] each) for loss_vertex.
 *   vertex_weights and weight_strides both NULL: each pixel's weight is its mask value converted to float, the
 *   loader's vertex_weights = mask.unsqueeze(0).float() (linemod_dataset.py:227), read where the weights would be
 *   read, so every output equals the call with that tensor; the mask is then needed for loss_vertex.  A NULL
 *   vertex_weights with non-NULL strides is refused.  The same rule holds for the _keypoints and _backward forms.
 * seg_pred and vertex_pred may be channel slices of one [b,C+ver_dim,h,w] tensor (Resnet18_8s.forward,
 * model_repository.py:77-78).  Sums are fp64 / int64 in a fixed order: run-to-run identical, graph capturable.
 * Workspace: pvnet_seg_vertex_losses_workspace_bytes(b, h, w). */
PVNET_API int pvnet_seg_vertex_losses_workspace_bytes(int b, int h, int w, size_t *bytes);
PVNET_API int pvnet_seg_vertex_losses(const float *seg_pred, const int64_t seg_strides[4],
                                      const void *mask, int mask_elem_size, const int64_t mask_strides[3],
                                      const float *vertex_pred, const int64_t pred_strides[4],
                                      const float *vertex, const int64_t vertex_strides[4],
                                      const float *vertex_weights, const int64_t weight_strides[4],
                                      int b, int h, int w, int C, int ver_dim, double sigma, int normalize,
                                      float *loss_seg, float *loss_vertex, float *precision, float *recall,
                                      void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* Keypoint targets (losses.cu, DESIGN.md §12): the ground-truth vertex field of the reference's loader,
 * compute_vertex_hcoords (lib/datasets/linemod_dataset.py:68-81; tools/demo.py:58-71 is the case hw = 1), built from
 * the mask and the keypoints instead of read from memory.  hcoords is device memory [b,K,3] contiguous, float32
 * (hcoords_f64 == 0) or float64; each (hx, hy, hw) is widened to fp64.  For a pixel (x, y) with mask == 1 (exactly 1:
 * a value of 2 is background) and keypoint k, every op rounded on its own as numpy does:
 *   vx = hx - x*hw, vy = hy - y*hw; unless use_motion: n = sqrt(vx*vx + vy*vy), n < 1e-3 -> n + 1e-3, v = v / n;
 *   channel 2k = (float)vx, channel 2k+1 = (float)vy (round to nearest); every other pixel +0.0f.
 * NaN and inf propagate as in numpy.  The field is bit-identical to the reference's for the hcoords passed in.
 *
 * pvnet_vertex_targets: writes the field to vertex_out f32 [b,2K,h,w] contiguous (the loader's [h,w,2K] after
 *   permute(2,0,1)).  mask as for pvnet_seg_vertex_losses (element strides, unit stride along w).
 * pvnet_seg_vertex_losses_keypoints: pvnet_seg_vertex_losses with the vertex targets computed as above in place of
 *   `vertex` (ver_dim must be 2K); the mask is read for loss_vertex too.  Every output is bit-identical to
 *   pvnet_seg_vertex_losses on the field pvnet_vertex_targets writes.  Same workspace query, same NULL-output rule,
 *   same determinism; graph capturable. */
PVNET_API int pvnet_vertex_targets(const void *mask, int mask_elem_size, const int64_t mask_strides[3],
                                   const void *hcoords, int hcoords_f64, int b, int h, int w, int K, int use_motion,
                                   float *vertex_out, pvnet_stream_t stream);
PVNET_API int pvnet_seg_vertex_losses_keypoints(const float *seg_pred, const int64_t seg_strides[4],
                                                const void *mask, int mask_elem_size, const int64_t mask_strides[3],
                                                const float *vertex_pred, const int64_t pred_strides[4],
                                                const void *hcoords, int hcoords_f64, int use_motion,
                                                const float *vertex_weights, const int64_t weight_strides[4],
                                                int b, int h, int w, int C, int ver_dim, double sigma, int normalize,
                                                float *loss_seg, float *loss_vertex, float *precision, float *recall,
                                                void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* Gradients of the training losses (losses.cu, DESIGN.md §13): d loss_seg / d seg_pred and d loss_vertex /
 * d vertex_pred for the normalised loss_vertex (normalize must be nonzero), each the sequence torch's CUDA autograd
 * runs through the reference's expressions (nn.CrossEntropyLoss(reduction='none') + .view(b,-1).mean(1);
 * net_utils.py:54-80 with torch.pow(diff, 2)), every op rounded on its own.  Per image, with N = h*w:
 *   seg:    g = gs * (1.0f / (float)N) with gs = grad_loss_seg[b]; lp_c = (x_c - m) - logf(s) as in the forward;
 *           S = 0 + sum_c gO_c in channel order with gO_t = -g at the target and 0 elsewhere;
 *           grad_seg_c = fmaf(-expf(lp_c), S, gO_c).  t = -100 gives gO = 0 (0 in every channel unless the pixel's
 *           log-softmax is NaN, as in torch); any other t outside [0,C) makes every element of the image NaN.
 *   vertex: gi = gv / (ver_dim*sum(w) + 1e-3f) with gv = grad_loss_vertex[b] and the forward's denominator bit for
 *           bit (recomputed in the forward's summation order); d = w*(p - t), s = |d| < 1/sigma^2,
 *           grad_vertex = (((gi*s)*c2)*(2*d) + (gi*(1 - s))*sgn(d)) * w, c2 = sigma^2/2 rounded to float,
 *           sgn(+-0) = sgn(NaN) = 0.
 * Inputs as for pvnet_seg_vertex_losses / _keypoints.  grad_loss_seg, grad_loss_vertex: f32 [b] device, each
 * nullable.  grad_seg f32 [b,C,h,w] and grad_vertex f32 [b,ver_dim,h,w] are written through element strides (unit
 * stride along w), each nullable; they may be channel slices of one [b,C+ver_dim,h,w] tensor.  A NULL loss
 * gradient means that loss contributes nothing: its output, when not NULL, is written as zeros, and the inputs only
 * that part needs are not read.  Precision and recall have no gradient.  No allocation, no synchronisation,
 * run-to-run identical, graph capturable.  Workspace: pvnet_seg_vertex_losses_workspace_bytes(b, h, w). */
PVNET_API int pvnet_seg_vertex_losses_backward(const float *seg_pred, const int64_t seg_strides[4],
                                               const void *mask, int mask_elem_size, const int64_t mask_strides[3],
                                               const float *vertex_pred, const int64_t pred_strides[4],
                                               const float *vertex, const int64_t vertex_strides[4],
                                               const float *vertex_weights, const int64_t weight_strides[4],
                                               int b, int h, int w, int C, int ver_dim, double sigma, int normalize,
                                               const float *grad_loss_seg, const float *grad_loss_vertex,
                                               float *grad_seg, const int64_t grad_seg_strides[4],
                                               float *grad_vertex, const int64_t grad_vertex_strides[4],
                                               void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
PVNET_API int pvnet_seg_vertex_losses_keypoints_backward(const float *seg_pred, const int64_t seg_strides[4],
                                                         const void *mask, int mask_elem_size,
                                                         const int64_t mask_strides[3],
                                                         const float *vertex_pred, const int64_t pred_strides[4],
                                                         const void *hcoords, int hcoords_f64, int use_motion,
                                                         const float *vertex_weights, const int64_t weight_strides[4],
                                                         int b, int h, int w, int C, int ver_dim, double sigma,
                                                         int normalize, const float *grad_loss_seg,
                                                         const float *grad_loss_vertex,
                                                         float *grad_seg, const int64_t grad_seg_strides[4],
                                                         float *grad_vertex, const int64_t grad_vertex_strides[4],
                                                         void *workspace, size_t workspace_bytes,
                                                         pvnet_stream_t stream);

/* ------------------------------------------------------------------ dataset tooling (extend.cu, DESIGN.md §11)
 * pvnet_farthest_point_sampling: replaces farthest_point_sampling / farthest_point_sampling_init_center
 *   (lib/utils/extend_utils/src/farthest_point_sampling.cpp:77-105,122-160,166-204, called by extend_utils.py:22-37).
 *   pts f32 [b,pn,3]; idxs int32 [b,sn] receives each cloud's sample indices in selection order.
 *   start int32 [b] (device) gives each cloud's first index, taken modulo pn as the reference takes rand() % pn;
 *   start == NULL is the init_center mode: the first index is the point farthest from the bounding-box centre.
 *   Bit-identical to the reference's binary: the same FP32 sequence, ties keep the lowest index, NaN distances
 *   never win, and a round where no unselected point has min_dist > 0 yields index 0 (even if already selected).
 *   sn == 0 does nothing.  Workspace: pvnet_farthest_point_sampling_workspace_bytes(b, pn) (0 for clouds that fit
 *   on chip; workspace may then be NULL).
 *
 * pvnet_mesh_binary_rasterization: replaces mesh_binary_rasterization (src/mesh_rasterization.cpp:43-71, called by
 *   extend_utils.py:7-20).  triangles f32 [b,tn,3,2] (x, y in pixels); mask uint8 [b,h,w] is overwritten with 0/1,
 *   bit-identical to the reference.  Triangles whose box the reference cannot convert to int (a bound of 2^31 or
 *   more in magnitude) are skipped: they cover no in-range pixel.  h, w >= 2; tn may be 0. */
PVNET_API int pvnet_farthest_point_sampling_workspace_bytes(int b, int pn, size_t *bytes);
PVNET_API int pvnet_farthest_point_sampling(const float *pts, const int32_t *start, int b, int pn, int sn,
                                            int32_t *idxs, void *workspace, size_t workspace_bytes,
                                            pvnet_stream_t stream);
PVNET_API int pvnet_mesh_binary_rasterization(const float *triangles, int b, int tn, int h, int w, uint8_t *mask,
                                              pvnet_stream_t stream);

/* pvnet_render_mesh: depth and flat-shaded RGB of one mesh at b poses, the reference's OpenGL render backend
 *   (lib/utils/opengl_render_backend.py:306-419, flat shading, no texture; DESIGN.md §24).
 *   verts f32 [nv,3]; faces int32 [nf,3] (a face with an index outside [0, nv), a repeated index, a non-finite
 *   vertex or a zero determinant covers nothing); colors f32 [nv,3] or NULL (0.5 grey); poses f32 [b,3,4] (R | t,
 *   object to OpenCV camera); K f32 [3,3], or [b,3,3] when k_per_image != 0 (fx, s, cx, fy, cy are read).
 *   Pixel (r, c) samples the image point (c + 0.5, r + 0.5).  A pixel is covered by the faces whose perspective-correct
 *   barycentrics there are all >= 0 at a camera depth Z with near <= Z <= far (0 < near < far); the one with the
 *   smallest (fp32(Z), face index) wins.  depth f32 [b,h,w] (NULL: not written) receives fp32(Z), 0 where nothing
 *   covers the pixel; rgb uint8 [b,h,w,3] (NULL: not written) receives round(255 * fp32(light_w * colour)),
 *   light_w = min(ambient + max(L . n, 0), 1), and the background bg (host f32 [3], NULL: black) where nothing
 *   covers the pixel.  At least one of depth and rgb.  Workspace: pvnet_render_workspace_bytes(b, h, w), one 64-bit
 *   key per pixel.  The output does not depend on scheduling. */
PVNET_API int pvnet_render_workspace_bytes(int b, int h, int w, size_t *bytes);
PVNET_API int pvnet_render_mesh(const float *verts, const int32_t *faces, const float *colors, int nv, int nf,
                                const float *poses, const float *K, int k_per_image, int b, int h, int w,
                                float near_clip, float far_clip, float ambient, const float *bg, float *depth,
                                uint8_t *rgb, void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

/* pvnet_render_label_map: the label map of several meshes at b images in one depth test, the reference's
 *   OcclusionLineModDB.get_mask_of_all_objects (lib/utils/data_utils.py:788-826; DESIGN.md §25).
 *   M meshes (1 <= M <= 255) packed one after the other: verts f32 [sum nv,3], faces int32 [nf_total,3] with indices
 *   local to their mesh, and mesh_table int32 [M,4] on the device, row m = {vert_off, nv, face_off, nf}, where
 *   face_off is the sum of the earlier meshes' nf and nf_total the sum of all.  labels uint8 [M] (host), each 1..255.
 *   poses f32 [b,M,3,4] (R | t of slot m in image i); present uint8 [b,M] (0: the slot is absent from the image) or
 *   NULL (all present); K f32 [3,3], or [b,3,3] when k_per_image != 0.  Coverage, clip planes and pixel convention
 *   are pvnet_render_mesh's.  A slot's depth at a pixel is pvnet_render_mesh's depth of that mesh alone divided by
 *   depth_divisor in one IEEE fp32 division (depth_divisor > 0 and finite, near / depth_divisor above 0).
 *   label uint8 [b,h,w] receives the label of the slot with the smallest depth strictly below max_depth (> 0, +inf
 *   allowed), ties to the lower slot, and 0 where there is none; depth f32 [b,h,w] (NULL: not written) receives that
 *   depth, max_depth where the label is 0.  Workspace: pvnet_render_workspace_bytes(b, h, w).  The output does not
 *   depend on scheduling. */
PVNET_API int pvnet_render_label_map(const float *verts, const int32_t *faces, const int32_t *mesh_table,
                                     const uint8_t *labels, int M, int nf_total, const float *poses,
                                     const uint8_t *present, const float *K, int k_per_image, int b, int h, int w,
                                     float near_clip, float far_clip, float depth_divisor, float max_depth,
                                     uint8_t *label, float *depth, void *workspace, size_t workspace_bytes,
                                     pvnet_stream_t stream);

/* The vanishing-point pair of the reference extension (ransac_voting.cpp:61-99 ->
 * ransac_voting_kernel.cu:170-260, :263-351; used by ransac_voting_vanish_point_layer,
 * ransac_voting_gpu.py:408-501): hypotheses are homogeneous points hypo [hn,vn,3]; the vote sets
 * inliers [hn,vn,tn] u8 (caller zero-fills; may be NULL) and/or writes the row sums counts [hn,vn]. */
PVNET_API int pvnet_generate_hypothesis_vanishing_point(const float *direct, const float *coords, const int32_t *idxs,
                                                        float *hypo, int tn, int vn, int hn, pvnet_stream_t stream);
PVNET_API int pvnet_voting_for_hypothesis_vanishing_point(const float *direct, const float *coords, const float *hypo,
                                                          uint8_t *inliers, int32_t *counts, int tn, int vn, int hn,
                                                          float inlier_thresh, pvnet_stream_t stream);

/* Number of kernels this library has launched on the calling thread since the last
 * reset (bench.py's "gpu_launches"). */
PVNET_API long long pvnet_launch_count(void);
PVNET_API void pvnet_launch_count_reset(void);

/* -------------------------------------------------------------------- backbone */

/* One NHWC convolution on the Hopper tensor cores (wgmma, TF32 inputs, fp32 accumulate), the
 * building block of Resnet18_8s (lib/networks/resnet.py:28-35,54-70; model_repository.py:22-58):
 *
 *   out[n,y,x,out_co+co] = act( bias[co] + res[n,y,x,res_co+co]
 *                               + sum_{kh,kw,ci} w[co][kh][kw][ci] * in[n, y*stride+(kh-c)*dil, x*stride+(kw-c)*dil, in_co+ci] )
 *
 *   in        NHWC buffer [b,H,W,in_cs]; the conv reads channels [in_co, in_co+Cin)
 *   w_packed  [Cout][ksize*ksize][cin_pad] fp32 (BatchNorm already folded in; cin_pad = Cin rounded up
 *             to a multiple of 32, zero padded; 16 stays 16), bias [Cout]
 *   res       NHWC [b,H/stride,W/stride,res_cs] read at res_co, or NULL
 *   out       NHWC [b,H/stride,W/stride,out_cs] written at channel offset out_co
 *             (writing into a slice of a wider buffer replaces torch.cat)
 *   ksize 1|3, stride 1|2 (2 needs even H,W, dilation 1), padding = dilation*(ksize-1)/2
 *   act 0 none, 1 ReLU, 2 LeakyReLU(0.1); round_out != 0 rounds the stored values to TF32
 *   Cin multiple of 4, Cout multiple of 32; strides/offsets multiples of 4 floats.
 */
PVNET_API int pvnet_conv2d_nhwc(const float *in, int in_cs, int in_co, int Cin,
                                const float *w_packed, const float *bias,
                                const float *res, int res_cs, int res_co,
                                float *out, int out_cs, int out_co, int Cout,
                                int b, int H, int W, int ksize, int stride, int dilation,
                                int act, int round_out, pvnet_stream_t stream);

/* Weight gradient of a stride-1 NHWC convolution on the Hopper tensor cores (wgmma, TF32 operands, fp32
 * accumulate): the dW half of the backward that autograd runs through the convolutions of
 * lib/networks/resnet.py:28-35,54-70 and model_repository.py:22-58 during training.
 *
 *   dw[co][ci][kh][kw] = sum_{n,y,x} dout[n,y,x,dout_co+co] * in[n, y+(kh-c)*dil, x+(kw-c)*dil, in_co+ci]
 *                        c = (ksize-1)/2, out-of-image `in` reads are zero (padding dilation*(ksize-1)/2)
 *
 *   in        NHWC [b,H,W,in_cs], the forward's input, read at channels [in_co, in_co+Cin)
 *   dout      NHWC [b,H,W,dout_cs], the gradient of the forward's output (same grid: stride 1), read at
 *             [dout_co, dout_co+Cout).  A stride-2 layer's gradient is first spread onto the input's grid
 *             with pvnet_zero_insert2x_nhwc; its dW is then this stride-1 form with the same padding.
 *   dw        [Cout][Cin][ksize][ksize] fp32 contiguous (torch's Conv2d.weight layout), overwritten
 *   ksize 1|3, dilation >= 1; Cin, Cout, strides and offsets multiples of 4 floats; in/dout 16-byte aligned.
 * Both operands enter the MMA as TF32 (the low 13 mantissa bits are ignored).  The pixels are split over CTAs
 * whose partial tiles go to `workspace` (pvnet_conv2d_nhwc_wgrad_workspace_bytes, which depends on the shape
 * and on the current device) and are summed in a fixed order: the result is identical run to run.  Allocates
 * nothing, launches two kernels on `stream`. */
PVNET_API int pvnet_conv2d_nhwc_wgrad_workspace_bytes(int Cin, int Cout, int b, int H, int W, int ksize,
                                                      size_t *bytes);
PVNET_API int pvnet_conv2d_nhwc_wgrad(const float *in, int in_cs, int in_co, int Cin,
                                      const float *dout, int dout_cs, int dout_co, int Cout, float *dw,
                                      int b, int H, int W, int ksize, int dilation,
                                      void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
/* Zero insertion for the stride-2 convolutions' backward (layer2.0.conv1, layer2.0.downsample.0):
 *   out[n,y,x,out_co+c] = (y, x even) ? in[n,y/2,x/2,in_co+c] : 0      on the full H x W grid
 * in NHWC [b,H/2,W/2,in_cs], out NHWC [b,H,W,out_cs]; H, W even; C, strides and offsets multiples of 4 floats.
 * With it dX = pvnet_conv2d_nhwc(out, flipped transposed weights, stride 1, padding (k-1)/2) and
 * dW = pvnet_conv2d_nhwc_wgrad(X, out). */
PVNET_API int pvnet_zero_insert2x_nhwc(const float *in, int in_cs, int in_co, int C, float *out, int out_cs,
                                       int out_co, int b, int H, int W, pvnet_stream_t stream);

/* Bilinear x2 upsampling with align_corners=True (nn.UpsamplingBilinear2d(scale_factor=2),
 * lib/networks/model_repository.py:35,43,51) for training, forward and backward.
 *
 * pvnet_upsample2x_nhwc: in NHWC [b,h,w,C] dense -> out NHWC [b,2h,2w,out_cs] at channels [out_co, out_co+C), the
 *   other channels untouched.  Exact fp32 (not rounded to TF32 like the eval path's upsampling): bit for bit what
 *   torch's CUDA F.interpolate(scale_factor=2, mode="bilinear", align_corners=True) returns for a channels_last input
 *   (shown for C >= 16; the decoder's C is 32 to 128).
 * pvnet_upsample2x_backward_nhwc: dout NHWC [b,2h,2w,dout_cs], read at channels [dout_co, dout_co+C) -> din NHWC
 *   [b,h,w,C] dense, overwritten with dX = U^T dout.  Each element is the sum of exactly the terms torch's CUDA
 *   backward adds to it with atomics -- (hl * wl) * g, two rounded fp32 products -- taken in a fixed order (output
 *   pixels ascending, then torch's term order within one output pixel): no atomics, identical run to run, and a
 *   result torch's own backward can return.
 * Both: C, strides and offsets multiples of 4 floats; pointers 16-byte aligned; b*4*h*w*cs and b*h*w*C below 2^32
 * elements.  Allocate nothing, launch one kernel on `stream`; bad arguments return PVNET_E_INVALID. */
PVNET_API int pvnet_upsample2x_nhwc(const float *in, int C, float *out, int out_cs, int out_co, int b, int h, int w,
                                    pvnet_stream_t stream);
PVNET_API int pvnet_upsample2x_backward_nhwc(const float *dout, int dout_cs, int dout_co, int C, float *din, int b,
                                             int h, int w, pvnet_stream_t stream);

/* Train-mode BatchNorm2d fused with its activation and the residual add of a BasicBlock (lib/networks/resnet.py
 * BasicBlock.forward, model_repository.py's Conv2d -> BatchNorm2d -> ReLU / LeakyReLU(0.1) sequences), forward and
 * backward, on dense NHWC fp32 tensors of npix = b*H*W pixels and C channels (C a multiple of 4, up to 1024 for
 * form 0 and up to 2048 for forms 1 and 2, the Bottleneck tails of Resnet50_8s's layer4;
 * pointers 16-byte aligned; element offsets are 64-bit).
 *
 *   form 0  y = act(bn(x))               act 0 none, 1 ReLU, 2 LeakyReLU(0.1)
 *   form 1  y = relu(bn(x) + z)          identity block tail: z is the skip
 *   form 2  y = relu(bn(x) + bn_z(z))    downsample block tail: z is the downsample convolution's output
 *
 * bn(v) = fma(v, scale, shift) rounded to fp32, then the add, then the activation (the module graph's rounding).
 * With batch_stats, mean and biased variance are fp64 over a fixed partition of the pixels (256-pixel partials
 * merged in a fixed order: identical run to run, whatever the device); scale = fp32(gamma*invstd) and
 * shift = fp32(beta - mean*scale), invstd = 1/sqrt(var + eps); running_mean/running_var (when non-NULL) become
 * (1-f)*r + f*stat in fp32, with the unbiased variance var*N/(N-1).  Without batch_stats (a module in eval mode)
 * the running statistics normalise and are left alone.
 *
 * The backward recomputes each element's pre-activation value from the same bits, g = dy*act'(pre) (ReLU: 0 where
 * pre <= 0; LeakyReLU: dy*0.1f where pre <= 0), and writes dx = A*g + B*x + Cc with per-channel fp32 coefficients
 * rounded once from fp64 sums of g and g*(x - mean) (B = Cc = 0 without batch_stats); dweight = invstd*sum g*(x-mean),
 * dbias = sum g (NULL: not written).  Form 1 writes dz = g, form 2 dz = bn_z's data gradient (and dweight_z, dbias_z).
 * The backward reads the `saved` and `coef` the forward wrote.  Allocate nothing; launch on `stream`. */
typedef struct pvnet_batchnorm {
    const float *weight;   /* [C] gamma, or NULL for 1 */
    const float *bias;     /* [C] beta, or NULL for 0 */
    float *running_mean;   /* [C] or NULL */
    float *running_var;    /* [C] or NULL */
    int batch_stats;       /* 1: normalise with the batch's statistics; 0: with running_mean/running_var */
    double factor;         /* running-stat factor f: momentum, or 1/num_batches_tracked when momentum is None */
    double eps;
    double *saved;         /* [3][C] fp64, written by the forward: mean, biased variance, invstd */
    float *coef;           /* [2][C] fp32, written by the forward: scale, shift */
} pvnet_batchnorm_t;
/* Workspace of one forward or backward call of `form` (fp64 partial sums and the backward's coefficients). */
PVNET_API int pvnet_batchnorm_workspace_bytes(int form, int C, long long npix, size_t *bytes);
PVNET_API int pvnet_batchnorm_act_forward(int form, int act, const float *x, const float *z, long long npix, int C,
                                          const pvnet_batchnorm_t *bn, const pvnet_batchnorm_t *bn_z, float *y,
                                          void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
PVNET_API int pvnet_batchnorm_act_backward(int form, int act, const float *dy, const float *x, const float *z,
                                           long long npix, int C, const pvnet_batchnorm_t *bn,
                                           const pvnet_batchnorm_t *bn_z, float *dx, float *dz, float *dweight,
                                           float *dbias, float *dweight_z, float *dbias_z, void *workspace,
                                           size_t workspace_bytes, pvnet_stream_t stream);

/* The stem, max-pool and head of Resnet18_8s's training step (lib/networks/resnet.py:201-204,
 * model_repository.py:57), forward and backward.  Each launches on `stream` and allocates nothing; bad arguments
 * return PVNET_E_INVALID with a message.
 *
 * pvnet_stem_s2d_nhwc: conv1 (3 -> 64, 7x7, stride 2, pad 3) of a training batch as the eval path computes it, the
 *   image in either form pvnet_backbone_forward / pvnet_backbone_forward_u8 take:
 *   - image_is_u8 = 0: image f32 NCHW [b,3,H,W] (8-byte aligned); mean3 and std3 must be NULL.
 *   - image_is_u8 = 1: image uint8 [b,H,W,3] contiguous (2-byte aligned), normalised on the device as torchvision's
 *     ToTensor + Normalize on the CPU compute it: v = (float(u) / 255 - mean3[c]) / std3[c], three correctly rounded
 *     fp32 ops (mean3 / std3: 3 host floats each, finite, std nonzero).  Every output below is the float form's for
 *     the image v.
 *   H, W even.  s2d [b,H/2,W/2,16] is written with the 2x2 space-to-depth image (channel (py*2+px)*3+c, 4 zero
 *   channels, rounded to TF32) and out NHWC [b,H/2,W/2,64] = the 4x4 stride-1 tensor-core convolution of s2d with
 *   w_s2d (packed [64][4][4][16] as backbone slot 0, TF32) plus bias [64], fp32, no activation.  s2d is what
 *   pvnet_stem_s2d_wgrad reads.  In the same pass the caller's channels_last buffer img NHWC [b,H,W,img_cs] gets the
 *   fp32 image unrounded in channels [img_co, img_co+3) and zeros in [img_co+3, img_co+8) (img_co, img_cs multiples
 *   of 4, img_co+8 <= img_cs): convraw.0's image and pad channels; its other channels are not touched.
 * pvnet_stem_s2d_wgrad: dw [64][3][7][7] (torch's layout, overwritten) = the weight gradient of that convolution for
 *   dout NHWC [b,H/2,W/2,64] dense: the 4x4 weight gradient on s2d (TF32 operands, dout truncated by the tensor
 *   cores, fp32 accumulation, pixel splits added in a fixed order: identical run to run), folded back onto the
 *   147 weights of the 7x7 kernel.  The workspace size depends on the current device's SM count.
 * pvnet_maxpool3x3s2_nhwc: nn.MaxPool2d(3, stride 2, padding 1) of in NHWC [b,H,W,C] dense (C a multiple of 4, H and
 *   W even) -> out NHWC [b,H/2,W/2,C] and code uint8 [b,H/2,W/2,C], the argmax's window position dy*3+dx (dy, dx in
 *   0..2 from the window origin (2oy-1, 2ox-1)).  torch's rule: the window scanned row-major from -inf, an element
 *   wins when v > max or v is NaN; with no winner the first in-image element is the argmax.
 * pvnet_maxpool3x3s2_backward_nhwc: din NHWC [b,H,W,C] (every element written) = each input's sum of the dout of
 *   the windows whose code points at it, outputs ascending from 0.0f (ATen's order), no atomics.
 * pvnet_head1x1_nchw: out NCHW [b,Cout,H,W] contiguous = bias[o] + sum_c w[o][c]*y[c], one fp32 fmaf chain per
 *   output (c ascending from bias[o]), for y NHWC [b,H,W,Cin] dense (Cin a multiple of 32) and w [Cout][Cin].
 * pvnet_head1x1_backward: for dout NCHW [b,Cout,H,W] contiguous: dy NHWC [b,H,W,Cin] = sum_o w[o][c]*dout[o] (an fmaf
 *   chain, o ascending from 0); dw [Cout][Cin] = sum_p dout[p][o]*y[p][c] and db [Cout] = sum_p dout[p][o] in fp64
 *   over a fixed partition of the pixels, merged in a fixed order and rounded once to fp32.  Any of dy, dw, db may
 *   be NULL (not computed); the workspace is needed only for dw / db.
 * All offsets are 64-bit; pointers 16-byte aligned unless stated. */
PVNET_API int pvnet_stem_s2d_nhwc(const void *image, int image_is_u8, const float *mean3, const float *std3,
                                  const float *w_s2d, const float *bias, float *s2d, float *out, float *img, int img_cs,
                                  int img_co, int b, int H, int W, pvnet_stream_t stream);
/* pvnet_stem_s2d_half_nhwc: pvnet_stem_s2d_nhwc with img at half resolution, NHWC [b,H/2,W/2,img_cs]: channels
 *   [img_co, img_co+3) get x_ds = F.interpolate(image, scale_factor=0.5, mode='bilinear') unrounded, bit for bit
 *   torch's CUDA result on the NCHW float image ((0.5a + 0.5b)*0.5 + (0.5c + 0.5d)*0.5 over each 2x2 block, rows
 *   first), and [img_co+3, img_co+8) zeros: conv2s.0's image and pad channels in Resnet50_8s_2o.  s2d and out are
 *   those of pvnet_stem_s2d_nhwc. */
PVNET_API int pvnet_stem_s2d_half_nhwc(const void *image, int image_is_u8, const float *mean3, const float *std3,
                                       const float *w_s2d, const float *bias, float *s2d, float *out, float *img,
                                       int img_cs, int img_co, int b, int H, int W, pvnet_stream_t stream);
PVNET_API int pvnet_stem_s2d_wgrad_workspace_bytes(int b, int H, int W, size_t *bytes);
PVNET_API int pvnet_stem_s2d_wgrad(const float *s2d, const float *dout, float *dw, int b, int H, int W,
                                   void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
PVNET_API int pvnet_maxpool3x3s2_nhwc(const float *in, float *out, uint8_t *code, int b, int H, int W, int C,
                                      pvnet_stream_t stream);
PVNET_API int pvnet_maxpool3x3s2_backward_nhwc(const float *dout, const uint8_t *code, float *din, int b, int H, int W,
                                               int C, pvnet_stream_t stream);
PVNET_API int pvnet_head1x1_nchw(const float *y, const float *w, const float *bias, float *out, int b, int H, int W,
                                 int Cin, int Cout, pvnet_stream_t stream);
PVNET_API int pvnet_head1x1_backward_workspace_bytes(int b, int H, int W, int Cin, int Cout, size_t *bytes);
PVNET_API int pvnet_head1x1_backward(const float *dout, const float *y, const float *w, float *dy, float *dw,
                                     float *db, int b, int H, int W, int Cin, int Cout, void *workspace,
                                     size_t workspace_bytes, pvnet_stream_t stream);
/* The detectors' score head (Conv2d(C, 1, 3, 1, 1) with bias; DESIGN.md §22), x NHWC [b,H,W,C] dense (C a multiple of
 * 32, at most 512), w [9][C] (tap ky*3+kx), bias [1]:
 * pvnet_head3x3_nchw: out [b,1,H,W] = one fp32 fmaf chain per output from bias[0]: 32-channel chunks ascending, within
 *   a chunk the taps ascending, within a tap the channels ascending; taps outside the image are skipped.
 * pvnet_head3x3_backward: for dout [b,1,H,W] contiguous: dx NHWC [b,H,W,C] = sum_t w[t][c]*dout[y+1-ky, x+1-kx] (an
 *   fmaf chain, t ascending from 0, taps outside the image skipped); dw [9][C] = sum_p dout[p]*x[p+(ky-1,kx-1)][c] and
 *   db [1] = sum_p dout[p] in fp64 over a fixed partition of the pixels, merged in a fixed order and rounded once to
 *   fp32.  Any of dx, dw, db may be NULL (not computed); the workspace is needed only for dw / db. */
PVNET_API int pvnet_head3x3_nchw(const float *x, const float *w, const float *bias, float *out, int b, int H, int W,
                                 int C, pvnet_stream_t stream);
PVNET_API int pvnet_head3x3_backward_workspace_bytes(int b, int H, int W, int C, size_t *bytes);
PVNET_API int pvnet_head3x3_backward(const float *dout, const float *x, const float *w, float *dx, float *dw,
                                     float *db, int b, int H, int W, int C, void *workspace, size_t workspace_bytes,
                                     pvnet_stream_t stream);

/* The optimizer step of tools/train_linemod.py:260 (optim.Adam(net.parameters(), lr=...)): one Adam step over a table
 * of fp32 tensors, in place, one pass (each element reads p, g, m, v once and writes p, m, v once).
 *
 * One table entry, all DEVICE pointers to `numel` dense fp32 elements in one common order, 4-byte aligned (16-byte
 * aligned entries use float4 accesses, the others scalar ones, with the same bits):
 *   param       the parameter, updated in place
 *   grad        its gradient, read only
 *   exp_avg     the first-moment state m, updated in place
 *   exp_avg_sq  the second-moment state v, updated in place
 *   numel       element count; an entry with numel == 0 is skipped and its pointers are not looked at */
typedef struct pvnet_adam_tensor {
    void *param;
    const void *grad;
    void *exp_avg;
    void *exp_avg_sq;
    int64_t numel;
} pvnet_adam_tensor_t;
/* pvnet_adam_step:
 *   tensors       HOST array of n_tensors entries (n_tensors == 0 is a no-op); read before the call returns.  The table
 *                 travels to the device in the kernel's parameter space, pvnet_adam_chunk_tensors() non-empty entries
 *                 per launch: no copy, no allocation, no synchronisation, launches on `stream` only.
 *   lr, beta1, beta2, eps, weight_decay   torch.optim.Adam's hyper-parameters as doubles: lr, eps and weight_decay
 *                 finite and >= 0, the betas in [0, 1).  weight_decay is the L2 form (added to the gradient).
 *   step          the step count these tensors reach with this call (1 on the first step), >= 1; one value for the
 *                 whole table -- tensors at different counts go into different calls.
 * What is computed is torch.optim.Adam(foreach=False)'s sequence with amsgrad, maximize, capturable and differentiable
 * off, per element in fp32, every operation rounded to nearest, the scalars prepared on the host in double and
 * converted to fp32 once (DESIGN.md §19 states it operation by operation; oracle/adam_oracle.py restates it):
 *   g += p*weight_decay (one FMA; skipped when weight_decay == 0);  m = fma(w1, g - m, m), w1 = float(1 - beta1)
 *   (for w1 >= 0.5: m = fma(-(g - m), 1 - w1, g));  v = fma(float(1 - beta2), g*g, v*float(beta2));
 *   denom = sqrt(v) * float(1.0 / sqrt(1 - beta2^step)) + float(eps);
 *   p = fma(float(-lr / (1 - beta1^step)), m / denom, p).
 * Bad arguments return PVNET_E_INVALID with a message before anything is launched. */
PVNET_API int pvnet_adam_step(const pvnet_adam_tensor_t *tensors, int n_tensors, double lr, double beta1, double beta2,
                              double eps, double weight_decay, int64_t step, pvnet_stream_t stream);
/* Table entries one launch of pvnet_adam_step carries: a table of n non-empty entries takes ceil(n / this) launches. */
PVNET_API int pvnet_adam_chunk_tensors(void);

/* Test hook: which convolution kernel pvnet_conv2d_nhwc uses for layers both can run (the backbone
 * always plans automatically).  0 = automatic (persistent weights-resident column kernel for 3x3
 * stride-1 layers with Cout <= 64 whose weights fit in shared memory, per-tap kernel otherwise),
 * 1 = per-tap kernel only, 2 = column kernel (error if the layer is not eligible). */
PVNET_API int pvnet_conv_set_mode(int mode);

/* Resnet18_8s.forward (lib/networks/model_repository.py:64-80), eval mode, whole batch (Resnet34_8s / Resnet50_8s:
 * pvnet_backbone_create_trunk below; the same calls with the handle's own slots and stages).
 *
 * The handle is a host-side table of per-convolution weight pointers plus cached tensor
 * maps; it owns no device memory.  Weights are DEVICE pointers owned by the caller and
 * must stay valid while the handle is used:
 *   slot 0               stem conv1+bn1, the 7x7 stride-2 conv written as a 4x4 stride-1 conv over
 *                        the 2x2 space-to-depth image, packed [64][4][4][16] (tap (ty,tx), channel
 *                        (py*2+px)*3+c holds w[c][2ty+py-1][2tx+px-1]; rest 0), bias [64]
 *   slots 1..24          the 3x3 / 1x1 convs in execution order (layer1.0.conv1, layer1.0.conv2,
 *                        layer1.1.conv1, layer1.1.conv2, layer2.0.conv1, layer2.0.downsample,
 *                        layer2.0.conv2, layer2.1.conv1, layer2.1.conv2, layer3.* and layer4.* in the
 *                        same pattern, fc.0, conv8s.0, conv4s.0, conv2s.0, convraw.0), each packed
 *                        [Cout][kh*kw][cin_pad] with its BatchNorm folded in, bias [Cout].  convraw.0 reads
 *                        s2dim+8 buffer channels (s2dim upsampled, 3 image, 5 zeros); cin_pad rounds up to 32.
 *   slot 25              convraw.3 (1x1, with bias): [seg_dim+ver_dim][32], bias [seg_dim+ver_dim]
 * pvnet_backbone_forward:
 *   image_nchw  f32 [b,3,h,w] (h,w multiples of 8)
 *   out_nchw    f32 [b,seg_dim+ver_dim,h,w]: seg logits are channels [0,seg_dim), the vertex
 *               field the rest (model_repository.py:77-78)
 *   mask_out    optional [b,h,w] argmax over the seg channels (first maximum), int64
 *               (mask_elem_size 8, what torch.argmax returns) or uint8 (1); NULL to skip
 */
typedef struct pvnet_backbone pvnet_backbone_t;
PVNET_API int pvnet_backbone_create(int ver_dim, int seg_dim, int fcdim, int s8dim, int s4dim, int s2dim,
                                    int raw_dim, pvnet_backbone_t **out);
/* The Resnet18_8s plan's conv-slot count (26); a handle's own: pvnet_backbone_handle_num_convs. */
PVNET_API int pvnet_backbone_num_convs(void);

/* A backbone over any trunk of lib/networks/resnet.py's ResNet(block, blocks, output_stride=8) under the
 * Resnet*_8s decoder (model_repository.py): block_kind PVNET_BLOCK_BASIC (resnet18 / resnet34) or
 * PVNET_BLOCK_BOTTLENECK (resnet50, expansion 4), blocks[4] the blocks per stage (each in [1,64]), raw_dim 32 or
 * 64, the other widths as pvnet_backbone_create takes them.  The conv slots follow the same pattern: slot 0 the
 * stem; then per block conv1, (conv2,) the downsample (first block of a stage that has one), and the conv whose
 * epilogue adds the skip (BasicBlock conv2, Bottleneck conv3); then fc.0, conv8s.0, conv4s.0, conv2s.0, convraw.0
 * and convraw.3 as [seg_dim+ver_dim][raw_dim].  The 2-2-2-2 BasicBlock trunk gives pvnet_backbone_create's plan. */
enum { PVNET_BLOCK_BASIC = 0, PVNET_BLOCK_BOTTLENECK = 1 };
PVNET_API int pvnet_backbone_create_trunk(int block_kind, const int *blocks, int ver_dim, int seg_dim, int fcdim,
                                          int s8dim, int s4dim, int s2dim, int raw_dim, pvnet_backbone_t **out);
/* Resnet50_8s_2o's decoder (model_repository.py:158-224) over the same trunks: conv8s, conv4s, then conv2s.0 over
 * cat[up(conv4s), x2s, x_ds] (x_ds = F.interpolate(image, scale_factor=0.5, mode='bilinear')) and the 1x1 head
 * conv2s.3, at half resolution.  The conv slots are the trunk's, then conv8s.0, conv4s.0, conv2s.0 (packed for
 * s4dim+64+8 input channels: s4dim upsampled, 64 x2s, 3 x_ds, 5 zeros) and conv2s.3 as [seg_dim+ver_dim][s2dim].
 * s2dim must be 32 or 64.  The forward calls then write out [b,seg_dim+ver_dim,h/2,w/2] (or [b,h/2,w/2,C]) and the
 * mask [b,h/2,w/2]; everything else is as for the full-resolution decoder. */
PVNET_API int pvnet_backbone_create_trunk_2o(int block_kind, const int *blocks, int ver_dim, int seg_dim, int fcdim,
                                             int s8dim, int s4dim, int s2dim, pvnet_backbone_t **out);
/* Resnet18_8s_detector / Resnet18_8s_detector_v2 (model_repository.py:302-331): no decoder.  last_stage 4: the trunk,
 * then its fc = Conv2d(512, 1, 3, 1, 1) with bias on layer4's output; last_stage 2: the stem, layer1 and layer2, then
 * out_conv = Conv2d(128, 1, 3, 1, 1) on layer2's output.  The conv slots are the trunk's up to that stage (no fc.0),
 * then the score head, packed fp32 [9][C] (tap ky*3+kx, then channel; not rounded) with bias [1]; C, the stage's
 * output channels, must be at most 512.  The forward calls write out [b,1,h/8,w/8] through pvnet_head3x3_nchw's
 * kernel; mask_out must be NULL and the output layout setting has no effect (one channel). */
PVNET_API int pvnet_backbone_create_detector(int block_kind, const int *blocks, int last_stage,
                                             pvnet_backbone_t **out);
/* The factor between the input and the output grid: 1, 2 for a pvnet_backbone_create_trunk_2o handle, 8 for a
 * pvnet_backbone_create_detector handle; -1 for a null handle. */
PVNET_API int pvnet_backbone_output_scale(const pvnet_backbone_t *m);
PVNET_API int pvnet_backbone_handle_num_convs(const pvnet_backbone_t *m);   /* -1 for a null handle */
PVNET_API void pvnet_backbone_destroy(pvnet_backbone_t *m);
PVNET_API int pvnet_backbone_set_conv(pvnet_backbone_t *m, int slot, const float *w_packed, const float *bias);
/* Output layout of the following forward calls on this handle: 0 (default) = out [b,C,h,w], the
 * reference's NCHW tensor whose channel slices are seg_pred / ver_pred (model_repository.py:77-78);
 * 1 = pixel-major out [b,h,w,C]: the same values as one contiguous record per pixel, which is the
 * vertex layout [b,h,w,K,2] the voting layer's gather reads without sector waste (the contiguous
 * form of the permuted view of tools/demo.py:48-50). */
PVNET_API int pvnet_backbone_set_output_layout(pvnet_backbone_t *m, int pixel_major);
PVNET_API int pvnet_backbone_workspace_bytes(const pvnet_backbone_t *m, int b, int h, int w, size_t *bytes);
PVNET_API int pvnet_backbone_forward(pvnet_backbone_t *m, const float *image_nchw, int b, int h, int w,
                                     float *out_nchw, void *mask_out, int mask_elem_size,
                                     void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
/* Same forward pass from a RAW image batch: image_hwc uint8 [b,h,w,3] (what an image decoder yields),
 * normalised on the device inside the packing kernel with torchvision's ToTensor + Normalize
 * arithmetic, (float(v)/255 - mean[c]) / std[c] in fp32 (tools/demo.py:89-95,
 * lib/datasets/linemod_dataset.py:191-195): bit-identical to pvnet_backbone_forward on the
 * torch-normalised float tensor, a quarter of the input bytes.  mean/std are HOST arrays. */
PVNET_API int pvnet_backbone_forward_u8(pvnet_backbone_t *m, const uint8_t *image_hwc, const float mean[3],
                                        const float std[3], int b, int h, int w,
                                        float *out_nchw, void *mask_out, int mask_elem_size,
                                        void *workspace, size_t workspace_bytes, pvnet_stream_t stream);
/* JPEG bytes -> the uint8 [b,h,w,3] RGB batch pvnet_backbone_forward_u8 takes, decoded on the device by
 * NVIDIA's nvJPEG (library code; dlopen'ed on first use -- pvnet_jpeg_available() says whether it was found).
 * Replaces the host-side `Image.open` of lib/datasets/linemod_dataset.py:180-195 / tools/demo.py:89.
 * jpeg_data / lengths: HOST arrays of b host pointers / sizes; every image must be h x w.  The decoder object
 * owns nvJPEG's internal buffers (the one place this library lets a dependency allocate).  Different decoder
 * than the reference's libjpeg: +-1 level from the IDCT, more at colour edges of chroma-subsampled files. */
typedef struct pvnet_jpeg_decoder pvnet_jpeg_decoder_t;
PVNET_API int pvnet_jpeg_available(void);
PVNET_API int pvnet_jpeg_decoder_create(pvnet_jpeg_decoder_t **out);
PVNET_API void pvnet_jpeg_decoder_destroy(pvnet_jpeg_decoder_t *d);
PVNET_API int pvnet_jpeg_decode_batch(pvnet_jpeg_decoder_t *d, const uint8_t *const *jpeg_data, const size_t *lengths,
                                      int b, int h, int w, uint8_t *out_hwc, pvnet_stream_t stream);

/* The forward pass is an ordered list of single-kernel stages; these run/describe one of
 * them with the same arguments (per-layer timing in bench.py, layer-wise parity tests).
 * pvnet_backbone_num_stages / _stage_name describe the Resnet18_8s plan, the _handle_ forms the handle's own
 * (its stage indices are what pvnet_backbone_run_stage takes; the name is valid while the handle lives). */
PVNET_API int pvnet_backbone_num_stages(void);
PVNET_API const char *pvnet_backbone_stage_name(int stage);
PVNET_API int pvnet_backbone_handle_num_stages(const pvnet_backbone_t *m);  /* -1 for a null handle */
PVNET_API const char *pvnet_backbone_handle_stage_name(const pvnet_backbone_t *m, int stage);
PVNET_API int pvnet_backbone_run_stage(pvnet_backbone_t *m, int stage, const float *image_nchw, int b, int h, int w,
                                       float *out_nchw, void *mask_out, int mask_elem_size,
                                       void *workspace, size_t workspace_bytes, pvnet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PVNET_B200_H_ */
