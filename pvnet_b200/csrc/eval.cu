// eval.cu -- pose evaluation on the device: the nearest-point search and the batched pose metrics that the
// reference computes per image on the host after the PnP (tools/train_linemod.py:177-229 `val()`).
//
// Reference:
//   lib/utils/extend_utils/src/nearest_neighborhood.cu:123-163   findNearestPointIdxLauncher (one thread per query,
//                                                                global loads, a malloc/copy/free round trip per call)
//   lib/utils/evaluation_utils.py:75-89                           projection_2d / projection_2d_sym
//   lib/utils/evaluation_utils.py:91-130                          add_metric / add_metric_sym (ADD, ADD-S)
//   lib/utils/evaluation_utils.py:132-141                         cm_degree_5_metric
//
// Nearest-point search (DESIGN.md §2 "FP sequence"): the reference kernel compiles (nvcc 12.9, sm_90a) to
//     dx = x1 - x2, dy = y1 - y2, dz = z1 - z2;  d = fma(dz, dz, fma(dx, dx, dy * dy))      (2-D: fma(dx, dx, dy * dy))
//     best = (FLT_MAX, 0); replace when d < best (FSETP.GEU: a NaN never wins, ties keep the lowest index)
// and the code below spells that sequence with __fsub_rn/__fmul_rn/__fmaf_rn, so the indices are bit-identical.
// The loop is FP32-issue-bound (about 8 instructions per pair), so reference points are staged in shared memory in
// tiles, every thread holds NN_Q queries in registers (one broadcast read serves NN_Q tests), all images run in one
// launch (grid.y) and an image's queries are split over CTAs (grid.x).
//
// Pose metrics: one fixed fp64 operation order for the transform R X + t and the projection (K p)[:2] / (K p)[2]
// (explicit __dmul_rn/__dadd_rn/__ddiv_rn, no contraction), restated in the same order by oracle/eval_oracle.py, so
// that the fp32 roundings ADD-S searches on, and therefore its indices, are equal on both sides.  The transformed
// clouds are never stored: each reference tile is transformed as it is loaded into shared memory and the winner's fp64
// coordinates are recomputed from model[idx].  Per-CTA partial sums go to the caller's workspace and one thread per
// image adds them in chunk order, so the result does not depend on scheduling (no fp64 atomics).
#include "common.cuh"

#include <cfloat>
#include <type_traits>

namespace {

constexpr int NN_THREADS = 128;
constexpr int NN_Q = 4;                          // queries per thread
constexpr int NN_TILE = 512;                     // reference points per shared-memory tile
constexpr int NN_QPB = NN_THREADS * NN_Q;        // queries per CTA

constexpr int PM_THREADS = 128;
constexpr int PM_Q = 4;
constexpr int PM_TILE = 512;
constexpr int PM_QPB = PM_THREADS * PM_Q;

template <int DIM>
using NnVec = typename std::conditional<DIM == 3, float4, float2>::type;

__device__ __forceinline__ float nn_dist(float4 r, float qx, float qy, float qz)
{
    const float dx = __fsub_rn(r.x, qx), dy = __fsub_rn(r.y, qy), dz = __fsub_rn(r.z, qz);
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}
__device__ __forceinline__ float nn_dist(float2 r, float qx, float qy, float)
{
    const float dx = __fsub_rn(r.x, qx), dy = __fsub_rn(r.y, qy);
    return __fmaf_rn(dx, dx, __fmul_rn(dy, dy));
}

// Scan one shared tile s[0..n) (global indices base..base+n) for Q queries, in index order.
template <int Q, typename V>
__device__ __forceinline__ void nn_scan_tile(const V *s, int n, int base, const float (&qx)[Q], const float (&qy)[Q],
                                             const float (&qz)[Q], float (&best)[Q], int (&bi)[Q])
{
#pragma unroll 4
    for (int k = 0; k < n; ++k) {
        const V p = s[k];
#pragma unroll
        for (int j = 0; j < Q; ++j) {
            const float d = nn_dist(p, qx[j], qy[j], qz[j]);
            if (d < best[j]) {
                best[j] = d;
                bi[j] = base + k;
            }
        }
    }
}

template <int DIM>
__global__ void __launch_bounds__(NN_THREADS)
    k_nearest_point(const float *__restrict__ ref, const float *__restrict__ que, int32_t *__restrict__ idxs, int pn1,
                    int pn2)
{
    using V = NnVec<DIM>;
    __shared__ V s_ref[NN_TILE];
    const int img = blockIdx.y;
    const float *r = ref + (size_t)img * pn1 * DIM;
    const float *q = que + (size_t)img * pn2 * DIM;
    const int q0 = blockIdx.x * NN_QPB + threadIdx.x;
    float qx[NN_Q], qy[NN_Q], qz[NN_Q], best[NN_Q];
    int bi[NN_Q];
#pragma unroll
    for (int j = 0; j < NN_Q; ++j) {
        const int qi = q0 + j * NN_THREADS;
        const bool ok = qi < pn2;
        qx[j] = ok ? q[(size_t)qi * DIM] : 0.f;
        qy[j] = ok ? q[(size_t)qi * DIM + 1] : 0.f;
        qz[j] = (ok && DIM == 3) ? q[(size_t)qi * DIM + 2] : 0.f;
        best[j] = FLT_MAX;
        bi[j] = 0;
    }
    for (int base = 0; base < pn1; base += NN_TILE) {
        const int n = min(NN_TILE, pn1 - base);
        __syncthreads();
        for (int k = threadIdx.x; k < n; k += NN_THREADS) {
            const float *p = r + (size_t)(base + k) * DIM;
            if constexpr (DIM == 3)
                s_ref[k] = make_float4(p[0], p[1], p[2], 0.f);
            else
                s_ref[k] = make_float2(p[0], p[1]);
        }
        __syncthreads();
        nn_scan_tile<NN_Q>(s_ref, n, base, qx, qy, qz, best, bi);
    }
#pragma unroll
    for (int j = 0; j < NN_Q; ++j) {
        const int qi = q0 + j * NN_THREADS;
        if (qi < pn2) idxs[(size_t)img * pn2 + qi] = bi[j];
    }
}

// ------------------------------------------------------------------------------------------------ pose metrics
// The fixed fp64 order (oracle/eval_oracle.py states the same):
//   p_r   = ((R[r,0] X + R[r,1] Y) + R[r,2] Z) + t[r]
//   h_r   = (K[r,0] p_0 + K[r,1] p_1) + K[r,2] p_2,   uv = (h_0 / h_2, h_1 / h_2)
//   |d|   = sqrt((d_0 d_0 + d_1 d_1) + d_2 d_2)        (2-D: sqrt(d_0 d_0 + d_1 d_1))
struct D3 {
    double x, y, z;
};

__device__ __forceinline__ double row3(const double *a, double x, double y, double z)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], x), __dmul_rn(a[1], y)), __dmul_rn(a[2], z));
}
// pose: row-major [3,4] (R | t)
__device__ __forceinline__ D3 transform(const double *pose, double x, double y, double z)
{
    return {__dadd_rn(row3(pose, x, y, z), pose[3]), __dadd_rn(row3(pose + 4, x, y, z), pose[7]),
            __dadd_rn(row3(pose + 8, x, y, z), pose[11])};
}
__device__ __forceinline__ void project(const double *K, D3 p, double &u, double &v)
{
    const double h0 = row3(K, p.x, p.y, p.z), h1 = row3(K + 3, p.x, p.y, p.z), h2 = row3(K + 6, p.x, p.y, p.z);
    u = __ddiv_rn(h0, h2);
    v = __ddiv_rn(h1, h2);
}
__device__ __forceinline__ double norm3(double a, double b, double c)
{
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)), __dmul_rn(c, c)));
}
__device__ __forceinline__ double norm2(double a, double b)
{
    return __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b)));
}

struct HostCam {
    double k[9];
};

// grid (chunks, b): every CTA handles PM_QPB model points of one image and writes its two partial sums
// (sum of ADD(-S) distances, sum of 2-D projection distances) to partial[(img * chunks + chunk) * 2 + {0,1}].
__global__ void __launch_bounds__(PM_THREADS)
    k_pose_metrics_partial(const double *__restrict__ pose_pred, const double *__restrict__ pose_gt,
                           const float *__restrict__ model, int n, HostCam cam, const double *__restrict__ cam_dev,
                           int symmetric, int sym_proj, double *__restrict__ partial)
{
    __shared__ double s_par[33];                 // pred pose [12], gt pose [12], K [9]
    __shared__ float4 s_p3[PM_TILE];             // fp32 roundings of a tile of the pred-transformed cloud
    __shared__ float2 s_p2[PM_TILE];             // ... and of its projections
    __shared__ double s_red[2][PM_THREADS];
    const int img = blockIdx.y, tid = threadIdx.x;
    if (tid < 12) s_par[tid] = pose_pred[(size_t)img * 12 + tid];
    else if (tid < 24) s_par[tid] = pose_gt[(size_t)img * 12 + tid - 12];
    else if (tid == 24)
#pragma unroll
        for (int i = 0; i < 9; ++i) s_par[24 + i] = cam_dev ? cam_dev[(size_t)img * 9 + i] : cam.k[i];
    __syncthreads();
    const double *Pp = s_par, *Pg = s_par + 12, *K = s_par + 24;

    const int q0 = blockIdx.x * PM_QPB + tid;
    // queries: the gt-transformed points (3-D) and their projections (2-D), rounded to fp32
    float qx[PM_Q], qy[PM_Q], qz[PM_Q], best3[PM_Q], ux[PM_Q], uy[PM_Q], uz[PM_Q], best2[PM_Q];
    int bi3[PM_Q], bi2[PM_Q];
#pragma unroll
    for (int j = 0; j < PM_Q; ++j) {
        const int qi = min(q0 + j * PM_THREADS, n - 1);
        const D3 g = transform(Pg, model[(size_t)qi * 3], model[(size_t)qi * 3 + 1], model[(size_t)qi * 3 + 2]);
        double gu, gv;
        project(K, g, gu, gv);
        qx[j] = __double2float_rn(g.x);
        qy[j] = __double2float_rn(g.y);
        qz[j] = __double2float_rn(g.z);
        ux[j] = __double2float_rn(gu);
        uy[j] = __double2float_rn(gv);
        uz[j] = 0.f;
        best3[j] = best2[j] = FLT_MAX;
        bi3[j] = bi2[j] = 0;
    }
    if (symmetric || sym_proj) {
        for (int base = 0; base < n; base += PM_TILE) {
            const int m = min(PM_TILE, n - base);
            __syncthreads();
            for (int k = tid; k < m; k += PM_THREADS) {
                const float *x = model + (size_t)(base + k) * 3;
                const D3 p = transform(Pp, x[0], x[1], x[2]);
                s_p3[k] = make_float4(__double2float_rn(p.x), __double2float_rn(p.y), __double2float_rn(p.z), 0.f);
                if (sym_proj) {
                    double pu, pv;
                    project(K, p, pu, pv);
                    s_p2[k] = make_float2(__double2float_rn(pu), __double2float_rn(pv));
                }
            }
            __syncthreads();
            if (symmetric) nn_scan_tile<PM_Q>(s_p3, m, base, qx, qy, qz, best3, bi3);
            if (sym_proj) nn_scan_tile<PM_Q>(s_p2, m, base, ux, uy, uz, best2, bi2);
        }
    }
    double sum_add = 0.0, sum_proj = 0.0;
#pragma unroll
    for (int j = 0; j < PM_Q; ++j) {
        const int qi = q0 + j * PM_THREADS;
        if (qi >= n) continue;
        const float *x = model + (size_t)qi * 3;
        const D3 g = transform(Pg, x[0], x[1], x[2]);
        double gu, gv;
        project(K, g, gu, gv);
        // ADD: the same vertex under the predicted pose; ADD-S: the nearest predicted vertex (fp64, from model[idx])
        const float *xa = symmetric ? model + (size_t)bi3[j] * 3 : x;
        const D3 pa = transform(Pp, xa[0], xa[1], xa[2]);
        sum_add = __dadd_rn(sum_add, norm3(__dsub_rn(pa.x, g.x), __dsub_rn(pa.y, g.y), __dsub_rn(pa.z, g.z)));
        const float *xp = sym_proj ? model + (size_t)bi2[j] * 3 : x;
        const D3 pp = (xp == xa) ? pa : transform(Pp, xp[0], xp[1], xp[2]);
        double pu, pv;
        project(K, pp, pu, pv);
        sum_proj = __dadd_rn(sum_proj, norm2(__dsub_rn(pu, gu), __dsub_rn(pv, gv)));
    }
    // fixed-order tree over the CTA
    s_red[0][tid] = sum_add;
    s_red[1][tid] = sum_proj;
    for (int s = PM_THREADS / 2; s > 0; s >>= 1) {
        __syncthreads();
        if (tid < s) {
            s_red[0][tid] += s_red[0][tid + s];
            s_red[1][tid] += s_red[1][tid + s];
        }
    }
    if (tid == 0) {
        double *o = partial + ((size_t)img * gridDim.x + blockIdx.x) * 2;
        o[0] = s_red[0][0];
        o[1] = s_red[1][0];
    }
}

// one thread per image: partial sums in chunk order -> out[img] = (add, proj, trans_cm, angle_deg)
__global__ void k_pose_metrics_final(const double *__restrict__ pose_pred, const double *__restrict__ pose_gt,
                                     const double *__restrict__ partial, int chunks, int n, int b,
                                     double *__restrict__ out)
{
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= b) return;
    double sa = 0.0, sp = 0.0;
    for (int c = 0; c < chunks; ++c) {
        sa += partial[((size_t)img * chunks + c) * 2];
        sp += partial[((size_t)img * chunks + c) * 2 + 1];
    }
    const double *Pp = pose_pred + (size_t)img * 12, *Pg = pose_gt + (size_t)img * 12;
    // evaluation_utils.py:136-140; tr(R_p R_g^T) = sum_r ((Rp[r,0] Rg[r,0] + Rp[r,1] Rg[r,1]) + Rp[r,2] Rg[r,2])
    const double trans = __dmul_rn(norm3(__dsub_rn(Pp[3], Pg[3]), __dsub_rn(Pp[7], Pg[7]), __dsub_rn(Pp[11], Pg[11])),
                                   100.0);
    double tr = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) tr = __dadd_rn(tr, row3(Pp + 4 * r, Pg[4 * r], Pg[4 * r + 1], Pg[4 * r + 2]));
    tr = (tr <= 3.0) ? tr : 3.0;                 // `trace if trace <= 3 else 3` (a NaN trace becomes 3, as there)
    const double ang = __dmul_rn(acos(__ddiv_rn(__dsub_rn(tr, 1.0), 2.0)), 180.0 / 3.141592653589793);
    double *o = out + (size_t)img * 4;
    o[0] = __ddiv_rn(sa, (double)n);
    o[1] = __ddiv_rn(sp, (double)n);
    o[2] = trans;
    o[3] = ang;
}

int pm_chunks(int n) { return (n + PM_QPB - 1) / PM_QPB; }

}  // namespace

extern "C" {

int pvnet_find_nearest_point_idx(const float *ref_pts, const float *que_pts, int32_t *idxs, int b, int pn1, int pn2,
                                 int dim, pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && pn1 >= 1 && pn2 >= 1, "non-positive dimension (b=%d, pn1=%d, pn2=%d)", b, pn1, pn2);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    PV_CHECK_ARG(dim == 2 || dim == 3, "dim %d is not 2 or 3", dim);
    PV_CHECK_ARG(ref_pts && que_pts && idxs, "null pointer");
    const dim3 grid((pn2 + NN_QPB - 1) / NN_QPB, b);
    if (dim == 3) {
        k_nearest_point<3><<<grid, NN_THREADS, 0, (cudaStream_t)stream>>>(ref_pts, que_pts, idxs, pn1, pn2);
        PV_LAUNCHED("k_nearest_point<3>");
    } else {
        k_nearest_point<2><<<grid, NN_THREADS, 0, (cudaStream_t)stream>>>(ref_pts, que_pts, idxs, pn1, pn2);
        PV_LAUNCHED("k_nearest_point<2>");
    }
    return PVNET_OK;
}

int pvnet_pose_metrics_workspace_bytes(int b, int n, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && n >= 1, "non-positive dimension (b=%d, n=%d)", b, n);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = (size_t)b * pm_chunks(n) * 2 * sizeof(double);
    return PVNET_OK;
}

int pvnet_pose_metrics(const double *pose_pred, const double *pose_gt, const float *model, int n,
                       const double camera_matrix[9], const double *camera_dev, int b, int symmetric, int sym_proj,
                       double *out, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && n >= 1, "non-positive dimension (b=%d, n=%d)", b, n);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    PV_CHECK_ARG(pose_pred && pose_gt && model && out && workspace, "null pointer");
    PV_CHECK_ARG((camera_matrix != nullptr) != (camera_dev != nullptr), "pass exactly one of camera_matrix / camera_dev");
    size_t need = 0;
    pvnet_pose_metrics_workspace_bytes(b, n, &need);
    PV_CHECK_ARG(workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);
    HostCam cam = {};
    if (camera_matrix)
        for (int i = 0; i < 9; ++i) cam.k[i] = camera_matrix[i];
    double *partial = static_cast<double *>(workspace);
    const int chunks = pm_chunks(n);
    k_pose_metrics_partial<<<dim3(chunks, b), PM_THREADS, 0, (cudaStream_t)stream>>>(
        pose_pred, pose_gt, model, n, cam, camera_dev, symmetric != 0, sym_proj != 0, partial);
    PV_LAUNCHED("k_pose_metrics_partial");
    k_pose_metrics_final<<<(b + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pose_pred, pose_gt, partial, chunks, n, b,
                                                                             out);
    PV_LAUNCHED("k_pose_metrics_final");
    return PVNET_OK;
}

}  // extern "C"
