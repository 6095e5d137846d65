// refine.cu -- silhouette pose refinement for a batch of poses (DESIGN.md §26): the four steps the reference's
// `post_refinement` docstring lists and leaves unimplemented (lib/utils/extend_utils/extend_utils.py:181-193).
//
// One round, per image: render the depth at the current pose with pvnet_render_mesh (the renderer itself, not a
// copy); take the silhouette (covered pixels with an uncovered or outside 4-neighbour) and back-project it to object
// space; take the mask's contour (foreground pixels with a background or outside 4-neighbour; the first round only,
// the mask does not change); pair each silhouette point with its nearest contour pixel; then, pairs held fixed, a few
// damped Gauss-Newton steps on sum |pi(K(R X + t)) - c|^2 with R <- exp(dw) R, t <- t + dt.  The next round's render
// evaluates the step: a round whose mean pair distance rose is undone and the image stops.  oracle/refine_oracle.py
// restates every stage; the boundary sets, back-projection and pairs follow it bit for bit (one rounded __d*_rn /
// __f*_rn intrinsic per operation where the order matters), the normal equations to rounding.
//
// Launches per evaluation: the renderer's three, k_refine_boundary (one 512-thread CTA per image and point set),
// k_refine_pairs (a 256-point tile of one image's silhouette per CTA against its whole contour, staged through shared
// memory) and k_refine_step (one CTA per image: the mean distance, the accept / reject decision and the
// Gauss-Newton steps, the 6x6 sums reduced in a fixed order).  Nothing is allocated and nothing synchronises.
//
// Keypoint anchoring (DESIGN.md §27, pvnet_refine_poses_keypoints): k_refine_step<true> adds the voted keypoints'
// weighted reprojection term (lambda / nk) sum_k |W_k (pi(R P_k + t) - x_k)|^2 to the pair term, which it then
// divides by the pair count, and judges each round by mean pair distance + lambda * mean_k |W_k e_k|.  Warp 0 holds
// one keypoint per lane; the other launches are the same as without keypoints.
#include "common.cuh"

#include <climits>
#include <cmath>

namespace {

constexpr int RF_BOUND_THREADS = 512;
constexpr int RF_PER_THREAD = 16;                 // consecutive pixels per thread in the boundary scan
constexpr int RF_CHUNK = RF_BOUND_THREADS * RF_PER_THREAD;
constexpr int RF_PAIR_THREADS = 256;
constexpr int RF_TILE = 2048;                     // contour points per shared-memory tile (16 KB)
constexpr int RF_STEP_THREADS = 256;
constexpr int RF_GN_STEPS = 3;
constexpr double RF_DAMPING = 1e-3;
constexpr int RF_MIN_PAIRS = 6;
constexpr int RF_NSUM = 27;                       // 21 entries of the upper triangle of A, then g

constexpr int RF_MAX_KP = 32;                     // keypoints: one lane of warp 0 each

constexpr int RF_NO_CONTOUR = 1, RF_NO_SILHOUETTE = 2, RF_FEW_PAIRS = 4, RF_SINGULAR = 8, RF_REJECTED = 16;
constexpr int RF_NO_INSTANCE = 32;                // pvnet_refine_poses_instances: a row past its image's count

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

struct Cam {
    double fx, s, cx, fy, cy;                     // K as the renderer reads it: fp32 widened
};

__device__ __forceinline__ Cam load_cam(const float *K)
{
    return {(double)K[0], (double)K[1], (double)K[2], (double)K[4], (double)K[5]};
}

// Per-image state across rounds (workspace).  cost*: the keypoint-anchored round cost (k_refine_step<true> only).
struct State {
    double backup[12];                            // the pose the current round started from
    double mean0, mean_prev, mean_after;
    double cost0, cost_prev, cost_after;
    int status, done, pairs, pad;
};

// The keypoint term's inputs (all device pointers; kp_eq nullable): keypoints f32 [b,nk,2] in pixels, model points
// f32 [nk,3], weights f32 [b,nk,3] = (wxx, wxy, wyy), lambda = keypoint_weight.
struct KpArgs {
    const float *kp, *pts, *wgt;
    int nk;
    double lambda;
    double *kp_eq;                                // trace: the first step's keypoint sums [b,27]
};

// Projection of X at pose P (row-major [3,4] fp64), the renderer's order: p = R X, Xc = p + t,
// u = ((fx X + s Y) + cx Z) / Z, v = (fy Y + cy Z) / Z.
__device__ __forceinline__ void project(const double *P, const Cam &c, double x, double y, double z, double &u,
                                        double &v)
{
    double Xc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) Xc[r] = da(da(da(dm(P[r * 4], x), dm(P[r * 4 + 1], y)), dm(P[r * 4 + 2], z)), P[r * 4 + 3]);
    u = dd(da(da(dm(c.fx, Xc[0]), dm(c.s, Xc[1])), dm(c.cx, Xc[2])), Xc[2]);
    v = dd(da(dm(c.fy, Xc[1]), dm(c.cy, Xc[2])), Xc[2]);
}

// Boundary of one point set of one image: blockIdx.y == 0 the silhouette (depth > 0), 1 the mask's contour (nonzero).
// Pass 1 counts the boundary pixels; pass 2 walks them again in row-major order and keeps rank % stride == 0,
// stride = ceil(n / max_points), writing each at rank / stride.  A silhouette point is back-projected at the pose
// it was rendered from.  skip_done: images already stopped are left alone.
// The count-then-rank scan of one point set of image img (the body of both boundary kernels): edge(p) says whether
// pixel p is in the set; dep is the image's rendered depth, read for the silhouette's back-projection.
template <class Edge>
__device__ __forceinline__ void boundary_scan(const Edge &edge, int img, int which, const float *__restrict__ dep,
                                              const float *__restrict__ K,
                                              int kstride, int h, int w, int max_points, int32_t *__restrict__ sil_idx,
                                              double *__restrict__ sil_obj, int32_t *__restrict__ con_idx,
                                              int32_t *__restrict__ counts, int *s_warp, int &s_total, double *s_pose)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long hw = static_cast<long long>(h) * w;
    int local = 0;
    for (long long base = 0; base < hw; base += RF_CHUNK)
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            if (p < hw && edge(p)) ++local;
        }
    atomicAdd(&s_total, local);                   // an integer sum: the same whatever the order
    __syncthreads();
    const int n = s_total;
    const int stride = n > max_points ? (n + max_points - 1) / max_points : 1;
    int32_t *idx_out = (which == 0 ? sil_idx : con_idx) + static_cast<size_t>(img) * max_points;
    double *obj_out = sil_obj + static_cast<size_t>(img) * max_points * 3;
    const Cam cam = load_cam(K + static_cast<size_t>(img) * kstride);
    int running = 0;                              // boundary pixels in earlier chunks
    for (long long base = 0; base < hw; base += RF_CHUNK) {
        unsigned bits = 0;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            if (p < hw && edge(p)) bits |= 1u << q;
        }
        const int cnt = __popc(bits);
        int incl = cnt;                           // inclusive scan over the warp
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int t = lane < RF_BOUND_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, t, o);
                if (lane >= o) t += y;
            }
            if (lane < RF_BOUND_THREADS / 32) s_warp[lane] = t;   // inclusive warp totals
        }
        __syncthreads();
        int rank = running + (warp ? s_warp[warp - 1] : 0) + incl - cnt;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            if (!(bits >> q & 1u)) continue;
            if (rank % stride == 0) {
                const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
                const int j = rank / stride;
                idx_out[j] = static_cast<int32_t>(p);
                if (which == 0) {
                    const int r = static_cast<int>(p / w), c = static_cast<int>(p - static_cast<long long>(r) * w);
                    const double u = c + 0.5, v = r + 0.5, Z = dep[p];
                    const double yn = dd(ds(v, cam.cy), cam.fy);
                    const double xn = dd(ds(ds(u, cam.cx), dm(cam.s, yn)), cam.fx);
                    const double d0 = ds(dm(Z, xn), s_pose[3]), d1 = ds(dm(Z, yn), s_pose[7]), d2 = ds(Z, s_pose[11]);
#pragma unroll
                    for (int k = 0; k < 3; ++k)
                        obj_out[j * 3 + k] = da(da(dm(s_pose[k], d0), dm(s_pose[4 + k], d1)), dm(s_pose[8 + k], d2));
                }
            }
            ++rank;
        }
        running += s_warp[RF_BOUND_THREADS / 32 - 1];
        __syncthreads();                          // s_warp is rewritten by the next chunk
    }
    if (tid == 0) counts[img * 2 + which] = n ? (n + stride - 1) / stride : 0;
}

__global__ void __launch_bounds__(RF_BOUND_THREADS, 1)
    k_refine_boundary(const float *__restrict__ depth, const uint8_t *__restrict__ mask, const double *__restrict__ pose,
                      const float *__restrict__ K, int kstride, int h, int w, int max_points, int skip_done,
                      const State *__restrict__ state, int32_t *__restrict__ sil_idx, double *__restrict__ sil_obj,
                      int32_t *__restrict__ con_idx, int32_t *__restrict__ counts)
{
    const int img = blockIdx.x, which = blockIdx.y;
    if (skip_done && state[img].done) return;
    __shared__ int s_warp[RF_BOUND_THREADS / 32];
    __shared__ int s_total;
    __shared__ double s_pose[12];
    const int tid = threadIdx.x;
    const long long hw = static_cast<long long>(h) * w;
    const float *dep = depth + img * hw;
    const uint8_t *msk = mask + img * hw;
    if (tid == 0) s_total = 0;
    if (tid < 12) s_pose[tid] = pose[img * 12 + tid];
    __syncthreads();
    auto on = [&](long long p) -> bool { return which == 0 ? dep[p] > 0.f : msk[p] != 0; };
    auto edge = [&](long long p) -> bool {
        if (!on(p)) return false;
        const int r = static_cast<int>(p / w), c = static_cast<int>(p - static_cast<long long>(r) * w);
        if (r == 0 || r == h - 1 || c == 0 || c == w - 1) return true;
        return !on(p - 1) || !on(p + 1) || !on(p - w) || !on(p + w);
    };
    boundary_scan(edge, img, which, dep, K, kstride, h, w, max_points, sil_idx, sil_obj, con_idx, counts, s_warp,
                  s_total, s_pose);
}

// The boundary sets of virtual image img = bi * L + j, instance j of image bi's label map (DESIGN.md §30).  The label
// values are read at their own width (T) and compared as integers; anything nonzero other than j+1, including values
// above L, is another instance.  Contour (blockIdx.y == 1): pixels of value j+1 with a 4-neighbour of value 0 or on
// the image border; a border with another instance is not outline evidence.  Silhouette (0): the rendered depth's
// covered-boundary pixels, as k_refine_boundary takes them, less those whose 3x3 neighbourhood (inside the image) holds
// another instance, where the outline may be hidden; they are left out before the max_points stride.  Rows already
// done (the absent instances, from the start) are skipped.
template <typename T>
__global__ void __launch_bounds__(RF_BOUND_THREADS, 1)
    k_refine_boundary_instances(const float *__restrict__ depth, const T *__restrict__ labels, int L,
                                const double *__restrict__ pose, const float *__restrict__ K, int kstride, int h,
                                int w, int max_points, const State *__restrict__ state, int32_t *__restrict__ sil_idx,
                                double *__restrict__ sil_obj, int32_t *__restrict__ con_idx,
                                int32_t *__restrict__ counts)
{
    const int img = blockIdx.x, which = blockIdx.y;
    if (state[img].done) return;
    __shared__ int s_warp[RF_BOUND_THREADS / 32];
    __shared__ int s_total;
    __shared__ double s_pose[12];
    const int tid = threadIdx.x;
    const long long hw = static_cast<long long>(h) * w;
    const int bi = img / L;
    const long long own = img - bi * L + 1;
    const float *dep = depth + img * hw;
    const T *lab = labels + bi * hw;
    if (tid == 0) s_total = 0;
    if (tid < 12) s_pose[tid] = pose[img * 12 + tid];
    __syncthreads();
    auto val = [&](long long p) -> long long { return static_cast<long long>(lab[p]); };
    auto other = [&](long long p) -> bool { const long long v = val(p); return v != 0 && v != own; };
    auto edge = [&](long long p) -> bool {
        const int r = static_cast<int>(p / w), c = static_cast<int>(p - static_cast<long long>(r) * w);
        const bool border = r == 0 || r == h - 1 || c == 0 || c == w - 1;
        if (which == 1) {
            if (val(p) != own) return false;
            if (border) return true;
            return val(p - 1) == 0 || val(p + 1) == 0 || val(p - w) == 0 || val(p + w) == 0;
        }
        if (!(dep[p] > 0.f)) return false;
        if (!border && dep[p - 1] > 0.f && dep[p + 1] > 0.f && dep[p - w] > 0.f && dep[p + w] > 0.f) return false;
        for (int dr = -1; dr <= 1; ++dr) {
            if (r + dr < 0 || r + dr >= h) continue;
            for (int dc = -1; dc <= 1; ++dc)
                if (c + dc >= 0 && c + dc < w && other(p + static_cast<long long>(dr) * w + dc)) return false;
        }
        return true;
    };
    boundary_scan(edge, img, which, dep, K, kstride, h, w, max_points, sil_idx, sil_obj, con_idx, counts, s_warp,
                  s_total, s_pose);
}

// Absent rows (j >= num[bi]) start done with status RF_NO_INSTANCE and keep their input pose.  Their fp32 render pose
// is all zeros: every vertex then sits at camera depth 0, below the near plane, so the renderer's face box rejects
// every face and rasterises nothing for them.
__global__ void k_refine_absent(const int32_t *__restrict__ num, int L, int nrows, State *__restrict__ state,
                                float *__restrict__ pose32)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows || i % L < num[i / L]) return;
    state[i].done = 1;
    state[i].status = RF_NO_INSTANCE;
    for (int q = 0; q < 12; ++q) pose32[i * 12 + q] = 0.f;
}

// Nearest contour pixel of each silhouette point: grid (ceil(max_points / 256), b).  The point is projected at the
// current pose and rounded to fp32; d2 = (cu - pu)^2 + (cv - pv)^2 in fp32, each operation rounded; the strictly
// smaller d2 wins while the contour is walked in order, so ties keep the lowest index.  pair = -1 when the nearest
// d2 is above gate2 or is not a number (or there is no contour).
__global__ void __launch_bounds__(RF_PAIR_THREADS)
    k_refine_pairs(const double *__restrict__ pose, const float *__restrict__ K, int kstride, int w, int max_points,
                   float gate2, int skip_done, const State *__restrict__ state, const int32_t *__restrict__ counts,
                   const double *__restrict__ sil_obj, const int32_t *__restrict__ con_idx,
                   int32_t *__restrict__ pair, float *__restrict__ pair_d2)
{
    const int img = blockIdx.y;
    if (skip_done && state[img].done) return;
    const int ns = counts[img * 2], nc = counts[img * 2 + 1];
    const int i = blockIdx.x * RF_PAIR_THREADS + threadIdx.x;
    if (static_cast<int>(blockIdx.x) * RF_PAIR_THREADS >= ns) return;
    __shared__ float2 s_c[RF_TILE];
    float pu = 0.f, pv = 0.f;
    if (i < ns) {
        const double *P = pose + img * 12;
        const double *X = sil_obj + (static_cast<size_t>(img) * max_points + i) * 3;
        double u, v;
        project(P, load_cam(K + static_cast<size_t>(img) * kstride), X[0], X[1], X[2], u, v);
        pu = __double2float_rn(u);
        pv = __double2float_rn(v);
    }
    float best = INFINITY;
    int bj = -1;
    const int32_t *con = con_idx + static_cast<size_t>(img) * max_points;
    for (int t0 = 0; t0 < nc; t0 += RF_TILE) {
        const int tn = min(RF_TILE, nc - t0);
        __syncthreads();
        for (int j = threadIdx.x; j < tn; j += RF_PAIR_THREADS) {
            const int p = con[t0 + j], r = p / w, c = p - r * w;
            s_c[j] = make_float2(c + 0.5f, r + 0.5f);
        }
        __syncthreads();
        for (int j = 0; j < tn; ++j) {
            const float2 cc = s_c[j];
            const float dx = __fsub_rn(cc.x, pu), dy = __fsub_rn(cc.y, pv);
            const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
            if (d2 < best) {
                best = d2;
                bj = t0 + j;
            }
        }
    }
    if (i < ns) {
        const size_t o = static_cast<size_t>(img) * max_points + i;
        pair[o] = best <= gate2 ? bj : -1;
        pair_d2[o] = best;
    }
}

// Xor butterflies at offsets 16, 8, 4, 2, 1 over the warp: every lane ends with the same sum of each entry.
template <int N>
__device__ __forceinline__ void warp_xor_sum(double (&v)[N])
{
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
}

// Block sum of n doubles per thread into out (thread 0's view): xor butterflies within each warp, then the warps'
// partials in warp order.  The same inputs give the same sum every run.
template <int N>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*s_part)[N], double *out)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    warp_xor_sum(v);
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) s_part[warp][k] = v[k];
    __syncthreads();
    if (threadIdx.x == 0)
        for (int k = 0; k < N; ++k) {
            double t = s_part[0][k];
            for (int q = 1; q < RF_STEP_THREADS / 32; ++q) t += s_part[q][k];
            out[k] = t;
        }
    __syncthreads();
}

// Rodrigues, pnp.cu's form: E = I + a [w]x + b [w]x^2, row-major.
__device__ void so3_exp(double wx, double wy, double wz, double (&E)[9])
{
    const double th2 = wx * wx + wy * wy + wz * wz;
    double a, b;
    if (th2 < 1e-16) {
        a = 1.0 - th2 / 6.0;
        b = 0.5 - th2 / 24.0;
    } else {
        const double th = sqrt(th2);
        a = sin(th) / th;
        b = (1.0 - cos(th)) / th2;
    }
    E[0] = 1.0 - b * (wy * wy + wz * wz);
    E[1] = -a * wz + b * wx * wy;
    E[2] = a * wy + b * wx * wz;
    E[3] = a * wz + b * wx * wy;
    E[4] = 1.0 - b * (wx * wx + wz * wz);
    E[5] = -a * wx + b * wy * wz;
    E[6] = -a * wy + b * wx * wz;
    E[7] = a * wx + b * wy * wz;
    E[8] = 1.0 - b * (wx * wx + wy * wy);
}

// (A + RF_DAMPING diag(A)) x = -g by Cholesky, A from the 21 upper-triangle sums.  false: not positive definite.
__device__ bool damped_solve(const double *sum, double (&x)[6])
{
    double L[6][6];
    int k = 0;
    for (int r = 0; r < 6; ++r)
        for (int c = r; c < 6; ++c) {
            L[c][r] = sum[k++];
            if (c == r) L[r][r] += RF_DAMPING * L[r][r];
        }
    for (int j = 0; j < 6; ++j) {
        double d = L[j][j];
        for (int q = 0; q < j; ++q) d -= L[j][q] * L[j][q];
        if (!(d > 0.0) || !isfinite(d)) return false;
        d = sqrt(d);
        L[j][j] = d;
        for (int r = j + 1; r < 6; ++r) {
            double t = L[r][j];
            for (int q = 0; q < j; ++q) t -= L[r][q] * L[j][q];
            L[r][j] = t / d;
        }
    }
    double y[6];
    for (int r = 0; r < 6; ++r) {
        double t = -sum[21 + r];
        for (int q = 0; q < r; ++q) t -= L[r][q] * y[q];
        y[r] = t / L[r][r];
    }
    for (int r = 5; r >= 0; --r) {
        double t = y[r];
        for (int q = r + 1; q < 6; ++q) t -= L[q][r] * x[q];
        x[r] = t / L[r][r];
    }
    for (int r = 0; r < 6; ++r)
        if (!isfinite(x[r])) return false;
    return true;
}

// Keypoint term, warp 0: lane l < nk holds keypoint l as (x, y, X, Y, Z, wxx, wxy, wyy) in fp64.  A keypoint with a
// non-finite coordinate or weight is left out (it adds zero to every sum).
__device__ __forceinline__ bool load_keypoint(const KpArgs &a, int img, int lane, double (&q)[8])
{
    if (lane >= a.nk) return false;
    const size_t e = static_cast<size_t>(img) * a.nk + lane;
    q[0] = a.kp[e * 2];
    q[1] = a.kp[e * 2 + 1];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        q[2 + r] = a.pts[lane * 3 + r];
        q[5 + r] = a.wgt[e * 3 + r];
    }
    bool ok = true;
#pragma unroll
    for (int r = 0; r < 8; ++r) ok = ok && isfinite(q[r]);
    return ok;
}

// |W (pi(R P + t) - x)| of one keypoint, each operation rounded (oracle/refine_keypoints_oracle.py restates it bit
// for bit): the projection is `project`'s, e = (u - x, v - y), r = (wxx eu + wxy ev, wxy eu + wyy ev),
// sqrt(r0 r0 + r1 r1).
__device__ __forceinline__ double keypoint_distance(const double *P, const Cam &c, const double *q)
{
    double u, v;
    project(P, c, q[2], q[3], q[4], u, v);
    const double eu = ds(u, q[0]), ev = ds(v, q[1]);
    const double r0 = da(dm(q[5], eu), dm(q[6], ev)), r1 = da(dm(q[6], eu), dm(q[7], ev));
    return __dsqrt_rn(da(dm(r0, r0), dm(r1, r1)));
}

// One keypoint's 27 sums of the weighted residual r = W e at pose P: J_w = W [Ju; Jv] with the pairs' Jacobian,
// the 21 upper-triangle entries of J_w^T J_w row by row, then J_w^T r.
__device__ __forceinline__ void keypoint_sums(const double *P, const Cam &cam, const double *q, double (&v)[RF_NSUM])
{
    double p[3], Xc[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        p[r] = P[r * 4] * q[2] + P[r * 4 + 1] * q[3] + P[r * 4 + 2] * q[4];
        Xc[r] = p[r] + P[r * 4 + 3];
    }
    const double iz = 1.0 / Xc[2];
    const double u = (cam.fx * Xc[0] + cam.s * Xc[1] + cam.cx * Xc[2]) * iz;
    const double vv = (cam.fy * Xc[1] + cam.cy * Xc[2]) * iz;
    const double eu = u - q[0], ev = vv - q[1];
    const double du[3] = {cam.fx * iz, cam.s * iz, -(u - cam.cx) * iz};
    const double dv[3] = {0.0, cam.fy * iz, -(vv - cam.cy) * iz};
    const double Ju[6] = {p[1] * du[2] - p[2] * du[1], p[2] * du[0] - p[0] * du[2], p[0] * du[1] - p[1] * du[0],
                          du[0], du[1], du[2]};
    const double Jv[6] = {p[1] * dv[2] - p[2] * dv[1], p[2] * dv[0] - p[0] * dv[2], p[0] * dv[1] - p[1] * dv[0],
                          dv[0], dv[1], dv[2]};
    double J0[6], J1[6];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        J0[r] = q[5] * Ju[r] + q[6] * Jv[r];
        J1[r] = q[6] * Ju[r] + q[7] * Jv[r];
    }
    const double r0 = q[5] * eu + q[6] * ev, r1 = q[6] * eu + q[7] * ev;
    int k = 0;
#pragma unroll
    for (int r = 0; r < 6; ++r)
#pragma unroll
        for (int c = r; c < 6; ++c) v[k++] = J0[r] * J0[c] + J1[r] * J1[c];
#pragma unroll
    for (int r = 0; r < 6; ++r) v[21 + r] = J0[r] * r0 + J1[r] * r1;
}

// One CTA per image: evaluation k of the pose (mean pair distance, accept or undo), then, unless k is the last
// evaluation, RF_GN_STEPS Gauss-Newton steps on the pairs.  The pose lives in `pose` (the caller's output); pose32
// is its fp32 copy for the next render.  normal_eq (nullable): the sums of the first step of evaluation 0.
// KP: the keypoint-anchored form.  Each step's pair sums (after block_sum) become, entry by entry and each
// operation rounded, pair / n + (lambda / nk) * kp, kp the keypoints' sums combined by warp 0's xor butterflies;
// the round's cost is C = m + lambda * (kd / nk), m the mean pair distance and kd the butterfly sum of the keypoint
// distances at the evaluated pose, and a round whose C rose is undone.
template <bool KP>
__global__ void __launch_bounds__(RF_STEP_THREADS)
    k_refine_step(double *__restrict__ pose, float *__restrict__ pose32, const float *__restrict__ K, int kstride,
                  int w, int max_points, int k, int last, State *__restrict__ state,
                  const int32_t *__restrict__ counts, const double *__restrict__ sil_obj,
                  const int32_t *__restrict__ con_idx, const int32_t *__restrict__ pair,
                  const float *__restrict__ pair_d2, double *__restrict__ normal_eq, KpArgs kpa)
{
    const int img = blockIdx.x;
    State &S = state[img];
    if (S.done) return;
    __shared__ double s_part[RF_STEP_THREADS / 32][RF_NSUM];
    __shared__ double s_sum[RF_NSUM];
    __shared__ double s_pose[12];
    __shared__ int s_go;
    __shared__ double s_kp[KP ? RF_MAX_KP : 1][8];
    __shared__ int s_kp_on[KP ? RF_MAX_KP : 1];
    const int ns = counts[img * 2], nc = counts[img * 2 + 1];
    const size_t o = static_cast<size_t>(img) * max_points;
    double acc[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < ns; i += RF_STEP_THREADS)
        if (pair[o + i] >= 0) {
            acc[0] += 1.0;
            acc[1] += sqrt(static_cast<double>(pair_d2[o + i]));
        }
    if constexpr (KP) {
        if (threadIdx.x < 12) s_pose[threadIdx.x] = pose[img * 12 + threadIdx.x];
        if (threadIdx.x < RF_MAX_KP) {
            double q[8];
            const bool on = load_keypoint(kpa, img, threadIdx.x, q);
#pragma unroll
            for (int r = 0; r < 8; ++r) s_kp[threadIdx.x][r] = on ? q[r] : 0.0;
            s_kp_on[threadIdx.x] = on;
        }
    }
    block_sum<2>(acc, reinterpret_cast<double (*)[2]>(&s_part[0][0]), s_sum);   // its barriers publish s_pose, s_kp
    double kd[1] = {0.0};
    if constexpr (KP) {
        if (threadIdx.x < 32) {
            if (s_kp_on[threadIdx.x])
                kd[0] = keypoint_distance(s_pose, load_cam(K + static_cast<size_t>(img) * kstride), s_kp[threadIdx.x]);
            warp_xor_sum(kd);
        }
    }
    if (threadIdx.x == 0) {
        const int n = static_cast<int>(s_sum[0]);
        const double m = n ? s_sum[1] / n : NAN;
        const double cost = KP ? da(m, dm(kpa.lambda, dd(kd[0], static_cast<double>(kpa.nk)))) : m;
        bool go = true;
        if (k == 0) {
            int st = 0;
            if (nc == 0) st = RF_NO_CONTOUR;
            else if (ns == 0) st = RF_NO_SILHOUETTE;
            else if (n < RF_MIN_PAIRS) st = RF_FEW_PAIRS;
            if (st) {
                S.status |= st;
                go = false;
            } else {
                S.mean0 = S.mean_after = m;
                if (KP) S.cost0 = S.cost_after = cost;
            }
        } else if (ns == 0 || n < RF_MIN_PAIRS || (KP ? !(cost <= S.cost_prev) : m > S.mean_prev)) {
            // a cost that is not a number (a keypoint at camera depth 0) is not shown to be no higher: undone too
            S.status |= RF_REJECTED;
            for (int q = 0; q < 12; ++q) pose[img * 12 + q] = S.backup[q];
            go = false;
        } else {
            S.mean_after = m;
            if (KP) S.cost_after = cost;
        }
        if (!go) S.done = 1;
        if (go && !last) {
            S.mean_prev = m;
            if (KP) S.cost_prev = cost;
            for (int q = 0; q < 12; ++q) S.backup[q] = pose[img * 12 + q];
            S.pairs = n;
        }
        s_go = go && !last;
    }
    if (threadIdx.x < 12) s_pose[threadIdx.x] = pose[img * 12 + threadIdx.x];
    __syncthreads();
    if (!s_go) return;
    const Cam cam = load_cam(K + static_cast<size_t>(img) * kstride);
    for (int step = 0; step < RF_GN_STEPS; ++step) {
        double v[RF_NSUM];
#pragma unroll
        for (int q = 0; q < RF_NSUM; ++q) v[q] = 0.0;
        for (int i = threadIdx.x; i < ns; i += RF_STEP_THREADS) {
            const int j = pair[o + i];
            if (j < 0) continue;
            const double *X = sil_obj + (o + i) * 3;
            const int cp = con_idx[o + j], cr = cp / w, cc = cp - cr * w;
            double p[3], Xc[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                p[r] = s_pose[r * 4] * X[0] + s_pose[r * 4 + 1] * X[1] + s_pose[r * 4 + 2] * X[2];
                Xc[r] = p[r] + s_pose[r * 4 + 3];
            }
            const double iz = 1.0 / Xc[2];
            const double u = (cam.fx * Xc[0] + cam.s * Xc[1] + cam.cx * Xc[2]) * iz;
            const double vv = (cam.fy * Xc[1] + cam.cy * Xc[2]) * iz;
            const double ru = u - (cc + 0.5), rv = vv - (cr + 0.5);
            const double du[3] = {cam.fx * iz, cam.s * iz, -(u - cam.cx) * iz};
            const double dv[3] = {0.0, cam.fy * iz, -(vv - cam.cy) * iz};
            // d/d(dw) of the projection for R <- exp(dw) R is p x d(proj)/dXc; d/d(dt) is d(proj)/dXc
            const double Ju[6] = {p[1] * du[2] - p[2] * du[1], p[2] * du[0] - p[0] * du[2], p[0] * du[1] - p[1] * du[0],
                                  du[0], du[1], du[2]};
            const double Jv[6] = {p[1] * dv[2] - p[2] * dv[1], p[2] * dv[0] - p[0] * dv[2], p[0] * dv[1] - p[1] * dv[0],
                                  dv[0], dv[1], dv[2]};
            int q = 0;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
                for (int c = r; c < 6; ++c) v[q++] += Ju[r] * Ju[c] + Jv[r] * Jv[c];
#pragma unroll
            for (int r = 0; r < 6; ++r) v[21 + r] += Ju[r] * ru + Jv[r] * rv;
        }
        block_sum<RF_NSUM>(v, s_part, s_sum);
        if constexpr (KP) {
            if (threadIdx.x < 32) {                   // v is free again: warp 0 reuses it for the keypoint sums
                if (s_kp_on[threadIdx.x]) {
                    keypoint_sums(s_pose, cam, s_kp[threadIdx.x], v);
                } else {
#pragma unroll
                    for (int q = 0; q < RF_NSUM; ++q) v[q] = 0.0;
                }
                warp_xor_sum(v);
            }
        }
        if (threadIdx.x == 0) {
            if (normal_eq && k == 0 && step == 0)
                for (int q = 0; q < RF_NSUM; ++q) normal_eq[img * RF_NSUM + q] = s_sum[q];
            if constexpr (KP) {
                if (kpa.kp_eq && k == 0 && step == 0)
                    for (int q = 0; q < RF_NSUM; ++q) kpa.kp_eq[img * RF_NSUM + q] = v[q];
                const double n = static_cast<double>(S.pairs), lk = dd(kpa.lambda, static_cast<double>(kpa.nk));
                for (int q = 0; q < RF_NSUM; ++q) s_sum[q] = da(dd(s_sum[q], n), dm(lk, v[q]));
            }
            double x[6];
            if (!damped_solve(s_sum, x)) {
                S.status |= RF_SINGULAR;
                S.done = 1;
                for (int q = 0; q < 12; ++q) s_pose[q] = S.backup[q];
                s_go = 0;
            } else {
                double E[9], R[9];
                so3_exp(x[0], x[1], x[2], E);
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c)
                        R[r * 3 + c] = E[r * 3] * s_pose[c] + E[r * 3 + 1] * s_pose[4 + c] + E[r * 3 + 2] * s_pose[8 + c];
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c) s_pose[r * 4 + c] = R[r * 3 + c];
                    s_pose[r * 4 + 3] += x[3 + r];
                }
            }
        }
        __syncthreads();
        if (!s_go) break;
    }
    if (threadIdx.x < 12) {
        pose[img * 12 + threadIdx.x] = s_pose[threadIdx.x];
        pose32[img * 12 + threadIdx.x] = __double2float_rn(s_pose[threadIdx.x]);
    }
}

__global__ void k_refine_init(const double *__restrict__ pose_in, double *__restrict__ pose, float *__restrict__ pose32,
                              State *__restrict__ state, int b)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b) return;
    for (int q = 0; q < 12; ++q) {
        pose[i * 12 + q] = pose_in[i * 12 + q];
        pose32[i * 12 + q] = __double2float_rn(pose_in[i * 12 + q]);
    }
    State &S = state[i];
    S.mean0 = S.mean_prev = S.mean_after = NAN;
    S.cost0 = S.cost_prev = S.cost_after = NAN;
    S.status = S.done = S.pairs = S.pad = 0;
}

__global__ void k_refine_finish(const State *__restrict__ state, int b, int32_t *__restrict__ info,
                                double *__restrict__ dist, double *__restrict__ cost)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b) return;
    if (info) {
        info[i * 2] = state[i].status;
        info[i * 2 + 1] = state[i].pairs;
    }
    if (dist) {
        dist[i * 2] = state[i].mean0;
        dist[i * 2 + 1] = state[i].mean_after;
    }
    if (cost) {
        cost[i * 2] = state[i].cost0;
        cost[i * 2 + 1] = state[i].cost_after;
    }
}

struct Layout {
    unsigned long long *keys;
    float *depth, *pose32, *d2;
    int32_t *sil, *con, *pair, *counts;
    double *obj;
    State *state;
    size_t bytes;
};

Layout carve(void *base, int b, int h, int w, int max_points)
{
    pvnet::Carver cv(base);
    Layout L;
    const size_t npix = static_cast<size_t>(b) * h * w, np = static_cast<size_t>(b) * max_points;
    L.keys = cv.take<unsigned long long>(npix);
    L.depth = cv.take<float>(npix);
    L.pose32 = cv.take<float>(static_cast<size_t>(b) * 12);
    L.sil = cv.take<int32_t>(np);
    L.con = cv.take<int32_t>(np);
    L.pair = cv.take<int32_t>(np);
    L.d2 = cv.take<float>(np);
    L.obj = cv.take<double>(np * 3);
    L.counts = cv.take<int32_t>(static_cast<size_t>(b) * 2);
    L.state = cv.take<State>(b);
    L.bytes = pvnet::align_up(cv.off, 256);
    return L;
}

}  // namespace

extern "C" {

int pvnet_refine_workspace_bytes(int b, int h, int w, int max_points, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && max_points >= 1, "non-positive dimension (b=%d, h=%d, w=%d, "
                 "max_points=%d)", b, h, w, max_points);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = carve(nullptr, b, h, w, max_points).bytes;
    return PVNET_OK;
}

}  // extern "C"

namespace {

// The label map of pvnet_refine_poses_instances: labels [b/L,h,w] of element size esz, counts num [b/L].
struct InstArgs {
    const void *labels;
    int esz;
    const int32_t *num;
    int L;
};

// Every entry point: kpa null runs k_refine_step<false>, the silhouette objective alone; inst non-null reads the
// contour and silhouette rules of a label map (mask is then unused) and b counts the virtual images.
int refine_poses(const uint8_t *mask, const double *poses_in, const float *K, int k_per_image, const float *verts,
                 const int32_t *faces, int nv, int nf, int b, int h, int w, float near_clip, float far_clip, int rounds,
                 float gate, int max_points, const KpArgs *kpa, double *poses_out, int32_t *info, double *dist,
                 double *cost, const pvnet_refine_trace_t *trace, void *workspace, size_t workspace_bytes,
                 pvnet_stream_t stream, const InstArgs *inst = nullptr)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && nv >= 0 && nf >= 0, "bad dimension (b=%d, h=%d, w=%d, nv=%d, nf=%d)",
                 b, h, w, nv, nf);
    PV_CHECK_ARG(static_cast<long long>(h) * w <= INT32_MAX, "image %dx%d too large", h, w);
    PV_CHECK_ARG(max_points >= 1 && static_cast<long long>(b) * max_points <= INT32_MAX / 3,
                 "max_points %d outside 1..%d for b = %d", max_points, INT32_MAX / 3 / b, b);
    PV_CHECK_ARG(rounds >= 0, "rounds must be >= 0 (got %d)", rounds);
    PV_CHECK_ARG(gate > 0.f, "gate must be positive (got %g)", gate);
    PV_CHECK_ARG((mask || inst) && poses_in && K && poses_out && (nf == 0 || faces) && (nv == 0 || verts),
                 "null pointer");
    size_t need = 0;
    pvnet_refine_workspace_bytes(b, h, w, max_points, &need);
    PV_CHECK_ARG(workspace && workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);
    const Layout L = carve(workspace, b, h, w, max_points);
    size_t render_need = 0;
    pvnet_render_workspace_bytes(b, h, w, &render_need);
    const cudaStream_t st = (cudaStream_t)stream;
    const int kstride = k_per_image ? 9 : 0;
    volatile float g2v = gate * gate;             // one rounded fp32 multiply
    const float gate2 = g2v;
    k_refine_init<<<(b + 127) / 128, 128, 0, st>>>(poses_in, poses_out, L.pose32, L.state, b);
    PV_LAUNCHED("k_refine_init");
    if (inst) {
        k_refine_absent<<<(b + 127) / 128, 128, 0, st>>>(inst->num, inst->L, b, L.state, L.pose32);
        PV_LAUNCHED("k_refine_absent");
    }
    for (int k = 0; k <= rounds; ++k) {
        const int rc = pvnet_render_mesh(verts, faces, nullptr, nv, nf, L.pose32, K, k_per_image, b, h, w, near_clip,
                                         far_clip, 0.5f, nullptr, L.depth, nullptr, L.keys, render_need, stream);
        if (rc != PVNET_OK) return rc;
        const dim3 bgrid(b, k == 0 ? 2 : 1);
        if (!inst) {
            k_refine_boundary<<<bgrid, RF_BOUND_THREADS, 0, st>>>(L.depth, mask, poses_out, K, kstride, h, w, max_points,
                                                                  k > 0, L.state, L.sil, L.obj, L.con, L.counts);
        } else {
#define PV_BOUNDARY_INSTANCES(T)                                                                                       \
    k_refine_boundary_instances<T><<<bgrid, RF_BOUND_THREADS, 0, st>>>(                                                \
        L.depth, static_cast<const T *>(inst->labels), inst->L, poses_out, K, kstride, h, w, max_points, L.state,     \
        L.sil, L.obj, L.con, L.counts)
            switch (inst->esz) {
            case 1: PV_BOUNDARY_INSTANCES(unsigned char); break;
            case 2: PV_BOUNDARY_INSTANCES(short); break;
            case 4: PV_BOUNDARY_INSTANCES(int); break;
            default: PV_BOUNDARY_INSTANCES(long long); break;
            }
#undef PV_BOUNDARY_INSTANCES
        }
        PV_LAUNCHED("k_refine_boundary");
        // absent instances are done from the start: their point sets were never written
        k_refine_pairs<<<dim3((max_points + RF_PAIR_THREADS - 1) / RF_PAIR_THREADS, b), RF_PAIR_THREADS, 0, st>>>(
            poses_out, K, kstride, w, max_points, gate2, inst || k > 0, L.state, L.counts, L.obj, L.con, L.pair, L.d2);
        PV_LAUNCHED("k_refine_pairs");
        if (k == 0 && trace) {
            const size_t np = static_cast<size_t>(b) * max_points;
            if (trace->sil_idx) PV_CUDA(cudaMemcpyAsync(trace->sil_idx, L.sil, np * 4, cudaMemcpyDeviceToDevice, st));
            if (trace->con_idx) PV_CUDA(cudaMemcpyAsync(trace->con_idx, L.con, np * 4, cudaMemcpyDeviceToDevice, st));
            if (trace->counts)
                PV_CUDA(cudaMemcpyAsync(trace->counts, L.counts, static_cast<size_t>(b) * 8, cudaMemcpyDeviceToDevice,
                                        st));
            if (trace->sil_obj)
                PV_CUDA(cudaMemcpyAsync(trace->sil_obj, L.obj, np * 24, cudaMemcpyDeviceToDevice, st));
            if (trace->pair_idx) PV_CUDA(cudaMemcpyAsync(trace->pair_idx, L.pair, np * 4, cudaMemcpyDeviceToDevice, st));
        }
        double *ne = trace ? trace->normal_eq : nullptr;
        if (kpa)
            k_refine_step<true><<<b, RF_STEP_THREADS, 0, st>>>(poses_out, L.pose32, K, kstride, w, max_points, k,
                                                               k == rounds, L.state, L.counts, L.obj, L.con, L.pair,
                                                               L.d2, ne, *kpa);
        else
            k_refine_step<false><<<b, RF_STEP_THREADS, 0, st>>>(poses_out, L.pose32, K, kstride, w, max_points, k,
                                                                k == rounds, L.state, L.counts, L.obj, L.con, L.pair,
                                                                L.d2, ne, KpArgs{});
        PV_LAUNCHED("k_refine_step");
    }
    if (info || dist || cost) {
        k_refine_finish<<<(b + 127) / 128, 128, 0, st>>>(L.state, b, info, dist, cost);
        PV_LAUNCHED("k_refine_finish");
    }
    return PVNET_OK;
}

}  // namespace

extern "C" {

int pvnet_refine_poses(const uint8_t *mask, const double *poses_in, const float *K, int k_per_image,
                       const float *verts, const int32_t *faces, int nv, int nf, int b, int h, int w, float near_clip,
                       float far_clip, int rounds, float gate, int max_points, double *poses_out, int32_t *info,
                       double *dist, const pvnet_refine_trace_t *trace, void *workspace, size_t workspace_bytes,
                       pvnet_stream_t stream)
{
    return refine_poses(mask, poses_in, K, k_per_image, verts, faces, nv, nf, b, h, w, near_clip, far_clip, rounds,
                        gate, max_points, nullptr, poses_out, info, dist, nullptr, trace, workspace, workspace_bytes,
                        stream);
}

int pvnet_refine_poses_keypoints(const uint8_t *mask, const double *poses_in, const float *K, int k_per_image,
                                 const float *verts, const int32_t *faces, int nv, int nf, int b, int h, int w,
                                 float near_clip, float far_clip, int rounds, float gate, int max_points,
                                 const float *keypoints, const float *points_3d, const float *weights_2d, int nk,
                                 double keypoint_weight, double *poses_out, int32_t *info, double *dist, double *cost,
                                 const pvnet_refine_trace_t *trace, double *keypoint_eq, void *workspace,
                                 size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(keypoints && points_3d && weights_2d, "null pointer");
    PV_CHECK_ARG(nk >= 4 && nk <= RF_MAX_KP, "keypoint count %d outside [4,%d] (one lane per keypoint)", nk,
                 RF_MAX_KP);
    PV_CHECK_ARG(keypoint_weight >= 0.0 && keypoint_weight < INFINITY, "keypoint_weight must be finite and >= 0 "
                 "(got %g)", keypoint_weight);
    const KpArgs kpa{keypoints, points_3d, weights_2d, nk, keypoint_weight, keypoint_eq};
    return refine_poses(mask, poses_in, K, k_per_image, verts, faces, nv, nf, b, h, w, near_clip, far_clip, rounds,
                        gate, max_points, &kpa, poses_out, info, dist, cost, trace, workspace, workspace_bytes, stream);
}

int pvnet_refine_poses_instances(const void *labels, int labels_elem_size, const int32_t *num, int L,
                                 const double *poses_in, const float *K, const float *verts, const int32_t *faces,
                                 int nv, int nf, int b, int h, int w, float near_clip, float far_clip, int rounds,
                                 float gate, int max_points, const float *keypoints, const float *points_3d,
                                 const float *weights_2d, int nk, double keypoint_weight, double *poses_out,
                                 int32_t *info, double *dist, double *cost, const pvnet_refine_trace_t *trace,
                                 double *keypoint_eq, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(labels && num && K, "null pointer");
    PV_CHECK_ARG(labels_elem_size == 1 || labels_elem_size == 2 || labels_elem_size == 4 || labels_elem_size == 8,
                 "labels_elem_size %d not 1, 2, 4 or 8", labels_elem_size);
    PV_CHECK_ARG(b >= 1 && L >= 1 && L <= 32 && static_cast<long long>(b) * L <= 1024,
                 "instance count %d outside 1..32 or b*L = %lld above 1024", L, static_cast<long long>(b) * L);
    const InstArgs inst{labels, labels_elem_size, num, L};
    if (!keypoints && !points_3d && !weights_2d)
        return refine_poses(nullptr, poses_in, K, 1, verts, faces, nv, nf, b * L, h, w, near_clip, far_clip, rounds,
                            gate, max_points, nullptr, poses_out, info, dist, nullptr, trace, workspace,
                            workspace_bytes, stream, &inst);
    PV_CHECK_ARG(keypoints && points_3d && weights_2d, "null pointer");
    PV_CHECK_ARG(nk >= 4 && nk <= RF_MAX_KP, "keypoint count %d outside [4,%d] (one lane per keypoint)", nk,
                 RF_MAX_KP);
    PV_CHECK_ARG(keypoint_weight >= 0.0 && keypoint_weight < INFINITY, "keypoint_weight must be finite and >= 0 "
                 "(got %g)", keypoint_weight);
    const KpArgs kpa{keypoints, points_3d, weights_2d, nk, keypoint_weight, keypoint_eq};
    return refine_poses(nullptr, poses_in, K, 1, verts, faces, nv, nf, b * L, h, w, near_clip, far_clip, rounds, gate,
                        max_points, &kpa, poses_out, info, dist, cost, trace, workspace, workspace_bytes, stream, &inst);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// Depth-anchored refinement (DESIGN.md §28, pvnet_refine_poses_depth): point-to-plane ICP of the rendered surface
// against the registered depth image, one object per image.  Per round: the render at the current pose (as above);
// k_refine_depth_pairs (one CTA per image) takes every pixel that the render covers, the mask holds and the sensor read,
// whose four 4-neighbours are inside the image, in the mask and read, and whose pair passes the gate; above max_points
// every ceil(n / max_points)-th, by k_refine_boundary's count-then-rank scan.  Each pair holds the model point X (the
// rendered point taken to object space at the round's pose), the observed point Y and the observed normal n from the
// neighbours' cross product.  k_refine_depth_step (one CTA per image) judges the round by the mean |n . (R X + t - Y)|
// and, pairs held fixed, takes RF_GN_STEPS damped Gauss-Newton steps on sum (n . (R X + t - Y))^2.
// oracle/refine_depth_oracle.py restates it; the pair sets, X, Y, n and the mean are bit for bit (one rounded __d*_rn
// per operation), the normal equations to rounding.
namespace {

constexpr int RD_PAIR_THREADS = 256;
constexpr int RD_CHUNK = RD_PAIR_THREADS * RF_PER_THREAD;
constexpr int RD_NCOUNT = 4;                      // per image: pairs kept, pairs, mask pixels, covered pixels

struct DepthIn {
    const void *depth;                            // f32 or u16 [b,h,w]
    int is_u16;
    float scale;                                  // u16 only: Z = fp32(d) * scale, one rounded multiply
};

// The observed depth of pixel p of the image at `base` (an element offset), 0 for no reading (<= 0 or not finite).
__device__ __forceinline__ float observed_depth(const DepthIn &d, long long base, long long p)
{
    const float z = d.is_u16 ? __fmul_rn(static_cast<float>(static_cast<const uint16_t *>(d.depth)[base + p]), d.scale)
                             : static_cast<const float *>(d.depth)[base + p];
    return z > 0.f && z < INFINITY ? z : 0.f;
}

// The normalised ray (xn, yn, 1) of pixel (r, c), k_refine_boundary's back-projection.
__device__ __forceinline__ void pixel_ray(const Cam &cam, int r, int c, double &xn, double &yn)
{
    const double u = c + 0.5, v = r + 0.5;
    yn = dd(ds(v, cam.cy), cam.fy);
    xn = dd(ds(ds(u, cam.cx), dm(cam.s, yn)), cam.fx);
}

// n . (R X + t - Y) at pose P, each operation rounded: Xc = project's R X + t, d = Xc - Y, (n0 d0 + n1 d1) + n2 d2.
// dist (optional): |R X + t - Y| = sqrt((d0 d0 + d1 d1) + d2 d2).
__device__ __forceinline__ double plane_residual(const double *P, const double *X, const double *Y, const double *n,
                                                 double *dist = nullptr)
{
    double d[3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
        d[r] = ds(da(da(da(dm(P[r * 4], X[0]), dm(P[r * 4 + 1], X[1])), dm(P[r * 4 + 2], X[2])), P[r * 4 + 3]), Y[r]);
    if (dist) *dist = __dsqrt_rn(da(da(dm(d[0], d[0]), dm(d[1], d[1])), dm(d[2], d[2])));
    return da(da(dm(n[0], d[0]), dm(n[1], d[1])), dm(n[2], d[2]));
}

// Pairs of one image (grid b): pass 1 counts the pixels that form a pair (and the mask and covered pixels), pass 2
// walks them again in row-major order and keeps rank % stride == 0, stride = ceil(n / max_points), writing each at
// rank / stride.  A pixel forms a pair when it is covered (rendered Z > 0), in the mask, read, its four 4-neighbours
// are inside the image, in the mask and read, |R X + t - Y| <= gate and the residual is a number.  skip_done: images
// already stopped are left alone.
__global__ void __launch_bounds__(RD_PAIR_THREADS)
    k_refine_depth_pairs(const float *__restrict__ rdepth, const uint8_t *__restrict__ mask, DepthIn obs,
                         const double *__restrict__ pose, const float *__restrict__ K, int kstride, int h, int w,
                         int max_points, double gate, int skip_done, const State *__restrict__ state,
                         int32_t *__restrict__ pix, double *__restrict__ pX, double *__restrict__ pY,
                         double *__restrict__ pN, int32_t *__restrict__ counts)
{
    const int img = blockIdx.x;
    if (skip_done && state[img].done) return;
    __shared__ int s_warp[RD_PAIR_THREADS / 32];
    __shared__ int s_total, s_mask, s_cover;
    __shared__ double s_pose[12];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long hw = static_cast<long long>(h) * w, ibase = img * hw;
    const float *ren = rdepth + ibase;
    const uint8_t *msk = mask + ibase;
    if (tid == 0) s_total = s_mask = s_cover = 0;
    if (tid < 12) s_pose[tid] = pose[img * 12 + tid];
    __syncthreads();
    const Cam cam = load_cam(K + static_cast<size_t>(img) * kstride);
    // pixel p as a pair: X (object space, round's pose), Y (observed), n (observed normal, n . Y <= 0)
    auto pair_at = [&](long long p, double (&X)[3], double (&Y)[3], double (&nn)[3]) -> bool {
        const float zr = ren[p];
        if (!(zr > 0.f) || !msk[p]) return false;
        const float zo = observed_depth(obs, ibase, p);
        if (zo == 0.f) return false;
        const int r = static_cast<int>(p / w), c = static_cast<int>(p - static_cast<long long>(r) * w);
        if (r == 0 || r == h - 1 || c == 0 || c == w - 1) return false;
        const long long nb[4] = {p + 1, p - 1, p + w, p - w};
        float zn[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (!msk[nb[q]]) return false;
            zn[q] = observed_depth(obs, ibase, nb[q]);
            if (zn[q] == 0.f) return false;
        }
        double xn, yn;
        pixel_ray(cam, r, c, xn, yn);
        const double Z = zr;
        const double d0 = ds(dm(Z, xn), s_pose[3]), d1 = ds(dm(Z, yn), s_pose[7]), d2 = ds(Z, s_pose[11]);
#pragma unroll
        for (int k = 0; k < 3; ++k) X[k] = da(da(dm(s_pose[k], d0), dm(s_pose[4 + k], d1)), dm(s_pose[8 + k], d2));
        const double zo64 = zo;
        Y[0] = dm(zo64, xn);
        Y[1] = dm(zo64, yn);
        Y[2] = zo64;
        double Q[4][3];                           // the neighbours' observed points: c + 1, c - 1, r + 1, r - 1
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double qx, qy;
            pixel_ray(cam, r + (q == 2) - (q == 3), c + (q == 0) - (q == 1), qx, qy);
            const double z = zn[q];
            Q[q][0] = dm(z, qx);
            Q[q][1] = dm(z, qy);
            Q[q][2] = z;
        }
        double a[3], bv[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            a[k] = ds(Q[0][k], Q[1][k]);
            bv[k] = ds(Q[2][k], Q[3][k]);
        }
        nn[0] = ds(dm(a[1], bv[2]), dm(a[2], bv[1]));
        nn[1] = ds(dm(a[2], bv[0]), dm(a[0], bv[2]));
        nn[2] = ds(dm(a[0], bv[1]), dm(a[1], bv[0]));
        const double len = __dsqrt_rn(da(da(dm(nn[0], nn[0]), dm(nn[1], nn[1])), dm(nn[2], nn[2])));
#pragma unroll
        for (int k = 0; k < 3; ++k) nn[k] = dd(nn[k], len);
        if (da(da(dm(nn[0], Y[0]), dm(nn[1], Y[1])), dm(nn[2], Y[2])) > 0.0)
#pragma unroll
            for (int k = 0; k < 3; ++k) nn[k] = -nn[k];
        double dist;
        const double e = plane_residual(s_pose, X, Y, nn, &dist);
        return dist <= gate && isfinite(e);
    };
    int local = 0, lmask = 0, lcover = 0;
    for (long long base = 0; base < hw; base += RD_CHUNK)
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            if (p >= hw) continue;
            lmask += msk[p] != 0;
            lcover += ren[p] > 0.f;
            double X[3], Y[3], nn[3];
            if (pair_at(p, X, Y, nn)) ++local;
        }
    atomicAdd(&s_total, local);                   // integer sums: the same whatever the order
    atomicAdd(&s_mask, lmask);
    atomicAdd(&s_cover, lcover);
    __syncthreads();
    const int n = s_total;
    const int stride = n > max_points ? (n + max_points - 1) / max_points : 1;
    const size_t o = static_cast<size_t>(img) * max_points;
    int running = 0;                              // pairs in earlier chunks
    for (long long base = 0; base < hw; base += RD_CHUNK) {
        unsigned bits = 0;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            double X[3], Y[3], nn[3];
            if (p < hw && pair_at(p, X, Y, nn)) bits |= 1u << q;
        }
        const int cnt = __popc(bits);
        int incl = cnt;                           // inclusive scan over the warp
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, s);
            if (lane >= s) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int t = lane < RD_PAIR_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, t, s);
                if (lane >= s) t += y;
            }
            if (lane < RD_PAIR_THREADS / 32) s_warp[lane] = t;   // inclusive warp totals
        }
        __syncthreads();
        int rank = running + (warp ? s_warp[warp - 1] : 0) + incl - cnt;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            if (!(bits >> q & 1u)) continue;
            if (rank % stride == 0) {
                const long long p = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
                const size_t j = o + rank / stride;
                double X[3], Y[3], nn[3];
                pair_at(p, X, Y, nn);
                pix[j] = static_cast<int32_t>(p);
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    pX[j * 3 + k] = X[k];
                    pY[j * 3 + k] = Y[k];
                    pN[j * 3 + k] = nn[k];
                }
            }
            ++rank;
        }
        running += s_warp[RD_PAIR_THREADS / 32 - 1];
        __syncthreads();                          // s_warp is rewritten by the next chunk
    }
    if (tid == 0) {
        int32_t *cn = counts + img * RD_NCOUNT;
        cn[0] = n ? (n + stride - 1) / stride : 0;
        cn[1] = n;
        cn[2] = s_mask;
        cn[3] = s_cover;
    }
}

// One CTA per image: evaluation k of the pose (mean |e| over the pairs, pair i on thread i % 256 and block_sum's
// order; accept or undo as k_refine_step does), then, unless k is the last evaluation, RF_GN_STEPS Gauss-Newton steps
// on sum e_i^2, e_i = n_i . (R X_i + t - Y_i), J_i = [(R X_i) x n_i ; n_i].  normal_eq (nullable): the sums of the
// first step of evaluation 0.
__global__ void __launch_bounds__(RF_STEP_THREADS)
    k_refine_depth_step(double *__restrict__ pose, float *__restrict__ pose32, int max_points, int k, int last,
                        State *__restrict__ state, const int32_t *__restrict__ counts, const double *__restrict__ pX,
                        const double *__restrict__ pY, const double *__restrict__ pN, double *__restrict__ normal_eq)
{
    const int img = blockIdx.x;
    State &S = state[img];
    if (S.done) return;
    __shared__ double s_part[RF_STEP_THREADS / 32][RF_NSUM];
    __shared__ double s_sum[RF_NSUM];
    __shared__ double s_pose[12];
    __shared__ int s_go;
    const int32_t *cn = counts + img * RD_NCOUNT;
    const int ns = cn[0];
    const size_t o = static_cast<size_t>(img) * max_points;
    if (threadIdx.x < 12) s_pose[threadIdx.x] = pose[img * 12 + threadIdx.x];
    __syncthreads();
    double acc[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < ns; i += RF_STEP_THREADS) {
        acc[0] += 1.0;
        acc[1] += fabs(plane_residual(s_pose, pX + (o + i) * 3, pY + (o + i) * 3, pN + (o + i) * 3));
    }
    block_sum<2>(acc, reinterpret_cast<double (*)[2]>(&s_part[0][0]), s_sum);
    if (threadIdx.x == 0) {
        const int n = static_cast<int>(s_sum[0]);
        const double m = n ? s_sum[1] / n : NAN;
        bool go = true;
        if (k == 0) {
            int st = 0;
            if (cn[2] == 0) st = RF_NO_CONTOUR;
            else if (cn[3] == 0) st = RF_NO_SILHOUETTE;
            else if (n < RF_MIN_PAIRS) st = RF_FEW_PAIRS;
            if (st) {
                S.status |= st;
                go = false;
            } else {
                S.mean0 = S.mean_after = m;
            }
        } else if (n < RF_MIN_PAIRS || m > S.mean_prev) {
            S.status |= RF_REJECTED;
            for (int q = 0; q < 12; ++q) pose[img * 12 + q] = S.backup[q];
            go = false;
        } else {
            S.mean_after = m;
        }
        if (!go) S.done = 1;
        if (go && !last) {
            S.mean_prev = m;
            for (int q = 0; q < 12; ++q) S.backup[q] = pose[img * 12 + q];
            S.pairs = n;
        }
        s_go = go && !last;
    }
    __syncthreads();
    if (!s_go) return;
    for (int step = 0; step < RF_GN_STEPS; ++step) {
        double v[RF_NSUM];
#pragma unroll
        for (int q = 0; q < RF_NSUM; ++q) v[q] = 0.0;
        for (int i = threadIdx.x; i < ns; i += RF_STEP_THREADS) {
            const double *X = pX + (o + i) * 3, *Y = pY + (o + i) * 3, *nn = pN + (o + i) * 3;
            double p[3], d[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                p[r] = s_pose[r * 4] * X[0] + s_pose[r * 4 + 1] * X[1] + s_pose[r * 4 + 2] * X[2];
                d[r] = p[r] + s_pose[r * 4 + 3] - Y[r];
            }
            const double e = nn[0] * d[0] + nn[1] * d[1] + nn[2] * d[2];
            // d e / d(dw) for R <- exp(dw) R is (R X) x n; d e / d(dt) is n
            const double J[6] = {p[1] * nn[2] - p[2] * nn[1], p[2] * nn[0] - p[0] * nn[2], p[0] * nn[1] - p[1] * nn[0],
                                 nn[0], nn[1], nn[2]};
            int q = 0;
#pragma unroll
            for (int r = 0; r < 6; ++r)
#pragma unroll
                for (int c = r; c < 6; ++c) v[q++] += J[r] * J[c];
#pragma unroll
            for (int r = 0; r < 6; ++r) v[21 + r] += J[r] * e;
        }
        block_sum<RF_NSUM>(v, s_part, s_sum);
        if (threadIdx.x == 0) {
            if (normal_eq && k == 0 && step == 0)
                for (int q = 0; q < RF_NSUM; ++q) normal_eq[img * RF_NSUM + q] = s_sum[q];
            double x[6];
            if (!damped_solve(s_sum, x)) {
                S.status |= RF_SINGULAR;
                S.done = 1;
                for (int q = 0; q < 12; ++q) s_pose[q] = S.backup[q];
                s_go = 0;
            } else {
                double E[9], R[9];
                so3_exp(x[0], x[1], x[2], E);
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c)
                        R[r * 3 + c] = E[r * 3] * s_pose[c] + E[r * 3 + 1] * s_pose[4 + c] + E[r * 3 + 2] * s_pose[8 + c];
                for (int r = 0; r < 3; ++r) {
                    for (int c = 0; c < 3; ++c) s_pose[r * 4 + c] = R[r * 3 + c];
                    s_pose[r * 4 + 3] += x[3 + r];
                }
            }
        }
        __syncthreads();
        if (!s_go) break;
    }
    if (threadIdx.x < 12) {
        pose[img * 12 + threadIdx.x] = s_pose[threadIdx.x];
        pose32[img * 12 + threadIdx.x] = __double2float_rn(s_pose[threadIdx.x]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Depth-anchored refinement per instance (DESIGN.md §31, pvnet_refine_poses_depth_instances): virtual image
// v = bi * L + j is instance j of image bi's label map, and row v is k_refine_depth_pairs's image v with the mask
// labels[bi] == j+1.  The labels do not change between rounds, so each instance's bounding box is found once per call
// and the pair scan walks only the box.

constexpr int RD_BOX_THREADS = 1024;

// Bounding box of each label 1..L of image blockIdx.x (grid b): boxes[bi * L + j] = (r0, c0, r1, c1), inclusive;
// r1 < r0 when label j+1 has no pixel.  One warp per row; the lanes holding one label are grouped by
// __match_any_sync and their lowest lane folds the group's column range into shared memory with integer atomics.
template <typename T>
__global__ void __launch_bounds__(RD_BOX_THREADS)
    k_refine_label_boxes(const T *__restrict__ labels, int L, int h, int w, int4 *__restrict__ boxes)
{
    __shared__ int s_box[32][4];
    const int bi = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < 32) {
        s_box[tid][0] = s_box[tid][1] = INT_MAX;
        s_box[tid][2] = s_box[tid][3] = -1;
    }
    __syncthreads();
    const T *lab = labels + static_cast<long long>(bi) * h * w;
    for (int r = warp; r < h; r += RD_BOX_THREADS / 32)
        for (int c0 = 0; c0 < w; c0 += 32) {
            const int c = c0 + lane;
            const long long v = c < w ? static_cast<long long>(lab[static_cast<long long>(r) * w + c]) : 0;
            const int key = v >= 1 && v <= L ? static_cast<int>(v) : 0;
            const unsigned grp = __match_any_sync(0xffffffffu, key);
            const int cmin = __reduce_min_sync(grp, c), cmax = __reduce_max_sync(grp, c);
            if (key && lane == __ffs(grp) - 1) {
                atomicMin(&s_box[key - 1][0], r);
                atomicMin(&s_box[key - 1][1], cmin);
                atomicMax(&s_box[key - 1][2], r);
                atomicMax(&s_box[key - 1][3], cmax);
            }
        }
    __syncthreads();
    if (tid < L) boxes[bi * L + tid] = make_int4(s_box[tid][0], s_box[tid][1], s_box[tid][2], s_box[tid][3]);
}

// k_refine_depth_pairs for virtual image img (grid b * L), with "in the mask" read as "carries label j+1" (labels at
// their own width, compared as integers).  Every pixel that can pair carries label j+1, so both passes walk only the
// instance's box, row-major: the pairs come in the image's row-major order and the ranks, stride and outputs are the
// whole-frame scan's.  The mask count is the box's; the covered count (counts[3], the round-0 status gate) is taken
// over the whole frame when count_cover is set (round 0) and left as it is otherwise.  Rows already done are skipped
// from round 0 on (the absent rows: their counts are zeroed in round 0, so a trace shows them empty).
template <typename T>
__global__ void __launch_bounds__(RD_PAIR_THREADS, 1)
    k_refine_depth_pairs_instances(const float *__restrict__ rdepth, const T *__restrict__ labels, int L,
                                   const int4 *__restrict__ boxes, DepthIn obs, const double *__restrict__ pose,
                                   const float *__restrict__ K, int h, int w, int max_points, double gate,
                                   int count_cover, const State *__restrict__ state, int32_t *__restrict__ pix,
                                   double *__restrict__ pX, double *__restrict__ pY, double *__restrict__ pN,
                                   int32_t *__restrict__ counts)
{
    const int img = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int32_t *cn = counts + img * RD_NCOUNT;
    if (state[img].done) {
        if (count_cover && tid < RD_NCOUNT) cn[tid] = 0;
        return;
    }
    __shared__ int s_warp[RD_PAIR_THREADS / 32];
    __shared__ int s_total, s_mask, s_cover;
    __shared__ double s_pose[12];
    const long long hw = static_cast<long long>(h) * w;
    const int bi = img / L;
    const long long own = img - bi * L + 1, ibase = bi * hw;
    const float *ren = rdepth + img * hw;
    const T *lab = labels + ibase;
    const int4 box = boxes[img];
    const int bw = box.w - box.y + 1;
    const long long nbox = box.z >= box.x ? static_cast<long long>(box.z - box.x + 1) * bw : 0;
    if (tid == 0) s_total = s_mask = s_cover = 0;
    if (tid < 12) s_pose[tid] = pose[img * 12 + tid];
    __syncthreads();
    const Cam cam = load_cam(K + static_cast<size_t>(img) * 9);
    auto mine = [&](long long p) -> bool { return static_cast<long long>(lab[p]) == own; };
    // box position q -> image pixel
    auto at = [&](long long q) -> long long { return (box.x + q / bw) * w + box.y + q % bw; };
    // k_refine_depth_pairs's pair_at with mine(.) for the mask
    auto pair_at = [&](long long p, double (&X)[3], double (&Y)[3], double (&nn)[3]) -> bool {
        const float zr = ren[p];
        if (!(zr > 0.f) || !mine(p)) return false;
        const float zo = observed_depth(obs, ibase, p);
        if (zo == 0.f) return false;
        const int r = static_cast<int>(p / w), c = static_cast<int>(p - static_cast<long long>(r) * w);
        if (r == 0 || r == h - 1 || c == 0 || c == w - 1) return false;
        const long long nb[4] = {p + 1, p - 1, p + w, p - w};
        float zn[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (!mine(nb[q])) return false;
            zn[q] = observed_depth(obs, ibase, nb[q]);
            if (zn[q] == 0.f) return false;
        }
        double xn, yn;
        pixel_ray(cam, r, c, xn, yn);
        const double Z = zr;
        const double d0 = ds(dm(Z, xn), s_pose[3]), d1 = ds(dm(Z, yn), s_pose[7]), d2 = ds(Z, s_pose[11]);
#pragma unroll
        for (int k = 0; k < 3; ++k) X[k] = da(da(dm(s_pose[k], d0), dm(s_pose[4 + k], d1)), dm(s_pose[8 + k], d2));
        const double zo64 = zo;
        Y[0] = dm(zo64, xn);
        Y[1] = dm(zo64, yn);
        Y[2] = zo64;
        double Q[4][3];                           // the neighbours' observed points: c + 1, c - 1, r + 1, r - 1
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double qx, qy;
            pixel_ray(cam, r + (q == 2) - (q == 3), c + (q == 0) - (q == 1), qx, qy);
            const double z = zn[q];
            Q[q][0] = dm(z, qx);
            Q[q][1] = dm(z, qy);
            Q[q][2] = z;
        }
        double a[3], bv[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            a[k] = ds(Q[0][k], Q[1][k]);
            bv[k] = ds(Q[2][k], Q[3][k]);
        }
        nn[0] = ds(dm(a[1], bv[2]), dm(a[2], bv[1]));
        nn[1] = ds(dm(a[2], bv[0]), dm(a[0], bv[2]));
        nn[2] = ds(dm(a[0], bv[1]), dm(a[1], bv[0]));
        const double len = __dsqrt_rn(da(da(dm(nn[0], nn[0]), dm(nn[1], nn[1])), dm(nn[2], nn[2])));
#pragma unroll
        for (int k = 0; k < 3; ++k) nn[k] = dd(nn[k], len);
        if (da(da(dm(nn[0], Y[0]), dm(nn[1], Y[1])), dm(nn[2], Y[2])) > 0.0)
#pragma unroll
            for (int k = 0; k < 3; ++k) nn[k] = -nn[k];
        double dist;
        const double e = plane_residual(s_pose, X, Y, nn, &dist);
        return dist <= gate && isfinite(e);
    };
    int local = 0, lmask = 0, lcover = 0;
    if (count_cover)
        for (long long p = tid; p < hw; p += RD_PAIR_THREADS) lcover += ren[p] > 0.f;
    for (long long base = 0; base < nbox; base += RD_CHUNK)
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long bq = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            if (bq >= nbox) continue;
            const long long p = at(bq);
            lmask += mine(p);
            double X[3], Y[3], nn[3];
            if (pair_at(p, X, Y, nn)) ++local;
        }
    atomicAdd(&s_total, local);                   // integer sums: the same whatever the order
    atomicAdd(&s_mask, lmask);
    atomicAdd(&s_cover, lcover);
    __syncthreads();
    const int n = s_total;
    const int stride = n > max_points ? (n + max_points - 1) / max_points : 1;
    const size_t o = static_cast<size_t>(img) * max_points;
    int running = 0;                              // pairs in earlier chunks
    for (long long base = 0; base < nbox; base += RD_CHUNK) {
        unsigned bits = 0;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            const long long bq = base + static_cast<long long>(tid) * RF_PER_THREAD + q;
            double X[3], Y[3], nn[3];
            if (bq < nbox && pair_at(at(bq), X, Y, nn)) bits |= 1u << q;
        }
        const int cnt = __popc(bits);
        int incl = cnt;                           // inclusive scan over the warp
#pragma unroll
        for (int s = 1; s < 32; s <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, s);
            if (lane >= s) incl += y;
        }
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int t = lane < RD_PAIR_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
            for (int s = 1; s < 32; s <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, t, s);
                if (lane >= s) t += y;
            }
            if (lane < RD_PAIR_THREADS / 32) s_warp[lane] = t;   // inclusive warp totals
        }
        __syncthreads();
        int rank = running + (warp ? s_warp[warp - 1] : 0) + incl - cnt;
        for (int q = 0; q < RF_PER_THREAD; ++q) {
            if (!(bits >> q & 1u)) continue;
            if (rank % stride == 0) {
                const long long p = at(base + static_cast<long long>(tid) * RF_PER_THREAD + q);
                const size_t j = o + rank / stride;
                double X[3], Y[3], nn[3];
                pair_at(p, X, Y, nn);
                pix[j] = static_cast<int32_t>(p);
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    pX[j * 3 + k] = X[k];
                    pY[j * 3 + k] = Y[k];
                    pN[j * 3 + k] = nn[k];
                }
            }
            ++rank;
        }
        running += s_warp[RD_PAIR_THREADS / 32 - 1];
        __syncthreads();                          // s_warp is rewritten by the next chunk
    }
    if (tid == 0) {
        cn[0] = n ? (n + stride - 1) / stride : 0;
        cn[1] = n;
        cn[2] = s_mask;
        if (count_cover) cn[3] = s_cover;
    }
}

struct DepthLayout {
    unsigned long long *keys;
    float *depth, *pose32;
    int32_t *pix, *counts;
    double *X, *Y, *N;
    State *state;
    size_t bytes;
};

DepthLayout carve_depth(void *base, int b, int h, int w, int max_points)
{
    pvnet::Carver cv(base);
    DepthLayout L;
    const size_t npix = static_cast<size_t>(b) * h * w, np = static_cast<size_t>(b) * max_points;
    L.keys = cv.take<unsigned long long>(npix);
    L.depth = cv.take<float>(npix);
    L.pose32 = cv.take<float>(static_cast<size_t>(b) * 12);
    L.pix = cv.take<int32_t>(np);
    L.X = cv.take<double>(np * 3);
    L.Y = cv.take<double>(np * 3);
    L.N = cv.take<double>(np * 3);
    L.counts = cv.take<int32_t>(static_cast<size_t>(b) * RD_NCOUNT);
    L.state = cv.take<State>(b);
    L.bytes = pvnet::align_up(cv.off, 256);
    return L;
}

}  // namespace

extern "C" {

int pvnet_refine_depth_workspace_bytes(int b, int h, int w, int max_points, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && max_points >= 1, "non-positive dimension (b=%d, h=%d, w=%d, "
                 "max_points=%d)", b, h, w, max_points);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = carve_depth(nullptr, b, h, w, max_points).bytes;
    return PVNET_OK;
}

}  // extern "C"

namespace {

// Both depth entry points: inst null reads mask [b,h,w] with K shared or per image (k_per_image); inst non-null reads
// its label map (mask unused), b counts the virtual images, K is per virtual image and the instances' boxes follow
// the §28 layout in the workspace.
int refine_depth(const uint8_t *mask, const void *depth, int depth_is_u16, float depth_scale, const double *poses_in,
                 const float *K, int k_per_image, const float *verts, const int32_t *faces, int nv, int nf, int b, int h,
                 int w, float near_clip, float far_clip, int rounds, double gate, int max_points, double *poses_out,
                 int32_t *info, double *dist, const pvnet_refine_depth_trace_t *trace, void *workspace,
                 size_t workspace_bytes, pvnet_stream_t stream, const InstArgs *inst = nullptr)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && nv >= 0 && nf >= 0, "bad dimension (b=%d, h=%d, w=%d, nv=%d, nf=%d)",
                 b, h, w, nv, nf);
    PV_CHECK_ARG(static_cast<long long>(h) * w <= INT32_MAX, "image %dx%d too large", h, w);
    PV_CHECK_ARG(max_points >= 1 && static_cast<long long>(b) * max_points <= INT32_MAX / 9,
                 "max_points %d outside 1..%d for b = %d", max_points, INT32_MAX / 9 / b, b);
    PV_CHECK_ARG(rounds >= 0, "rounds must be >= 0 (got %d)", rounds);
    PV_CHECK_ARG(gate > 0.0 && gate < INFINITY, "gate must be positive and finite (got %g)", gate);
    PV_CHECK_ARG(!depth_is_u16 || (depth_scale > 0.f && depth_scale < INFINITY),
                 "depth_scale must be positive and finite (got %g)", depth_scale);
    PV_CHECK_ARG((mask || inst) && depth && poses_in && K && poses_out && (nf == 0 || faces) && (nv == 0 || verts),
                 "null pointer");
    size_t need = 0;
    pvnet_refine_depth_workspace_bytes(b, h, w, max_points, &need);
    int4 *boxes = nullptr;
    if (inst) {
        boxes = reinterpret_cast<int4 *>(static_cast<char *>(workspace) + need);
        need += pvnet::align_up(static_cast<size_t>(b) * sizeof(int4), 256);
    }
    PV_CHECK_ARG(workspace && workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);
    const DepthLayout L = carve_depth(workspace, b, h, w, max_points);
    size_t render_need = 0;
    pvnet_render_workspace_bytes(b, h, w, &render_need);
    const cudaStream_t st = (cudaStream_t)stream;
    const int kstride = k_per_image ? 9 : 0;
    const DepthIn obs{depth, depth_is_u16 ? 1 : 0, depth_is_u16 ? depth_scale : 1.f};
    k_refine_init<<<(b + 127) / 128, 128, 0, st>>>(poses_in, poses_out, L.pose32, L.state, b);
    PV_LAUNCHED("k_refine_init");
    if (inst) {
        k_refine_absent<<<(b + 127) / 128, 128, 0, st>>>(inst->num, inst->L, b, L.state, L.pose32);
        PV_LAUNCHED("k_refine_absent");
#define PV_LABEL_BOXES(T)                                                                                              \
    k_refine_label_boxes<T><<<b / inst->L, RD_BOX_THREADS, 0, st>>>(static_cast<const T *>(inst->labels), inst->L, h, \
                                                                    w, boxes)
        switch (inst->esz) {
        case 1: PV_LABEL_BOXES(unsigned char); break;
        case 2: PV_LABEL_BOXES(short); break;
        case 4: PV_LABEL_BOXES(int); break;
        default: PV_LABEL_BOXES(long long); break;
        }
#undef PV_LABEL_BOXES
        PV_LAUNCHED("k_refine_label_boxes");
    }
    for (int k = 0; k <= rounds; ++k) {
        const int rc = pvnet_render_mesh(verts, faces, nullptr, nv, nf, L.pose32, K, k_per_image, b, h, w, near_clip,
                                         far_clip, 0.5f, nullptr, L.depth, nullptr, L.keys, render_need, stream);
        if (rc != PVNET_OK) return rc;
        if (!inst) {
            k_refine_depth_pairs<<<b, RD_PAIR_THREADS, 0, st>>>(L.depth, mask, obs, poses_out, K, kstride, h, w,
                                                                max_points, gate, k > 0, L.state, L.pix, L.X, L.Y, L.N,
                                                                L.counts);
        } else {
#define PV_DEPTH_PAIRS_INSTANCES(T)                                                                                    \
    k_refine_depth_pairs_instances<T><<<b, RD_PAIR_THREADS, 0, st>>>(                                                  \
        L.depth, static_cast<const T *>(inst->labels), inst->L, boxes, obs, poses_out, K, h, w, max_points, gate,      \
        k == 0, L.state, L.pix, L.X, L.Y, L.N, L.counts)
            switch (inst->esz) {
            case 1: PV_DEPTH_PAIRS_INSTANCES(unsigned char); break;
            case 2: PV_DEPTH_PAIRS_INSTANCES(short); break;
            case 4: PV_DEPTH_PAIRS_INSTANCES(int); break;
            default: PV_DEPTH_PAIRS_INSTANCES(long long); break;
            }
#undef PV_DEPTH_PAIRS_INSTANCES
        }
        PV_LAUNCHED("k_refine_depth_pairs");
        if (k == 0 && trace) {
            const size_t np = static_cast<size_t>(b) * max_points;
            if (trace->pair_idx) PV_CUDA(cudaMemcpyAsync(trace->pair_idx, L.pix, np * 4, cudaMemcpyDeviceToDevice, st));
            if (trace->counts)
                PV_CUDA(cudaMemcpyAsync(trace->counts, L.counts, static_cast<size_t>(b) * RD_NCOUNT * 4,
                                        cudaMemcpyDeviceToDevice, st));
            if (trace->X) PV_CUDA(cudaMemcpyAsync(trace->X, L.X, np * 24, cudaMemcpyDeviceToDevice, st));
            if (trace->Y) PV_CUDA(cudaMemcpyAsync(trace->Y, L.Y, np * 24, cudaMemcpyDeviceToDevice, st));
            if (trace->n) PV_CUDA(cudaMemcpyAsync(trace->n, L.N, np * 24, cudaMemcpyDeviceToDevice, st));
        }
        k_refine_depth_step<<<b, RF_STEP_THREADS, 0, st>>>(poses_out, L.pose32, max_points, k, k == rounds, L.state,
                                                           L.counts, L.X, L.Y, L.N,
                                                           trace ? trace->normal_eq : nullptr);
        PV_LAUNCHED("k_refine_depth_step");
    }
    if (info || dist) {
        k_refine_finish<<<(b + 127) / 128, 128, 0, st>>>(L.state, b, info, dist, nullptr);
        PV_LAUNCHED("k_refine_finish");
    }
    return PVNET_OK;
}

}  // namespace

extern "C" {

int pvnet_refine_poses_depth(const uint8_t *mask, const void *depth, int depth_is_u16, float depth_scale,
                             const double *poses_in, const float *K, int k_per_image, const float *verts,
                             const int32_t *faces, int nv, int nf, int b, int h, int w, float near_clip,
                             float far_clip, int rounds, double gate, int max_points, double *poses_out, int32_t *info,
                             double *dist, const pvnet_refine_depth_trace_t *trace, void *workspace,
                             size_t workspace_bytes, pvnet_stream_t stream)
{
    return refine_depth(mask, depth, depth_is_u16, depth_scale, poses_in, K, k_per_image, verts, faces, nv, nf, b, h,
                        w, near_clip, far_clip, rounds, gate, max_points, poses_out, info, dist, trace, workspace,
                        workspace_bytes, stream);
}

int pvnet_refine_depth_instances_workspace_bytes(int b, int L, int h, int w, int max_points, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && L >= 1 && L <= 32 && static_cast<long long>(b) * L <= 1024,
                 "instance count %d outside 1..32 or b*L = %lld above 1024", L, static_cast<long long>(b) * L);
    PV_CHECK_ARG(h >= 1 && w >= 1 && max_points >= 1, "non-positive dimension (h=%d, w=%d, max_points=%d)", h, w,
                 max_points);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = carve_depth(nullptr, b * L, h, w, max_points).bytes +
             pvnet::align_up(static_cast<size_t>(b) * L * sizeof(int4), 256);
    return PVNET_OK;
}

int pvnet_refine_poses_depth_instances(const void *labels, int labels_elem_size, const int32_t *num, int L,
                                       const void *depth, int depth_is_u16, float depth_scale, const double *poses_in,
                                       const float *K, const float *verts, const int32_t *faces, int nv, int nf, int b,
                                       int h, int w, float near_clip, float far_clip, int rounds, double gate,
                                       int max_points, double *poses_out, int32_t *info, double *dist,
                                       const pvnet_refine_depth_trace_t *trace, void *workspace,
                                       size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(labels && num && K, "null pointer");
    PV_CHECK_ARG(labels_elem_size == 1 || labels_elem_size == 2 || labels_elem_size == 4 || labels_elem_size == 8,
                 "labels_elem_size %d not 1, 2, 4 or 8", labels_elem_size);
    PV_CHECK_ARG(b >= 1 && L >= 1 && L <= 32 && static_cast<long long>(b) * L <= 1024,
                 "instance count %d outside 1..32 or b*L = %lld above 1024", L, static_cast<long long>(b) * L);
    const InstArgs inst{labels, labels_elem_size, num, L};
    return refine_depth(nullptr, depth, depth_is_u16, depth_scale, poses_in, K, 1, verts, faces, nv, nf, b * L, h, w,
                        near_clip, far_clip, rounds, gate, max_points, poses_out, info, dist, trace, workspace,
                        workspace_bytes, stream, &inst);
}

}  // extern "C"
