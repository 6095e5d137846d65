// extend.cu -- the dataset tooling of the reference's lib/utils/extend_utils on the device: farthest point sampling
// (the keypoints the network votes for) and binary mesh rasterisation.
//
// Reference (DESIGN.md §11):
//   lib/utils/extend_utils/src/farthest_point_sampling.cpp   farthest_point_sampling[_init_center] (single thread)
//   lib/utils/extend_utils/src/mesh_rasterization.cpp        mesh_binary_rasterization (single thread)
// Both are compiled there with -O2 and no FMA contraction, so every operation below is one rounded __f*_rn
// intrinsic, in the source's order, and the indices and masks are bit-identical to the reference's binary.
//
// Farthest point sampling: one thread-block cluster per cloud.  The cluster's CTAs own contiguous slices of the
// cloud in index order; a resident slice keeps x, y, z and min_dist (SoA) in shared memory for all sn rounds, and
// the selection bit is folded into min_dist (a selected point holds -1, which no distance replaces and no argmax
// takes).  Per round every thread updates its points and keeps its best 64-bit key
//     key = (d > 0) ? bits(d) << 32 | ~idx : 0          (d > 0 is false for NaN, 0 and the selected -1)
// -- non-negative floats order like their bit patterns, so the largest distance wins and the lowest index breaks
// ties, as the reference's strict `>` scan from (0, 0.f) does -- reduces it over the CTA into one of two
// alternating slots, and passes one cluster barrier.  Every CTA then reads all slots of the round over DSMEM and
// takes the same maximum, so all agree on the winner without a second barrier; a zero key means index 0, the
// reference's result when no unselected point has min_dist > 0.  The winner's coordinates come from its owner's
// shared memory.  Clouds above FPS_MAX_CLUSTER * FPS_SLICE points run the same kernel with the slice re-read from
// global memory (L2) every round and min_dist in the caller's workspace.
//
// Rasterisation: the mask is zeroed, then a warp takes a triangle and its lanes walk the clamped box, storing 1
// into every covered byte (the reference's result does not depend on the triangle order, so racing stores of 1
// are exact).  Boxes above RS_BIG pixels are deferred to the whole CTA, which splits their rows over its warps.
#include "common.cuh"
#include "ptx.cuh"

#include <cfloat>

namespace {

constexpr int FPS_THREADS = 512;
constexpr int FPS_WARPS = FPS_THREADS / 32;
constexpr int FPS_SLICE = 14336;                 // resident points per CTA: 16 B each, 224 KB of shared memory
constexpr int FPS_MAX_CLUSTER = 8;               // portable cluster size
constexpr int FPS_CTA_POINTS = 4096;             // below this many points per CTA, a smaller cluster is used
constexpr float FPS_SELECTED = -1.f;

constexpr int RS_WARPS = 8;
constexpr int RS_THREADS = RS_WARPS * 32;
constexpr int RS_BIG = 1024;                     // box pixels above which a triangle is shared by the CTA's warps

// farthest_point_sampling.cpp Vec3::operator-, squared_norm: ((dx*dx) + (dy*dy)) + (dz*dz), each op rounded once
__device__ __forceinline__ float fps_dist(float x, float y, float z, float cx, float cy, float cz)
{
    const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy), dz = __fsub_rn(z, cz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ unsigned long long fps_key(float d, int i)
{
    return d > 0.f ? (static_cast<unsigned long long>(__float_as_uint(d)) << 32) | static_cast<uint32_t>(~i) : 0ull;
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long k)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xffffffffu, k, o);
        k = v > k ? v : k;
    }
    return k;
}

// The cluster-wide argmax of one round: the CTA's key goes to slot[buf], one cluster barrier, then every warp
// of every CTA reads the cluster's slots in rank order.  slot[buf] is written again two rounds later, after the
// next barrier, by which time every peer has read it.
__device__ __forceinline__ int fps_cluster_argmax(unsigned long long key, unsigned long long *s_wkey,
                                                  unsigned long long *slot, int csize)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    key = warp_max_u64(key);
    if (lane == 0) s_wkey[warp] = key;
    __syncthreads();
    if (warp == 0) {
        unsigned long long k = lane < FPS_WARPS ? s_wkey[lane] : 0ull;
        k = warp_max_u64(k);
        if (lane == 0) *slot = k;
    }
    ptx::cluster_sync();
    unsigned long long k = lane < csize ? ptx::ld_cluster_u64(ptx::mapa(slot, lane)) : 0ull;
    k = warp_max_u64(k);
    return k ? static_cast<int>(~static_cast<uint32_t>(k)) : 0;
}

// grid: b clusters of csize CTAs.  resident: the slice lives in shared memory (4 * slice floats of dynamic
// smem); otherwise coordinates are read from pts and min_dist lives in gdist [b,pn].
__global__ void __launch_bounds__(FPS_THREADS, 1)
    k_farthest_point_sampling(const float *__restrict__ pts, const int32_t *__restrict__ start, int pn, int sn,
                              int slice, int resident, float *__restrict__ gdist, int32_t *__restrict__ idxs)
{
    extern __shared__ float fps_smem[];          // resident: x [slice], y [slice], z [slice], min_dist [slice]
    __shared__ unsigned long long s_wkey[FPS_WARPS];
    __shared__ unsigned long long s_slot[2];
    __shared__ float s_wbox[FPS_WARPS][6];
    __shared__ float s_box[6];                   // this CTA's (max x, y, z, min x, y, z)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = ptx::cluster_ctarank();
    uint32_t nct;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(nct));
    const int C = static_cast<int>(nct);
    const int cloud = blockIdx.x / C;
    const float *P = pts + static_cast<size_t>(cloud) * pn * 3;
    const int lo = static_cast<int>(rank) * slice;
    const int n = max(0, min(pn - lo, slice));
    float *sx = fps_smem, *sy = sx + slice, *sz = sy + slice;
    float *D = resident ? sz + slice : gdist + static_cast<size_t>(cloud) * pn + lo;

    // load the slice (resident) and fold this CTA's bounding box; NaN never enters (a NaN compare is false)
    float bx = -FLT_MAX, by = -FLT_MAX, bz = -FLT_MAX, mx = FLT_MAX, my = FLT_MAX, mz = FLT_MAX;
    for (int j = tid; j < n; j += FPS_THREADS) {
        const float x = P[(size_t)(lo + j) * 3], y = P[(size_t)(lo + j) * 3 + 1], z = P[(size_t)(lo + j) * 3 + 2];
        if (resident) {
            sx[j] = x;
            sy[j] = y;
            sz[j] = z;
        }
        if (start == nullptr) {
            bx = (bx < x) ? x : bx;
            by = (by < y) ? y : by;
            bz = (bz < z) ? z : bz;
            mx = (x < mx) ? x : mx;
            my = (y < my) ? y : my;
            mz = (z < mz) ? z : mz;
        } else {
            D[j] = FLT_MAX;
        }
    }
    int cur;
    if (start == nullptr) {
        // farthest_point_sampling.cpp:124-134.  The fold keeps max/min in index order; the parallel fold below gives
        // the same values up to the sign of a zero, which (max + min) and the squares below cannot see.
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            bx = fmaxf(bx, __shfl_xor_sync(0xffffffffu, bx, o));
            by = fmaxf(by, __shfl_xor_sync(0xffffffffu, by, o));
            bz = fmaxf(bz, __shfl_xor_sync(0xffffffffu, bz, o));
            mx = fminf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            my = fminf(my, __shfl_xor_sync(0xffffffffu, my, o));
            mz = fminf(mz, __shfl_xor_sync(0xffffffffu, mz, o));
        }
        if (lane == 0) {
            s_wbox[warp][0] = bx;
            s_wbox[warp][1] = by;
            s_wbox[warp][2] = bz;
            s_wbox[warp][3] = mx;
            s_wbox[warp][4] = my;
            s_wbox[warp][5] = mz;
        }
        __syncthreads();
        if (tid < 6) {
            float v = s_wbox[0][tid];
            for (int w = 1; w < FPS_WARPS; ++w) v = tid < 3 ? fmaxf(v, s_wbox[w][tid]) : fminf(v, s_wbox[w][tid]);
            s_box[tid] = v;
        }
        ptx::cluster_sync();                     // also publishes the resident slices to the cluster
        float box[6];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            float v = ptx::ld_cluster_f32(ptx::mapa(&s_box[k], 0));
            for (int r = 1; r < C; ++r) {
                const float u = ptx::ld_cluster_f32(ptx::mapa(&s_box[k], r));
                v = k < 3 ? fmaxf(v, u) : fminf(v, u);
            }
            box[k] = v;
        }
        // center = (max + min) / 2.f, which Vec3::operator/ computes as * (1.f / 2.f)
        const float cx = __fmul_rn(__fadd_rn(box[0], box[3]), 0.5f);
        const float cy = __fmul_rn(__fadd_rn(box[1], box[4]), 0.5f);
        const float cz = __fmul_rn(__fadd_rn(box[2], box[5]), 0.5f);
        unsigned long long key = 0ull;
        for (int j = tid; j < n; j += FPS_THREADS) {
            float x, y, z;
            if (resident) {
                x = sx[j];
                y = sy[j];
                z = sz[j];
            } else {
                x = P[(size_t)(lo + j) * 3];
                y = P[(size_t)(lo + j) * 3 + 1];
                z = P[(size_t)(lo + j) * 3 + 2];
            }
            const float d = fps_dist(x, y, z, cx, cy, cz);
            const float m = (FLT_MAX < d) ? FLT_MAX : d;     // std::min(d, FLT_MAX): NaN stays, inf -> FLT_MAX
            D[j] = m;
            const unsigned long long k = fps_key(m, lo + j);
            key = k > key ? k : key;
        }
        cur = fps_cluster_argmax(key, s_wkey, &s_slot[1], C);
    } else {
        ptx::cluster_sync();                     // the resident slices are visible to the cluster
        const int s = start[cloud] % pn;         // the reference's rand() % pn, with the draw as an input
        cur = s < 0 ? s + pn : s;
    }

    int32_t *out = idxs + static_cast<size_t>(cloud) * sn;
    for (int r = 0; r < sn; ++r) {
        if (rank == 0 && tid == 0) out[r] = cur;
        if (r == sn - 1) break;
        const int owner = cur / slice, oj = cur - owner * slice;
        float cx, cy, cz;
        if (resident) {
            cx = ptx::ld_cluster_f32(ptx::mapa(sx + oj, owner));
            cy = ptx::ld_cluster_f32(ptx::mapa(sy + oj, owner));
            cz = ptx::ld_cluster_f32(ptx::mapa(sz + oj, owner));
        } else {
            cx = P[(size_t)cur * 3];
            cy = P[(size_t)cur * 3 + 1];
            cz = P[(size_t)cur * 3 + 2];
        }
        const int cj = cur - lo;                 // cur's slot in this slice, if it is ours
        unsigned long long key = 0ull;
        for (int j = tid; j < n; j += FPS_THREADS) {
            float x, y, z;
            if (resident) {
                x = sx[j];
                y = sy[j];
                z = sz[j];
            } else {
                x = P[(size_t)(lo + j) * 3];
                y = P[(size_t)(lo + j) * 3 + 1];
                z = P[(size_t)(lo + j) * 3 + 2];
            }
            // update_min_dist: a selected point keeps -1 (no distance is below it); cur joins them
            const float d = fps_dist(x, y, z, cx, cy, cz);
            float m = D[j];
            if (j == cj)
                m = FPS_SELECTED;
            else if (d < m)
                m = d;
            D[j] = m;
            const unsigned long long k = fps_key(m, lo + j);
            key = k > key ? k : key;
        }
        cur = fps_cluster_argmax(key, s_wkey, &s_slot[r & 1], C);
    }
    ptx::cluster_sync();                         // no CTA leaves while a peer may still read its shared memory
}

// ------------------------------------------------------------------------------------------------ rasterisation
struct Tri {
    float ax[3], ay[3], nx[3], ny[3], v0[3];     // per edge: origin, normal (-dy, dx), the opposite vertex's side
    int bx, ex, by, ey;                          // inclusive pixel box
};

// mesh_rasterization.cpp:58-67.  false: the box is empty, or int() of it would be undefined in the reference
// (a bound at or beyond 2^31 in magnitude), where no in-range pixel can be covered.
__device__ __forceinline__ bool tri_setup(const float *__restrict__ t, int h, int w, Tri &T)
{
    const float x0 = t[0], y0 = t[1], x1 = t[2], y1 = t[3], x2 = t[4], y2 = t[5];
    // std::min({a,b,c}) / std::max({a,b,c}) (min_element / max_element: first extreme, `<` only)
    float minx = x0, maxx = x0, miny = y0, maxy = y0;
    if (x1 < minx) minx = x1;
    if (x2 < minx) minx = x2;
    if (maxx < x1) maxx = x1;
    if (maxx < x2) maxx = x2;
    if (y1 < miny) miny = y1;
    if (y2 < miny) miny = y2;
    if (maxy < y1) maxy = y1;
    if (maxy < y2) maxy = y2;
    // std::max(0.f, m) = (0.f < m) ? m : 0.f;  std::min(float(w-2), m) = (m < float(w-2)) ? m : float(w-2)
    minx = (0.f < minx) ? minx : 0.f;
    miny = (0.f < miny) ? miny : 0.f;
    const float wl = static_cast<float>(w - 2), hl = static_cast<float>(h - 2);
    maxx = (maxx < wl) ? maxx : wl;
    maxy = (maxy < hl) ? maxy : hl;
    const float ex = __fadd_rn(maxx, 1.f), ey = __fadd_rn(maxy, 1.f);
    if (!(minx < 2147483648.f) || !(miny < 2147483648.f) || !(ex >= -2147483648.f) || !(ey >= -2147483648.f))
        return false;
    T.bx = static_cast<int>(minx);
    T.by = static_cast<int>(miny);
    T.ex = static_cast<int>(ex);
    T.ey = static_cast<int>(ey);
    if (T.bx > T.ex || T.by > T.ey) return false;
    // same_side(a, b, o, p) for the edges (v0,v1; v2), (v1,v2; v0), (v2,v0; v1)
    const float vx[3] = {x0, x1, x2}, vy[3] = {y0, y1, y2};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int b = (e + 1) % 3, o = (e + 2) % 3;
        const float dx = __fsub_rn(vx[b], vx[e]), dy = __fsub_rn(vy[b], vy[e]);
        T.ax[e] = vx[e];
        T.ay[e] = vy[e];
        T.nx[e] = -dy;
        T.ny[e] = dx;
        T.v0[e] = __fadd_rn(__fmul_rn(__fsub_rn(vx[o], vx[e]), -dy), __fmul_rn(__fsub_rn(vy[o], vy[e]), dx));
    }
    return true;
}

__device__ __forceinline__ bool tri_inside(const Tri &T, float px, float py)
{
    bool in = true;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const float v1 = __fadd_rn(__fmul_rn(__fsub_rn(px, T.ax[e]), T.nx[e]), __fmul_rn(__fsub_rn(py, T.ay[e]), T.ny[e]));
        in = in && (__fmul_rn(T.v0[e], v1) >= 0.f);
    }
    return in;
}

// grid: ceil(b * tn / RS_WARPS) CTAs; warp w of CTA c takes triangle c * RS_WARPS + w of the flattened batch.
__global__ void __launch_bounds__(RS_THREADS)
    k_mesh_rasterization(const float *__restrict__ tris, int total, int tn, int h, int w, uint8_t *__restrict__ mask)
{
    __shared__ int s_big[RS_WARPS];
    __shared__ int s_nbig;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_nbig = 0;
    __syncthreads();
    const int t = blockIdx.x * RS_WARPS + warp;
    Tri T;
    if (t < total && tri_setup(tris + static_cast<size_t>(t) * 6, h, w, T)) {
        const int bw = T.ex - T.bx + 1, npix = bw * (T.ey - T.by + 1);
        if (npix > RS_BIG) {
            if (lane == 0) s_big[atomicAdd(&s_nbig, 1)] = t;
        } else {
            uint8_t *m = mask + static_cast<size_t>(t / tn) * h * w;
            for (int p = lane; p < npix; p += 32) {
                const int yi = T.by + p / bw, xi = T.bx + p % bw;
                if (tri_inside(T, static_cast<float>(xi), static_cast<float>(yi))) m[static_cast<size_t>(yi) * w + xi] = 1;
            }
        }
    }
    __syncthreads();
    for (int i = 0; i < s_nbig; ++i) {
        const int tb = s_big[i];
        tri_setup(tris + static_cast<size_t>(tb) * 6, h, w, T);
        uint8_t *m = mask + static_cast<size_t>(tb / tn) * h * w;
        for (int yi = T.by + warp; yi <= T.ey; yi += RS_WARPS)
            for (int xi = T.bx + lane; xi <= T.ex; xi += 32)
                if (tri_inside(T, static_cast<float>(xi), static_cast<float>(yi))) m[static_cast<size_t>(yi) * w + xi] = 1;
    }
}

struct FpsPlan {
    int csize, slice, resident;
};

FpsPlan fps_plan(int pn)
{
    FpsPlan p;
    p.csize = 1;
    while (p.csize < FPS_MAX_CLUSTER && (pn + p.csize - 1) / p.csize > FPS_CTA_POINTS) p.csize *= 2;
    p.slice = (pn + p.csize - 1) / p.csize;
    p.resident = p.slice <= FPS_SLICE;
    return p;
}

}  // namespace

extern "C" {

int pvnet_farthest_point_sampling_workspace_bytes(int b, int pn, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && pn >= 1, "non-positive dimension (b=%d, pn=%d)", b, pn);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = fps_plan(pn).resident ? 0 : static_cast<size_t>(b) * pn * sizeof(float);
    return PVNET_OK;
}

int pvnet_farthest_point_sampling(const float *pts, const int32_t *start, int b, int pn, int sn, int32_t *idxs,
                                  void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && pn >= 1, "non-positive dimension (b=%d, pn=%d)", b, pn);
    PV_CHECK_ARG(sn >= 0, "negative sample count %d", sn);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    PV_CHECK_ARG(pn <= INT32_MAX / 3, "pn %d too large", pn);
    if (sn == 0) return PVNET_OK;
    PV_CHECK_ARG(pts && idxs, "null pointer");
    const FpsPlan p = fps_plan(pn);
    size_t need = 0;
    pvnet_farthest_point_sampling_workspace_bytes(b, pn, &need);
    PV_CHECK_ARG(workspace_bytes >= need && (need == 0 || workspace), "workspace %zu bytes < %zu", workspace_bytes,
                 need);
    const int smem = p.resident ? p.slice * 4 * static_cast<int>(sizeof(float)) : 0;
    PV_CUDA(pvnet::ensure_max_smem((const void *)k_farthest_point_sampling, FPS_SLICE * 4 * sizeof(float)));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(b * p.csize));
    cfg.blockDim = dim3(FPS_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = p.csize;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    PV_CUDA(cudaLaunchKernelEx(&cfg, k_farthest_point_sampling, pts, start, pn, sn, p.slice, p.resident,
                               static_cast<float *>(workspace), idxs));
    PV_LAUNCHED("k_farthest_point_sampling");
    return PVNET_OK;
}

int pvnet_mesh_binary_rasterization(const float *triangles, int b, int tn, int h, int w, uint8_t *mask,
                                    pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && tn >= 0, "bad dimension (b=%d, tn=%d)", b, tn);
    PV_CHECK_ARG(h >= 2 && w >= 2, "mask %dx%d is below 2x2", h, w);
    PV_CHECK_ARG(h <= (1 << 24) && w <= (1 << 24) && static_cast<long long>(h) * w <= INT32_MAX,
                 "mask %dx%d too large", h, w);
    PV_CHECK_ARG(static_cast<long long>(b) * tn <= INT32_MAX - RS_WARPS, "b * tn too large");
    PV_CHECK_ARG(mask && (tn == 0 || triangles), "null pointer");
    PV_CUDA(cudaMemsetAsync(mask, 0, static_cast<size_t>(b) * h * w, (cudaStream_t)stream));
    const int total = b * tn;
    if (total == 0) return PVNET_OK;
    k_mesh_rasterization<<<(total + RS_WARPS - 1) / RS_WARPS, RS_THREADS, 0, (cudaStream_t)stream>>>(triangles, total,
                                                                                                     tn, h, w, mask);
    PV_LAUNCHED("k_mesh_rasterization");
    return PVNET_OK;
}

}  // extern "C"
