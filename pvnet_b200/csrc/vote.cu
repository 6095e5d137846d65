// vote.cu -- PVNet RANSAC voting layer for H100 (sm_90a).
//
// What the reference does per image (lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:514-598):
// torch.nonzero / masked_select compaction, generate_hypothesis kernel, a u8
// [hn,vn,tn] inlier tensor written by voting_for_hypothesis_kernel
// (src/ransac_voting_kernel.cu:88-126), torch.sum over it, max, a second vote for
// the winner and an fp32 least-squares refit -- with >= 3 host syncs per image.
//
// Here the whole batch runs as one short launch sequence with no host sync:
//   k_chunk_count   per-2048-pixel foreground counts
//   k_chunk_kept    per-chunk kept counts (only when an image may be subsampled)
//   k_compact_write stable (row-major) list of foreground pixels, packed (y<<16|x)
//   k_gather        ONE pass over the vector field: direct[b][k][t] (float2, compact, keypoint-
//                   major); every later kernel streams these coalesced lists instead of
//                   gathering sectors from the field again
//   k_gen_hyp       ray-ray intersections, bit-exact op sequence of the reference
//   k_vote3         persistent kernel of autonomous warps: a warp takes (image, keypoint, 256
//                   hypotheses, pixel segment), stages 64 pixels at a time in its private
//                   shared memory as the two edge functionals of the inlier cone, keeps 8
//                   hypotheses per lane and their counts in registers; the [hn,vn,tn]
//                   tensor never exists
//   k_refit         argmax (lowest index on ties) + inlier sums of the winner in fp64
//   k_refit_final   fixed-order reduction + 2x2 solve
//   k_cov           estimate_voting_distribution_with_mean's weighted covariance
//
// Bit-exact inlier counts.  The reference predicate is
//     num/(norm1*norm2) > thresh,  norm = sqrt.rn(fma(..)),  '/' = div.rn
// (two correctly rounded sqrt, one correctly rounded division: ~30 issue slots).  With
// theta the angle between the pixel's direction n and d = hypothesis - pixel, that is
// |theta| < theta_T (cos theta_T = thresh), i.e.
//     m = |d| sin(theta_T - |theta|) = sin(theta_T) (d.u) - cos(theta_T) |d.v| > 0,
// u = n/|n|, v = (-u_y, u_x): two linear functionals of the hypothesis per pixel.  k_vote3
// evaluates them in segment-centred coordinates (4 FMA), -m (1 FADD), counts its sign bit and tracks
// min |m| against a per-hypothesis guard band B (DESIGN.md section 3 bounds both the reference's rounding,
// <= (7 + 1/T) ulp on the cosine, and ours): m > B counts, |m| <= B (or NaN) is re-decided by
// exact_inlier(), the reference's own instruction sequence.  Tests outside the band cannot
// change sign under either rounding, so the counts are identical to the reference's, at
// 4.5 issue slots per test (13.6 in round 1's num*|num| - T^2 d^2 form, kept as k_vote for A/B).
#include "common.cuh"

#include <cfloat>
#include <cmath>
#include <cstdlib>

namespace {

using pvnet::Carver;

constexpr int CH_PX = 2048;       // pixels per compaction chunk
constexpr int CH_THREADS = 256;   // 8 consecutive pixels per thread
constexpr int VT_THREADS = 256;
constexpr int VT_WARPS = VT_THREADS / 32;
constexpr int VT_TILE = 512;      // pixels per staged tile (k_gather's bounding boxes use the same tiling)
constexpr int VT_MAX_B = 1024;    // images per call (prefix table in shared memory)
constexpr int RF_CHUNKS = 8;      // CTAs per (image, keypoint) in the refit pass
constexpr int RF_THREADS = 256;
constexpr float GUARD_EPS = 6e-6f;

struct Strides {
    long long s[5];
};

// ------------------------------------------------------------------ exact sequences
// src/ransac_voting_kernel.cu:107-125 as nvcc compiles it (SASS checked):
// intrinsics pin every rounding so this compiler cannot contract differently.
__device__ __forceinline__ bool exact_inlier(float nx, float ny, float cx, float cy, float hx, float hy,
                                             float thresh)
{
    const float dx = __fsub_rn(hx, cx);
    const float dy = __fsub_rn(hy, cy);
    const float norm1 = __fsqrt_rn(__fmaf_rn(nx, nx, __fmul_rn(ny, ny)));
    const float norm2 = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    if (fmin((double)norm1, (double)norm2) < 1e-6) return false;
    const float num = __fmaf_rn(dx, nx, __fmul_rn(dy, ny));
    const float den = __fmul_rn(norm1, norm2);
    const float ang = __fdiv_rn(num, den);
    return ang > thresh;
}

// src/ransac_voting_kernel.cu:28-48 (contraction read off the SASS of the sm_90a build, DESIGN.md "FP sequence")
__device__ __forceinline__ float2 exact_hypothesis(float d0x, float d0y, float cx0, float cy0, float d1x,
                                                   float d1y, float cx1, float cy1)
{
    const float p = __fmul_rn(d0y, d1x);
    const float q = __fmul_rn(d0x, d1y);
    const float det_y = __fsub_rn(p, q);
    if ((double)fabsf(det_y) < 1e-6) return make_float2(0.f, 0.f);
    const float det_x = __fsub_rn(q, p);
    if ((double)fabsf(det_x) < 1e-6) return make_float2(0.f, 0.f);
    const float s1 = __fmaf_rn(d1y, cx1, -__fmul_rn(d1x, cy1));
    const float s0 = __fmaf_rn(d0y, cx0, -__fmul_rn(d0x, cy0));
    const float y = __fdiv_rn(__fmaf_rn(d1y, s0, -__fmul_rn(d0y, s1)), det_y);
    const float x = __fdiv_rn(__fmaf_rn(-d1x, s0, __fmul_rn(d0x, s1)), det_x);
    return make_float2(x, y);
}

// ------------------------------------------------------------------ block helpers
__device__ __forceinline__ int warp_sum(int v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// sums up to 3 ints over the block; every thread gets the totals. blockDim.x <= 1024
__device__ __forceinline__ void block_sum3(int &a, int &b, int &c, int *scratch /* >= 3*32 ints */)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    a = warp_sum(a);
    b = warp_sum(b);
    c = warp_sum(c);
    __syncthreads();
    if (lane == 0) {
        scratch[warp] = a;
        scratch[32 + warp] = b;
        scratch[64 + warp] = c;
    }
    __syncthreads();
    int ta = 0, tb = 0, tc = 0;
    for (int i = 0; i < nw; ++i) {
        ta += scratch[i];
        tb += scratch[32 + i];
        tc += scratch[64 + i];
    }
    a = ta;
    b = tb;
    c = tc;
}

template <typename T>
__device__ __forceinline__ bool is_foreground(T v, int mode)
{
    if (mode == PVNET_MASK_EQUALS_ONE) return v == (T)1;
    return (unsigned char)v != 0;  // `.byte()` keeps the low 8 bits (ransac_voting_gpu.py:527)
}

// `max_num / foreground.float()`: torch evaluates int / tensor as reciprocal() * int
// in float32 (ransac_voting_gpu.py:539)
__device__ __forceinline__ float subsample_p(int fg, int max_num)
{
    return __fmul_rn(__frcp_rn((float)fg), (float)max_num);
}

// ------------------------------------------------------------------ device RNG
// Philox4x32-10 (Salmon et al. 2011; the generator behind torch.cuda's random_/uniform_), used when
// the caller passes no idxs / selection tensors: counter = (item, image | stream<<28, call offset),
// key = seed.  rng_state is a DEVICE pointer {seed, offset}; the last kernel of a call bumps the
// offset, so a captured CUDA graph draws fresh samples on every replay.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}
enum { RNG_SELECTION = 0, RNG_IDXS_V3 = 1, RNG_IDXS_COV = 2 };
__device__ __forceinline__ uint4 rng_draw(const unsigned long long *__restrict__ rng_state, unsigned item,
                                          unsigned image, unsigned stream)
{
    const unsigned long long seed = rng_state[0], off = rng_state[1];
    return philox4x32_10(make_uint4(item, image | (stream << 28), (unsigned)off, (unsigned)(off >> 32)),
                         make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
}
// the uniform field of ransac_voting_gpu.py:538: caller's tensor, or 24 random bits * 2^-24 (torch's uniform_)
__device__ __forceinline__ float selection_value(const float *__restrict__ sel_field,
                                                 const unsigned long long *__restrict__ rng_state, int b, int npx, int i)
{
    if (sel_field) return sel_field[(size_t)b * npx + i];
    return (float)(rng_draw(rng_state, (unsigned)i, (unsigned)b, RNG_SELECTION).x & 0xffffffu) * 5.9604644775390625e-8f;
}
__global__ void k_rng_bump(unsigned long long *rng_state) { rng_state[1] += 1ull; }

// ------------------------------------------------------------------ compaction
// pass 1: foreground count of every 2048-pixel chunk
template <typename T>
__global__ void __launch_bounds__(CH_THREADS) k_chunk_count(const T *__restrict__ mask, int mode, int npx,
                                                             int nchunk, int *__restrict__ chunk_fg)
{
    __shared__ int scratch[96];
    const int c = blockIdx.x, b = blockIdx.y;
    const T *m = mask + (size_t)b * npx;
    const int base = c * CH_PX + threadIdx.x * 8;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int i = base + j;
        if (i < npx) cnt += is_foreground(m[i], mode) ? 1 : 0;
    }
    int z0 = 0, z1 = 0;
    block_sum3(cnt, z0, z1, scratch);
    if (threadIdx.x == 0) chunk_fg[b * nchunk + c] = cnt;
}

// pass 2: kept pixels per chunk.  Equals the foreground count unless the image has
// more than max_num foreground pixels, in which case pixel i survives iff
// selection[i] < p (ransac_voting_gpu.py:537-540).  Images below min_num keep nothing.
template <typename T>
__global__ void __launch_bounds__(CH_THREADS)
    k_chunk_kept(const T *__restrict__ mask, int mode, const float *__restrict__ selection,
                 const unsigned long long *__restrict__ rng_state, int npx, int nchunk, int min_num, int max_num,
                 const int *__restrict__ chunk_fg, int *__restrict__ chunk_kept, int *__restrict__ status)
{
    __shared__ int scratch[96];
    const int c = blockIdx.x, b = blockIdx.y;
    int tot = 0, z0 = 0, z1 = 0;
    for (int i = threadIdx.x; i < nchunk; i += blockDim.x) tot += chunk_fg[b * nchunk + i];
    block_sum3(tot, z0, z1, scratch);
    const bool skip = tot < min_num;
    const bool have_sel = selection != nullptr || rng_state != nullptr;
    const bool sub = tot > max_num;
    if (!sub || !have_sel) {
        if (threadIdx.x == 0) {
            chunk_kept[b * nchunk + c] = skip ? 0 : chunk_fg[b * nchunk + c];
            if (c == 0) status[b] = (skip ? 1 : 0) | ((sub && !have_sel) ? 4 : 0);
        }
        return;
    }
    const float p = subsample_p(tot, max_num);
    const T *m = mask + (size_t)b * npx;
    const int base = c * CH_PX + threadIdx.x * 8;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int i = base + j;
        if (i < npx) cnt += (is_foreground(m[i], mode) && selection_value(selection, rng_state, b, npx, i) < p) ? 1 : 0;
    }
    block_sum3(cnt, z0, z1, scratch);
    if (threadIdx.x == 0) {
        chunk_kept[b * nchunk + c] = cnt;
        if (c == 0) status[b] = 2;
    }
}

// pass 3: write the stable pixel list.  pix[b][r] = (y<<16)|x of the r-th kept pixel
// in row-major order == row r of torch.nonzero (ransac_voting_gpu.py:542).
template <typename T>
__global__ void __launch_bounds__(CH_THREADS)
    k_compact_write(const T *__restrict__ mask, int mode, const float *__restrict__ selection,
                    const unsigned long long *__restrict__ rng_state, int npx, int width, int nchunk, int min_num,
                    int max_num, const int *__restrict__ chunk_fg, const int *__restrict__ chunk_kept_or_null,
                    unsigned *__restrict__ pix, int *__restrict__ tn_out, int *__restrict__ fg_out)
{
    __shared__ int scratch[96];
    __shared__ int warp_off[CH_THREADS / 32];
    const int c = blockIdx.x, b = blockIdx.y;
    // chunk_kept_or_null == nullptr: nothing can be subsampled (no selection source), so the kept
    // counts are the foreground counts (or 0 for an image below min_num) and pass 2 is not launched
    const int *chunk_kept = chunk_kept_or_null ? chunk_kept_or_null : chunk_fg;
    int tot_fg = 0, prefix = 0, tot_kept = 0;
    for (int i = threadIdx.x; i < nchunk; i += blockDim.x) {
        const int k = chunk_kept[b * nchunk + i];
        tot_fg += chunk_fg[b * nchunk + i];
        tot_kept += k;
        if (i < c) prefix += k;
    }
    block_sum3(tot_fg, prefix, tot_kept, scratch);
    if (!chunk_kept_or_null && tot_fg < min_num) tot_kept = 0;
    if (c == 0 && threadIdx.x == 0) {
        tn_out[b] = tot_kept;
        fg_out[b] = tot_fg;
    }
    if (tot_kept == 0 || chunk_kept[b * nchunk + c] == 0) return;
    const bool sub = (tot_fg > max_num) && chunk_kept_or_null && (selection != nullptr || rng_state != nullptr);
    const float p = sub ? subsample_p(tot_fg, max_num) : 0.f;
    const T *m = mask + (size_t)b * npx;
    const int base = c * CH_PX + threadIdx.x * 8;
    unsigned flags = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int i = base + j;
        if (i < npx) {
            bool keep = is_foreground(m[i], mode);
            if (sub && keep) keep = selection_value(selection, rng_state, b, npx, i) < p;
            flags |= (keep ? 1u : 0u) << j;
        }
    }
    const int mine = __popc(flags);
    // exclusive scan over the block, thread order == pixel order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) warp_off[warp] = inc;
    __syncthreads();
    int woff = 0;
    for (int i = 0; i < warp; ++i) woff += warp_off[i];
    int r = prefix + woff + inc - mine;
    unsigned *out = pix + (size_t)b * npx;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (flags & (1u << j)) {
            const int i = base + j;
            const int y = i / width, x = i - y * width;
            out[r++] = ((unsigned)y << 16) | (unsigned)x;
        }
    }
}

// reduce chunk counts to per-image totals (pvnet_mask_foreground_count)
__global__ void k_sum_chunks(const int *__restrict__ chunk_fg, int nchunk, int *__restrict__ fg_out)
{
    __shared__ int scratch[96];
    const int b = blockIdx.x;
    int tot = 0, z0 = 0, z1 = 0;
    for (int i = threadIdx.x; i < nchunk; i += blockDim.x) tot += chunk_fg[b * nchunk + i];
    block_sum3(tot, z0, z1, scratch);
    if (threadIdx.x == 0) fg_out[b] = tot;
}

// ------------------------------------------------------------------ gather
// One CTA per (512-pixel tile, image): direct[b][k][t] = vertex[b, y_t, x_t, k, :] for every keypoint,
// read through the caller's strides (thread = pixel: coalesced along mask rows for the NCHW view,
// L1-resident 8-byte pieces of one record for a pixel-major field), written coalesced.  Every later
// kernel streams these compact lists instead of gathering sectors from the field again.
__global__ void __launch_bounds__(256)
    k_gather(const float *__restrict__ vertex, Strides st, const unsigned *__restrict__ pix,
             const int *__restrict__ tn_arr, int npx, int cap, int vn, float2 *__restrict__ direct)
{
    const int g = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int tn = tn_arr[b];
    const int t0 = g * VT_TILE;
    if (t0 >= tn) return;
    const int len = min(VT_TILE, tn - t0);
    const bool vec2 = st.s[4] == 1 && ((st.s[0] | st.s[1] | st.s[2] | st.s[3]) & 1) == 0 &&
                      (reinterpret_cast<uintptr_t>(vertex) & 7) == 0;
    for (int i = tid; i < len; i += 256) {
        const unsigned p = pix[(size_t)b * npx + t0 + i];
        const int x = p & 0xffff, y = p >> 16;
        const long long base = (long long)b * st.s[0] + (long long)y * st.s[1] + (long long)x * st.s[2];
        float2 *o = direct + (size_t)b * vn * cap + t0 + i;
        for (int k = 0; k < vn; ++k) {
            const long long off = base + (long long)k * st.s[3];
            float2 v;
            if (vec2) v = __ldg(reinterpret_cast<const float2 *>(vertex + off));
            else v = make_float2(__ldg(vertex + off), __ldg(vertex + off + st.s[4]));
            o[(size_t)k * cap] = v;
        }
    }
}

// ------------------------------------------------------------------ hypotheses
// idxs [b,hn,vn,2] (or the device RNG) -> hyp [b][vn][HT] at column h_off + h (keypoint-major so a
// vote CTA reads one row).  Samples index the compact direct list.
__global__ void __launch_bounds__(256)
    k_gen_hyp(const float2 *__restrict__ direct, const int *__restrict__ idxs,
              const unsigned long long *__restrict__ rng_state, int rng_stream, const unsigned *__restrict__ pix,
              const int *__restrict__ tn_arr, int npx, int cap, int vn, int hn, int HT, int h_off,
              float2 *__restrict__ hyp)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (i >= hn * vn) return;
    const int hi = i / vn, vi = i - hi * vn;
    const int tn = tn_arr[b];
    float2 out = make_float2(0.f, 0.f);
    if (tn > 0) {
        unsigned t0, t1;
        if (idxs) {
            const size_t ib = (((size_t)b * hn + hi) * vn + vi) * 2;
            t0 = (unsigned)idxs[ib] % (unsigned)tn;
            t1 = (unsigned)idxs[ib + 1] % (unsigned)tn;
        } else {       // torch's random_(0, tn) is a 32-bit draw modulo tn as well
            const uint4 r = rng_draw(rng_state, (unsigned)i, (unsigned)b, (unsigned)rng_stream);
            t0 = r.x % (unsigned)tn;
            t1 = r.y % (unsigned)tn;
        }
        const unsigned p0 = pix[(size_t)b * npx + t0], p1 = pix[(size_t)b * npx + t1];
        const float2 d0 = direct[((size_t)b * vn + vi) * cap + t0], d1 = direct[((size_t)b * vn + vi) * cap + t1];
        out = exact_hypothesis(d0.x, d0.y, (float)(p0 & 0xffff), (float)(p0 >> 16), d1.x, d1.y, (float)(p1 & 0xffff),
                               (float)(p1 >> 16));
    }
    hyp[((size_t)b * vn + vi) * HT + h_off + hi] = out;
}

// fast-path helpers of the vote kernels
constexpr int VT_GROUP = 4;       // pixels per guard-band check
__device__ __forceinline__ uint32_t ptx_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float4 lds_f4(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
// cnt += (a > b): one FSETP + one predicated IADD (the C form compiled to add + predicated move + move)
__device__ __forceinline__ void count_if_gt(int &cnt, float a, float b)
{
    asm("{\n\t.reg .pred p;\n\tsetp.gt.f32 p, %1, %2;\n\t@p add.s32 %0, %0, 1;\n\t}" : "+r"(cnt) : "f"(a), "f"(b));
}

// ------------------------------------------------------------------ the vote
// Persistent CTAs walk items (pixel tile, keypoint, hypothesis group).  Warps are
// split wh (hypothesis groups of 128) x wp (pixel interleave); each lane owns
// VT_HPL hypotheses; pixels come from shared memory as one broadcast LDS.128.
template <int HPL, int TILE>
__global__ void __launch_bounds__(VT_THREADS, HPL > 4 ? 2 : 4)
    k_vote(const float *__restrict__ vertex, Strides st, const unsigned *__restrict__ pix,
           const int *__restrict__ tn_arr, int npx, int nb, int vn, int hn, int HT, int h0, int wh,
           const float2 *__restrict__ hyp, int *__restrict__ counts, float thresh, float t2, float band)
{
    __shared__ float4 tile[TILE];
    __shared__ int red[VT_WARPS * 32 * HPL];
    __shared__ int tile_prefix[VT_MAX_B + 1];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        int acc = 0;
        for (int i = 0; i < nb; ++i) {
            tile_prefix[i] = acc;
            acc += (tn_arr[i] + TILE - 1) / TILE;
        }
        tile_prefix[nb] = acc;
    }
    __syncthreads();
    const int total_tiles = tile_prefix[nb];
    const int HC = wh * 32 * HPL;               // hypotheses per item
    const int hcn = (hn + HC - 1) / HC;
    const long long n_items = (long long)total_tiles * vn * hcn;
    const int wp_count = VT_WARPS / wh;
    const int my_wh = warp % wh, my_wp = warp / wh;

    for (long long it = blockIdx.x; it < n_items; it += gridDim.x) {
        const int hc = (int)(it % hcn);
        const long long r = it / hcn;
        const int k = (int)(r % vn);
        const int g = (int)(r / vn);
        int lo = 0, hi = nb;                         // b with tile_prefix[b] <= g < tile_prefix[b+1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (tile_prefix[mid] <= g) lo = mid; else hi = mid;
        }
        const int b = lo;
        const int tn = tn_arr[b];
        const int t0 = (g - tile_prefix[b]) * TILE;
        const int len = min(TILE, tn - t0);
        const long long vbase = (long long)b * st.s[0] + (long long)k * st.s[3];

        // ---- stage: gather this tile's pixels and unit directions
        for (int i = tid; i < len; i += VT_THREADS) {
            const unsigned p = __ldg(pix + (size_t)b * npx + t0 + i);
            const int x = p & 0xffff, y = p >> 16;
            const long long off = vbase + y * st.s[1] + x * st.s[2];
            const float nx = __ldg(vertex + off), ny = __ldg(vertex + off + st.s[4]);
            const float n2 = fmaf(nx, nx, ny * ny);
            const float rinv = rsqrtf(n2);
            float ux = nx * rinv, uy = ny * rinv;
            if (!(n2 > 1e-11f && n2 < 1e30f)) ux = uy = __int_as_float(0x7fc00000);  // -> exact path
            tile[i] = make_float4((float)x, (float)y, ux, uy);
        }
        for (int i = tid; i < HC; i += VT_THREADS) red[i] = 0;
        __syncthreads();

        // ---- this lane's hypotheses
        const int hbase = hc * HC + my_wh * (32 * HPL);
        float hx[HPL], hy[HPL];
        int cnt[HPL];
#pragma unroll
        for (int j = 0; j < HPL; ++j) {
            const int h = hbase + j * 32 + lane;
            float2 hp = make_float2(3.0e8f, 3.0e8f);   // padding hypothesis, count discarded
            if (h < hn) hp = __ldg(hyp + ((size_t)b * vn + k) * HT + h0 + h);
            hx[j] = hp.x;
            hy[j] = hp.y;
            cnt[j] = 0;
        }

        // ---- sweep the tile, VT_GROUP pixels at a time.  The fast path only counts and ORs one
        // "some test fell inside the guard band" flag per lane; when any lane of the warp raises it
        // (rare), the group is re-walked and exactly those tests are re-decided with the reference's
        // own instruction sequence (they were NOT counted by the fast path: |e| <= bd excludes e > bd).
        const uint32_t tile_u = ptx_smem_u32(tile);
        auto sweep = [&](int i0, int n) {           // pixels i0, i0 + wp_count, ... (n of them, n <= VT_GROUP)
            bool unc = false;
#pragma unroll
            for (int u = 0; u < VT_GROUP; ++u) {
                if (u < n) {
                    const float4 p = lds_f4(tile_u + (uint32_t)(i0 + u * wp_count) * 16u);
#pragma unroll
                    for (int j = 0; j < HPL; ++j) {
                        const float dx = hx[j] - p.x, dy = hy[j] - p.y;
                        const float d2 = fmaf(dx, dx, dy * dy);
                        const float num = fmaf(dx, p.z, dy * p.w);
                        const float s = num * fabsf(num);
                        const float e = fmaf(-t2, d2, s);
                        const float bd = fmaf(band, d2, 4e-12f);
                        count_if_gt(cnt[j], e, bd);
                        unc |= !(fabsf(e) > bd);
                    }
                }
            }
            if (__any_sync(0xffffffffu, unc)) {
                if (unc) {
                    for (int u = 0; u < n; ++u) {
                        const float4 p = tile[i0 + u * wp_count];
                        const long long off = vbase + (long long)p.y * st.s[1] + (long long)p.x * st.s[2];
                        const float nx = __ldg(vertex + off), ny = __ldg(vertex + off + st.s[4]);
#pragma unroll
                        for (int j = 0; j < HPL; ++j) {
                            const float dx = hx[j] - p.x, dy = hy[j] - p.y;
                            const float d2 = fmaf(dx, dx, dy * dy);
                            const float num = fmaf(dx, p.z, dy * p.w);
                            const float s = num * fabsf(num);
                            const float e = fmaf(-t2, d2, s);
                            const float bd = fmaf(band, d2, 4e-12f);
                            if (!(fabsf(e) > bd))
                                cnt[j] += exact_inlier(nx, ny, p.x, p.y, hx[j], hy[j], thresh) ? 1 : 0;
                        }
                    }
                }
            }
        };
        int i = my_wp;
        for (; i + (VT_GROUP - 1) * wp_count < len; i += VT_GROUP * wp_count) sweep(i, VT_GROUP);
        if (i < len) sweep(i, (len - i + wp_count - 1) / wp_count);

        // ---- combine the pixel-interleaved warps, then one atomic per hypothesis
#pragma unroll
        for (int j = 0; j < HPL; ++j)
            if (cnt[j]) atomicAdd(&red[my_wh * (32 * HPL) + j * 32 + lane], cnt[j]);
        __syncthreads();
        for (int i = tid; i < HC; i += VT_THREADS) {
            const int h = hc * HC + i;
            const int v = red[i];
            if (h < hn && v) atomicAdd(counts + ((size_t)b * vn + k) * HT + h0 + h, v);
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ the vote (round 2)
// k_vote3: persistent kernel of AUTONOMOUS WARPS.  A warp pulls (image, keypoint, group of 32*HPL hypotheses,
// pixel segment) items from a ticket counter, keeps its hypotheses and counts in registers for the whole segment,
// stages 64 pixels at a time from the COMPACT lists (coalesced 4-/8-byte streams) into its private 3 KB of shared
// memory (next sub-chunk prefetched into registers during the sweep; only __syncwarp) and publishes the counts
// with one RED per hypothesis.  No CTA barrier after the prologue.  (An earlier form with CTA-wide tiles spent 48 %
// of its stall samples outside the test loop: dependent global loads of staging / hypothesis set-up, three CTA
// barriers per item.)
//
// The test.  Staged per pixel: the two edge functionals of the inlier cone in segment-centred coordinates,
//     s = sin(theta_T) u,  c = cos(theta_T) v:   num = h'.s - p'.s,   perp = h'.c - p'.c,
// so one test is  num = fma(hx', sx, fma(hy', sy, -s.p'));  perp = fma(hx', cx, fma(hy', cy, -c.p'));
// m = num - |perp|;  inlier if m > B;  IN BAND if !(|m| > B).
// B = beta (|hx'| + |hy'| + r1) + b0 per hypothesis and segment (|d| <= |h'|_1 + r1): beta carries the
// reference's rounding band (7 + 1/T) ulp T / sin(theta_T) and ours, see DESIGN.md section 3.
//
// Instruction mix:
//   * two hypotheses are kept as a pair (f32x2) so a pair of pixel operands comes straight out of one LDS.128
//     (the pixel operands are stored pre-duplicated); sm_90a evaluates the pair as two lane-wise FFMA;
//   * the FAST decision is the sign bit of  e = |perp| - num = -m  (one FADD), added to an integer count by ONE
//     ALU-pipe instruction (LEA.HI cnt, e, cnt, RZ, 1  =  cnt + (e >> 31)); a NaN e is the canonical positive NaN:
//     not counted;
//   * the guard band is NOT tested per test: every hypothesis keeps  mab = min over the sub-chunk of |e|  (NaN-
//     propagating min with |.| operands), compared with B once per 64 pixels.  A hypothesis with !(mab > B) is
//     re-walked by the whole warp (2 pixels per lane, the same fma chains bit for bit) and exactly its in-band tests
//     get exact_inlier() on the raw values; one RED adds  exact - fast.  Outside the band sign(m) IS the reference's
//     decision (that is what B bounds), inside it is corrected: the counts are the reference's.
typedef unsigned long long f32x2;
__device__ __forceinline__ f32x2 pk2(float a, float b)
{
    f32x2 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ void upk2(f32x2 v, float &a, float &b)
{
    asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
}
// two lane-wise fma.rn (sm_90a has no packed fp32 FMA; the results are the same bits)
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c)
{
    float a0, a1, b0, b1, c0, c1;
    upk2(a, a0, a1);
    upk2(b, b0, b1);
    upk2(c, c0, c1);
    return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ void lds_2x64(uint32_t addr, f32x2 &a, f32x2 &b)
{
    asm volatile("ld.shared.v2.b64 {%0, %1}, [%2];" : "=l"(a), "=l"(b) : "r"(addr));
}
constexpr int VT_SUB = 64;        // pixels per staged sub-chunk (2 per lane)

__device__ __forceinline__ float min3_nan_abs(float a, float b, float c)     // min(a, |b|, |c|), NaN if any is
{
    float r;
    asm("{\n\t.reg .f32 t;\n\tmin.NaN.f32 t, %1, %2;\n\tmin.NaN.f32 %0, t, %3;\n\t}" : "=f"(r) : "f"(a), "f"(fabsf(b)), "f"(fabsf(c)));
    return r;
}

template <int HPL, int G>
__global__ void __launch_bounds__(VT_THREADS, HPL > 4 ? 2 : 3)
    k_vote3(const unsigned *__restrict__ pix, const float2 *__restrict__ direct, const int *__restrict__ tn_arr, int npx,
            int cap, int nb, int vn, int hn, int HT, int h0, const float2 *__restrict__ hyp, int *__restrict__ counts,
            unsigned *__restrict__ ticket, float thresh, float sn, float cs, float beta, float b0, int items_per_warp)
{
    static_assert(G % 2 == 0 && VT_SUB % G == 0, "pixels are swept in pairs");
    // per warp, per pixel 48 bytes: {sx,sx,sy,sy} {ns,ns,cx,cx} {cy,cy,nc,nc}
    __shared__ float4 rec_all[VT_WARPS * 3 * VT_SUB];
    __shared__ int seg_prefix[VT_MAX_B + 1];
    __shared__ int s_seg;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int HC = 32 * HPL;
    const int hcn = (hn + HC - 1) / HC;
    if (tid == 0) {
        // pixels per item: the largest power-of-two multiple of VT_SUB (<= 4096) that still leaves items_per_warp items
        // per resident warp, so hypotheses are set up rarely and the tail of the ticket queue stays short
        long long px = 0;
        for (int i = 0; i < nb; ++i) px += tn_arr[i];
        const long long want = (long long)gridDim.x * VT_WARPS * items_per_warp;
        int seg = 4096;
        while (seg > 4 * VT_SUB && (px / seg + nb) * vn * hcn < want) seg >>= 1;
        int acc = 0;
        for (int i = 0; i < nb; ++i) {
            seg_prefix[i] = acc;
            acc += (tn_arr[i] + seg - 1) / seg;
        }
        seg_prefix[nb] = acc;
        s_seg = seg;
    }
    __syncthreads();
    const int SEG = s_seg;
    const long long n_items = (long long)seg_prefix[nb] * vn * hcn;
    const float qnan = __int_as_float(0x7fc00000);
    const float finf = __int_as_float(0x7f800000);
    float4 *rec = rec_all + warp * (3 * VT_SUB);
    const uint32_t rec_u = ptx_smem_u32(rec);

    for (;;) {
        unsigned item_u = 0;
        if (lane == 0) item_u = atomicAdd(ticket, 1u);
        const long long it = (long long)__shfl_sync(0xffffffffu, item_u, 0);
        if (it >= n_items) break;
        const int hc = (int)(it % hcn);
        const long long r = it / hcn;
        const int k = (int)(r % vn);
        const int g = (int)(r / vn);
        int lo = 0, hi = nb;                         // b with seg_prefix[b] <= g < seg_prefix[b+1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (seg_prefix[mid] <= g) lo = mid; else hi = mid;
        }
        const int b = lo;
        const int tn = tn_arr[b];
        const int t0 = (g - seg_prefix[b]) * SEG;
        const int len = min(SEG, tn - t0);
        const unsigned *pix_t = pix + (size_t)b * npx + t0;
        const float2 *dir_t = direct + ((size_t)b * vn + k) * cap + t0;

        const int hbase = hc * HC;
        const float2 *hyp_row = hyp + ((size_t)b * vn + k) * HT + h0;
        int *cnt_row = counts + ((size_t)b * vn + k) * HT + h0;
        float2 hraw[HPL];
#pragma unroll
        for (int j = 0; j < HPL; ++j) {
            const int h = hbase + j * 32 + lane;
            hraw[j] = (h < hn) ? __ldg(hyp_row + h) : make_float2(0.f, 0.f);
        }
        unsigned pp[2];
        float2 pn[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int i = e * 32 + lane;
            pp[e] = (i < len) ? __ldg(pix_t + i) : 0u;
            pn[e] = (i < len) ? __ldg(dir_t + i) : make_float2(0.f, 0.f);
        }
        int xmin = 0x7fffffff, xmax = -1;
        for (int i = lane; i < len; i += 32) {
            const int x = (int)(__ldg(pix_t + i) & 0xffffu);
            xmin = min(xmin, x);
            xmax = max(xmax, x);
        }
        xmin = __reduce_min_sync(0xffffffffu, xmin);
        xmax = __reduce_max_sync(0xffffffffu, xmax);
        const int ymin = (int)(__ldg(pix_t) >> 16), ymax = (int)(__ldg(pix_t + len - 1) >> 16);
        const float xc = (float)((xmin + xmax) >> 1), yc = (float)((ymin + ymax) >> 1);
        const float r1 = (float)(max((int)xc - xmin, xmax - (int)xc) + max((int)yc - ymin, ymax - (int)yc));

        // centred hypothesis and its band; ONE definition, used by the set-up and by the re-walk
        auto centre = [&](float2 hp, float &hxv, float &hyv, float &bd) {
            hxv = hp.x - xc;
            hyv = hp.y - yc;
            bd = fmaf(beta, fabsf(hxv) + fabsf(hyv) + r1, b0);
            if (!(bd < 1e18f)) bd = qnan;           // absurdly far / non-finite: every test exact
        };
        f32x2 hx2[HPL / 2], hy2[HPL / 2];
        float bdv[HPL], mab[HPL];                   // band, min |m| over the current sub-chunk
        int cnt[HPL];
#pragma unroll
        for (int j = 0; j < HPL; j += 2) {
            float hxv[2], hyv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int h = hbase + (j + e) * 32 + lane;
                float bd = -1.f;                    // padding: never in band, count discarded
                hxv[e] = hyv[e] = 0.f;
                if (h < hn) centre(hraw[j + e], hxv[e], hyv[e], bd);
                bdv[j + e] = bd;
                cnt[j + e] = 0;
                mab[j + e] = finf;
            }
            hx2[j / 2] = pk2(hxv[0], hxv[1]);
            hy2[j / 2] = pk2(hyv[0], hyv[1]);
        }

        for (int c0 = 0; c0 < len; c0 += VT_SUB) {
            const int clen = min(VT_SUB, len - c0);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = e * 32 + lane;
                const unsigned p = pp[e];
                const float2 n = pn[e];
                const float xr = (float)(int)(p & 0xffff) - xc, yr = (float)(int)(p >> 16) - yc;
                const float n2 = fmaf(n.x, n.x, n.y * n.y);
                const float rinv = rsqrtf(n2);
                const float ux = n.x * rinv, uy = n.y * rinv;
                float sx = sn * ux, sy = sn * uy, cx = -cs * uy, cy = cs * ux;
                float ns = -fmaf(sx, xr, sy * yr), nc = -fmaf(cx, xr, cy * yr);
                if (!(n2 > 1e-11f && n2 < 1e30f)) sx = sy = cx = cy = ns = nc = qnan;   // -> exact path
                if (i >= clen) {                    // padding pixel: m = -1e30, never counted, never in band
                    sx = sy = cx = cy = nc = 0.f;
                    ns = -1e30f;
                }
                rec[3 * i] = make_float4(sx, sx, sy, sy);
                rec[3 * i + 1] = make_float4(ns, ns, cx, cx);
                rec[3 * i + 2] = make_float4(cy, cy, nc, nc);
            }
            __syncwarp();
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int i = c0 + VT_SUB + e * 32 + lane;
                pp[e] = (i < len) ? __ldg(pix_t + i) : 0u;
                pn[e] = (i < len) ? __ldg(dir_t + i) : make_float2(0.f, 0.f);
            }
            // ---- sweep, two pixels at a time (branch-free)
            const int cend = (clen + G - 1) / G * G;
            for (int i0 = 0; i0 < cend; i0 += G) {
                const uint32_t base = rec_u + (uint32_t)i0 * 48u;
#pragma unroll
                for (int u = 0; u < G; u += 2) {
                    f32x2 SX0, SY0, NS0, CX0, CY0, NC0, SX1, SY1, NS1, CX1, CY1, NC1;
                    lds_2x64(base + (uint32_t)u * 48u, SX0, SY0);
                    lds_2x64(base + (uint32_t)u * 48u + 16u, NS0, CX0);
                    lds_2x64(base + (uint32_t)u * 48u + 32u, CY0, NC0);
                    lds_2x64(base + (uint32_t)u * 48u + 48u, SX1, SY1);
                    lds_2x64(base + (uint32_t)u * 48u + 64u, NS1, CX1);
                    lds_2x64(base + (uint32_t)u * 48u + 80u, CY1, NC1);
#pragma unroll
                    for (int j = 0; j < HPL / 2; ++j) {
                        const f32x2 p0 = fma2(hx2[j], SX0, fma2(hy2[j], SY0, NS0));       // num,  pixel u
                        const f32x2 q0 = fma2(hx2[j], CX0, fma2(hy2[j], CY0, NC0));       // perp, pixel u
                        const f32x2 p1 = fma2(hx2[j], SX1, fma2(hy2[j], SY1, NS1));       // pixel u + 1
                        const f32x2 q1 = fma2(hx2[j], CX1, fma2(hy2[j], CY1, NC1));
                        float p0a, p0b, q0a, q0b, p1a, p1b, q1a, q1b;
                        upk2(p0, p0a, p0b);
                        upk2(q0, q0a, q0b);
                        upk2(p1, p1a, p1b);
                        upk2(q1, q1a, q1b);
                        // e = -m = |perp| - num: its sign bit IS the fast decision (LEA.HI adds it to the count)
                        const float e0a = fabsf(q0a) - p0a, e0b = fabsf(q0b) - p0b;
                        const float e1a = fabsf(q1a) - p1a, e1b = fabsf(q1b) - p1b;
                        cnt[2 * j] += (int)(__float_as_uint(e0a) >> 31);
                        cnt[2 * j + 1] += (int)(__float_as_uint(e0b) >> 31);
                        cnt[2 * j] += (int)(__float_as_uint(e1a) >> 31);
                        cnt[2 * j + 1] += (int)(__float_as_uint(e1b) >> 31);
                        mab[2 * j] = min3_nan_abs(mab[2 * j], e0a, e1a);
                        mab[2 * j + 1] = min3_nan_abs(mab[2 * j + 1], e0b, e1b);
                    }
                }
            }
            // ---- guard band, once per sub-chunk: which of my hypotheses came within B of a cone edge?
            unsigned fl = 0;
#pragma unroll
            for (int j = 0; j < HPL; ++j) {
                if (!(mab[j] > bdv[j])) fl |= 1u << j;
                mab[j] = finf;
            }
            unsigned lanes = __ballot_sync(0xffffffffu, fl != 0);
            while (lanes) {                                        // rare: ~1 hypothesis in 1000 per sub-chunk
                const int src = __ffs(lanes) - 1;
                lanes &= lanes - 1;
                unsigned fm = __shfl_sync(0xffffffffu, fl, src);
                while (fm) {
                    const int j = __ffs(fm) - 1;
                    fm &= fm - 1;
                    const int h = hbase + j * 32 + src;
                    if (h >= hn) continue;
                    const float2 hp = __ldg(hyp_row + h);
                    float hxs, hys, bd;
                    centre(hp, hxs, hys, bd);
                    int add = 0;                            // exact decision minus what the sweep counted
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int pi = e * 32 + lane;
                        if (pi < clen) {
                            const float4 ra = rec[3 * pi], rb = rec[3 * pi + 1], rc = rec[3 * pi + 2];
                            const float num = fmaf(hxs, ra.x, fmaf(hys, ra.z, rb.x));
                            const float perp = fmaf(hxs, rb.z, fmaf(hys, rc.x, rc.z));
                            const float ev = fabsf(perp) - num;
                            if (!(fabsf(ev) > bd)) {
                                const unsigned p = __ldg(pix_t + c0 + pi);
                                const float2 nraw = __ldg(dir_t + c0 + pi);
                                add += (exact_inlier(nraw.x, nraw.y, (float)(p & 0xffff), (float)(p >> 16), hp.x, hp.y, thresh)
                                            ? 1
                                            : 0) -
                                       (int)(__float_as_uint(ev) >> 31);
                            }
                        }
                    }
                    add = __reduce_add_sync(0xffffffffu, add);
                    if (lane == 0 && add) atomicAdd(cnt_row + h, add);
                }
            }
            __syncwarp();
        }

#pragma unroll
        for (int j = 0; j < HPL; ++j) {
            const int h = hbase + j * 32 + lane;
            if (h < hn && cnt[j]) atomicAdd(cnt_row + h, cnt[j]);
        }
    }
}

// ------------------------------------------------------------------ argmax + refit
__device__ __forceinline__ double warp_sum_d(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// grid (RF_CHUNKS, b*vn).  Winner = max count, lowest hypothesis index on ties
// (torch.max, ransac_voting_gpu.py:562); kept only if its count is > 0 (:567).  Then the
// inliers of the winner (:582-584) feed  sum n n^T  and  sum n (n.c),  n = (d_y,-d_x)
// (:579-593), accumulated in fp64.
__global__ void __launch_bounds__(RF_THREADS)
    k_refit(const float2 *__restrict__ direct, int cap, const unsigned *__restrict__ pix,
            const int *__restrict__ tn_arr, int npx, int vn, int hn, int HT, const float2 *__restrict__ hyp,
            const int *__restrict__ counts, float thresh, double *__restrict__ part, float2 *__restrict__ win,
            const float2 *__restrict__ win_in)
{
    __shared__ unsigned long long s_key[RF_THREADS / 32];
    __shared__ double s_acc[RF_THREADS / 32][5];
    const int rc = blockIdx.x, bk = blockIdx.y, b = bk / vn, k = bk - b * vn;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tn = tn_arr[b];
    double *my_part = part + ((size_t)bk * RF_CHUNKS + rc) * 5;
    if (tn == 0) {
        if (tid < 5) my_part[tid] = 0.0;
        if (rc == 0 && tid == 0) win[bk] = make_float2(0.f, 0.f);
        return;
    }
    unsigned long long key = 0;
    for (int h = tid; h < (win_in ? 0 : hn); h += RF_THREADS) {
        const unsigned long long kk =
            ((unsigned long long)(unsigned)counts[(size_t)bk * HT + h] << 32) | (unsigned long long)(0xffffffffu - (unsigned)h);
        key = kk > key ? kk : key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
        key = other > key ? other : key;
    }
    if (lane == 0) s_key[warp] = key;
    __syncthreads();
    key = s_key[0];
    for (int i = 1; i < RF_THREADS / 32; ++i) key = s_key[i] > key ? s_key[i] : key;
    const unsigned best_cnt = (unsigned)(key >> 32);
    const unsigned best_h = 0xffffffffu - (unsigned)(key & 0xffffffffu);
    float2 wp = make_float2(0.f, 0.f);
    if (win_in) wp = win_in[bk];                 // refinement round: the caller's point instead of the winner
    else if (best_cnt > 0) wp = hyp[(size_t)bk * HT + best_h];
    if (rc == 0 && tid == 0) win[bk] = wp;

    const int per = (tn + RF_CHUNKS - 1) / RF_CHUNKS;
    const int lo = rc * per, hi = min(tn, lo + per);
    const float2 *dir_k = direct + (size_t)bk * cap;
    (void)k;
    double a00 = 0, a01 = 0, a11 = 0, b0 = 0, b1 = 0;
    for (int t = lo + tid; t < hi; t += RF_THREADS) {
        const unsigned p = pix[(size_t)b * npx + t];
        const int x = p & 0xffff, y = p >> 16;
        const float2 dv = dir_k[t];
        const float dxv = dv.x, dyv = dv.y;
        if (exact_inlier(dxv, dyv, (float)x, (float)y, wp.x, wp.y, thresh)) {
            const double n0 = (double)dyv, n1 = -(double)dxv;
            const double bb = n0 * (double)x + n1 * (double)y;
            a00 += n0 * n0;
            a01 += n0 * n1;
            a11 += n1 * n1;
            b0 += n0 * bb;
            b1 += n1 * bb;
        }
    }
    a00 = warp_sum_d(a00);
    a01 = warp_sum_d(a01);
    a11 = warp_sum_d(a11);
    b0 = warp_sum_d(b0);
    b1 = warp_sum_d(b1);
    if (lane == 0) {
        s_acc[warp][0] = a00;
        s_acc[warp][1] = a01;
        s_acc[warp][2] = a11;
        s_acc[warp][3] = b0;
        s_acc[warp][4] = b1;
    }
    __syncthreads();
    if (tid < 5) {
        double v = 0;
        for (int i = 0; i < RF_THREADS / 32; ++i) v += s_acc[i][tid];
        my_part[tid] = v;
    }
}

// thread per (image, keypoint): fixed-order sum of the partials, 2x2 solve (:594)
__global__ void k_refit_final(const double *__restrict__ part, const int *__restrict__ tn_arr, int nb, int vn,
                              float *__restrict__ out_pts)
{
    const int bk = blockIdx.x * blockDim.x + threadIdx.x;
    if (bk >= nb * vn) return;
    const int b = bk / vn;
    float px = 0.f, py = 0.f;
    if (tn_arr[b] > 0) {
        double a[5] = {0, 0, 0, 0, 0};
        for (int rc = 0; rc < RF_CHUNKS; ++rc)
            for (int i = 0; i < 5; ++i) a[i] += part[((size_t)bk * RF_CHUNKS + rc) * 5 + i];
        const double det = a[0] * a[2] - a[1] * a[1];
        px = (float)((a[2] * a[3] - a[1] * a[4]) / det);
        py = (float)((a[0] * a[4] - a[1] * a[3]) / det);
    }
    out_pts[bk * 2] = px;
    out_pts[bk * 2 + 1] = py;
}

// ransac_voting_layer_v5's confidence (ransac_voting_gpu.py:850-852): inliers of the REFITTED
// point at a fixed threshold, divided by the pixel count.  grid (RF_CHUNKS, b*vn), integer atomics.
__global__ void __launch_bounds__(RF_THREADS)
    k_conf_count(const float2 *__restrict__ direct, int cap, const unsigned *__restrict__ pix,
                 const int *__restrict__ tn_arr, int npx, int vn, const float *__restrict__ pts, float thresh,
                 int *__restrict__ conf_cnt)
{
    __shared__ int scratch[96];
    const int rc = blockIdx.x, bk = blockIdx.y, b = bk / vn;
    const int tn = tn_arr[b];
    if (tn == 0) return;
    const float hx = pts[bk * 2], hy = pts[bk * 2 + 1];
    const int per = (tn + RF_CHUNKS - 1) / RF_CHUNKS;
    const int lo = rc * per, hi = min(tn, lo + per);
    const float2 *dir_k = direct + (size_t)bk * cap;
    int c = 0, z0 = 0, z1 = 0;
    for (int t = lo + threadIdx.x; t < hi; t += RF_THREADS) {
        const unsigned p = pix[(size_t)b * npx + t];
        const int x = p & 0xffff, y = p >> 16;
        const float2 dv = dir_k[t];
        c += exact_inlier(dv.x, dv.y, (float)x, (float)y, hx, hy, thresh) ? 1 : 0;
    }
    block_sum3(c, z0, z1, scratch);
    if (threadIdx.x == 0 && c) atomicAdd(conf_cnt + bk, c);
}

__global__ void k_conf_final(const int *__restrict__ conf_cnt, const int *__restrict__ tn_arr, int nb, int vn,
                             float *__restrict__ out_conf)
{
    const int bk = blockIdx.x * blockDim.x + threadIdx.x;
    if (bk >= nb * vn) return;
    const int tn = tn_arr[bk / vn];
    out_conf[bk] = tn > 0 ? __fdiv_rn((float)conf_cnt[bk], (float)tn) : 0.f;   // skipped image: zeros (:792)
}

// ------------------------------------------------------------------ v4 residual variance, motion voting
// block-wide fixed-order sum of two doubles (RF_THREADS threads); result valid in thread 0
__device__ __forceinline__ void block_sum2_d(double &a, double &b, double (*s_acc)[2])
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    a = warp_sum_d(a);
    b = warp_sum_d(b);
    if (lane == 0) {
        s_acc[warp][0] = a;
        s_acc[warp][1] = b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        a = b = 0.0;
        for (int i = 0; i < RF_THREADS / 32; ++i) {
            a += s_acc[i][0];
            b += s_acc[i][1];
        }
    }
}

// ransac_voting_layer_v4 (ransac_voting_gpu.py:733-752): over the inliers of the WINNING hypothesis
// (the set the refit used), residual r = n.p - n.c with n = (d_y,-d_x) and p the refitted point;
// partial sums of r^2 and of the inlier count in fp64.  grid (RF_CHUNKS, b*vn).
__global__ void __launch_bounds__(RF_THREADS)
    k_resid_sum(const float2 *__restrict__ direct, int cap, const unsigned *__restrict__ pix,
                const int *__restrict__ tn_arr, int npx, int vn, const float2 *__restrict__ win,
                const float *__restrict__ pts, float thresh, double *__restrict__ part)
{
    __shared__ double s_acc[RF_THREADS / 32][2];
    const int rc = blockIdx.x, bk = blockIdx.y, b = bk / vn;
    const int tn = tn_arr[b];
    double *my_part = part + ((size_t)bk * RF_CHUNKS + rc) * 2;
    double r2 = 0.0, cnt = 0.0;
    if (tn > 0) {
        const float2 wp = win[bk];
        const double px = (double)pts[bk * 2], py = (double)pts[bk * 2 + 1];
        const int per = (tn + RF_CHUNKS - 1) / RF_CHUNKS;
        const int lo = rc * per, hi = min(tn, lo + per);
        const float2 *dir_k = direct + (size_t)bk * cap;
        for (int t = lo + threadIdx.x; t < hi; t += RF_THREADS) {
            const unsigned p = pix[(size_t)b * npx + t];
            const int x = p & 0xffff, y = p >> 16;
            const float2 dv = dir_k[t];
            const float dxv = dv.x, dyv = dv.y;
            if (exact_inlier(dxv, dyv, (float)x, (float)y, wp.x, wp.y, thresh)) {
                const double n0 = (double)dyv, n1 = -(double)dxv;
                const double r = n0 * px + n1 * py - (n0 * (double)x + n1 * (double)y);
                r2 += r * r;
                cnt += 1.0;
            }
        }
    }
    block_sum2_d(r2, cnt, s_acc);
    if (threadIdx.x == 0) {
        my_part[0] = r2;
        my_part[1] = cnt;
    }
}

// var = sum r^2 / #inliers (0/0 = NaN like torch); skipped image: 1 (:688)
__global__ void k_resid_final(const double *__restrict__ part, const int *__restrict__ tn_arr, int nb, int vn,
                              float *__restrict__ out_var)
{
    const int bk = blockIdx.x * blockDim.x + threadIdx.x;
    if (bk >= nb * vn) return;
    float v = 1.f;
    if (tn_arr[bk / vn] > 0) {
        double r2 = 0.0, cnt = 0.0;
        for (int rc = 0; rc < RF_CHUNKS; ++rc) {
            r2 += part[((size_t)bk * RF_CHUNKS + rc) * 2];
            cnt += part[((size_t)bk * RF_CHUNKS + rc) * 2 + 1];
        }
        v = (float)(r2 / cnt);
    }
    out_var[bk] = v;
}

// ransac_motion_voting (ransac_voting_gpu.py:960-981): sum over the foreground pixels of
// vertex + (x, y), fp64 partials.  grid (RF_CHUNKS, b*vn).
__global__ void __launch_bounds__(RF_THREADS)
    k_motion_sum(const float2 *__restrict__ direct, int cap, const unsigned *__restrict__ pix,
                 const int *__restrict__ tn_arr, int npx, int vn, double *__restrict__ part)
{
    __shared__ double s_acc[RF_THREADS / 32][2];
    const int rc = blockIdx.x, bk = blockIdx.y, b = bk / vn;
    const int tn = tn_arr[b];
    double sx = 0.0, sy = 0.0;
    const int per = (tn + RF_CHUNKS - 1) / RF_CHUNKS;
    const int lo = rc * per, hi = min(tn, lo + per);
    const float2 *dir_k = direct + (size_t)bk * cap;
    for (int t = lo + threadIdx.x; t < hi; t += RF_THREADS) {
        const unsigned p = pix[(size_t)b * npx + t];
        const int x = p & 0xffff, y = p >> 16;
        const float2 dv = dir_k[t];
        // the reference adds in fp32 before averaging: cur_vert[cur_mask] + coords (:978)
        sx += (double)__fadd_rn(dv.x, (float)x);
        sy += (double)__fadd_rn(dv.y, (float)y);
    }
    block_sum2_d(sx, sy, s_acc);
    if (threadIdx.x == 0) {
        double *my_part = part + ((size_t)bk * RF_CHUNKS + rc) * 2;
        my_part[0] = sx;
        my_part[1] = sy;
    }
}

__global__ void k_motion_final(const double *__restrict__ part, const int *__restrict__ tn_arr, int nb, int vn,
                               float *__restrict__ out_pts)
{
    const int bk = blockIdx.x * blockDim.x + threadIdx.x;
    if (bk >= nb * vn) return;
    const int tn = tn_arr[bk / vn];
    float px = 0.f, py = 0.f;      // empty mask: zeros (:971-973)
    if (tn > 0) {
        double sx = 0.0, sy = 0.0;
        for (int rc = 0; rc < RF_CHUNKS; ++rc) {
            sx += part[((size_t)bk * RF_CHUNKS + rc) * 2];
            sy += part[((size_t)bk * RF_CHUNKS + rc) * 2 + 1];
        }
        px = (float)(sx / (double)tn);
        py = (float)(sy / (double)tn);
    }
    out_pts[bk * 2] = px;
    out_pts[bk * 2 + 1] = py;
}

// internal [b][vn][hn] -> API layouts [b,hn,vn(,2)]
__global__ void k_export(const float2 *__restrict__ hyp, const int *__restrict__ counts,
                         const int *__restrict__ tn_arr, int nb, int vn, int hn, int HT, int h_off,
                         float *__restrict__ out_hyp, int *__restrict__ out_counts, int *__restrict__ out_tn)
{
    const long long n = (long long)nb * vn * hn;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
         i += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(i % vn);
        const long long r = i / vn;
        const int h = (int)(r % hn);
        const int b = (int)(r / hn);
        const size_t src = ((size_t)b * vn + k) * HT + h_off + h;
        if (out_counts) out_counts[i] = counts[src];
        if (out_hyp) {
            const float2 v = hyp[src];
            out_hyp[i * 2] = v.x;
            out_hyp[i * 2 + 1] = v.y;
        }
    }
    if (out_tn && blockIdx.x == 0)
        for (int i = threadIdx.x; i < nb; i += blockDim.x) out_tn[i] = tn_arr[i];
}

// ------------------------------------------------------------------ covariance
// block per (image, keypoint); ransac_voting_gpu.py:392-401
__global__ void __launch_bounds__(256)
    k_cov(const float2 *__restrict__ hyp_all, const int *__restrict__ counts_all, const int *__restrict__ tn_arr,
          const float *__restrict__ mean, int vn, int hn, int HT, int h_off, int min_hyp_num,
          float *__restrict__ out_cov)
{
    // this (image, keypoint)'s row of hn hypotheses inside the [b][vn][HT] tables
    const float2 *hyp = hyp_all + (size_t)blockIdx.x * HT + h_off;
    const int *counts = counts_all + (size_t)blockIdx.x * HT + h_off;
    __shared__ int s_max[8];
    __shared__ double s_acc[8][5];
    const int bk = blockIdx.x, b = bk / vn;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tn = tn_arr[b];
    const float mx = mean[bk * 2], my = mean[bk * 2 + 1];
    const bool skipped = tn == 0;
    const int rows = skipped ? min_hyp_num : hn;       // :343-348 vs :363-384
    int cmax = 0;
    if (!skipped)
        for (int h = tid; h < hn; h += 256) cmax = max(cmax, counts[h]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = max(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
    if (lane == 0) s_max[warp] = cmax;
    __syncthreads();
    cmax = s_max[0];
    for (int i = 1; i < 8; ++i) cmax = max(cmax, s_max[i]);
    const float ftn = (float)tn;
    const float rmax = skipped ? 1.0f : __fdiv_rn((float)cmax, ftn);
    const float thr = __fsub_rn(rmax, 0.1f);                                       // :394
    double c00 = 0, c01 = 0, c10 = 0, c11 = 0, ws = 0;
    for (int h = tid; h < rows; h += 256) {
        float w, hxv, hyv;
        if (skipped) {
            w = 1.0f;
            hxv = 0.f;
            hyv = 0.f;
        } else {
            w = __fdiv_rn((float)counts[h], ftn);
            const float2 hp = hyp[h];
            hxv = hp.x;
            hyv = hp.y;
        }
        if (w < thr) w = 0.0f;                                                     // :395
        const float dx = __fsub_rn(hxv, mx), dy = __fsub_rn(hyv, my);              // :398
        const float wdx = __fmul_rn(dx, w), wdy = __fmul_rn(dy, w);                // :399
        c00 += (double)dx * (double)wdx;                                           // :400
        c01 += (double)dx * (double)wdy;
        c10 += (double)dy * (double)wdx;
        c11 += (double)dy * (double)wdy;
        ws += (double)w;
    }
    c00 = warp_sum_d(c00);
    c01 = warp_sum_d(c01);
    c10 = warp_sum_d(c10);
    c11 = warp_sum_d(c11);
    ws = warp_sum_d(ws);
    if (lane == 0) {
        s_acc[warp][0] = c00;
        s_acc[warp][1] = c01;
        s_acc[warp][2] = c10;
        s_acc[warp][3] = c11;
        s_acc[warp][4] = ws;
    }
    __syncthreads();
    if (tid == 0) {
        double a[5] = {0, 0, 0, 0, 0};
        for (int i = 0; i < 8; ++i)
            for (int j = 0; j < 5; ++j) a[j] += s_acc[i][j];
        const float den = __fadd_rn((float)a[4], 1e-3f);                           // :401
        for (int j = 0; j < 4; ++j) out_cov[(size_t)bk * 4 + j] = __fdiv_rn((float)a[j], den);
    }
}

// ------------------------------------------------------------------ 1:1 stand-ins
__global__ void k_compat_gen_hyp(const float *__restrict__ direct, const float *__restrict__ coords,
                                 const int *__restrict__ idxs, float *__restrict__ hypo, int tn, int vn, int hn)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hn * vn) return;
    const int vi = i % vn;
    const int t0 = idxs[i * 2], t1 = idxs[i * 2 + 1];
    (void)tn;
    const float2 r = exact_hypothesis(direct[((size_t)t0 * vn + vi) * 2], direct[((size_t)t0 * vn + vi) * 2 + 1],
                                      coords[(size_t)t0 * 2], coords[(size_t)t0 * 2 + 1],
                                      direct[((size_t)t1 * vn + vi) * 2], direct[((size_t)t1 * vn + vi) * 2 + 1],
                                      coords[(size_t)t1 * 2], coords[(size_t)t1 * 2 + 1]);
    hypo[i * 2] = r.x;
    hypo[i * 2 + 1] = r.y;
}

// grid (ceil(tn/256), vn, hn)
__global__ void k_compat_vote(const float *__restrict__ direct, const float *__restrict__ coords,
                              const float *__restrict__ hypo, unsigned char *__restrict__ inliers, int tn, int vn,
                              int hn, float thresh)
{
    const int ti = blockIdx.x * blockDim.x + threadIdx.x;
    const int vi = blockIdx.y, hi = blockIdx.z;
    if (ti >= tn) return;
    (void)hn;
    if (exact_inlier(direct[((size_t)ti * vn + vi) * 2], direct[((size_t)ti * vn + vi) * 2 + 1],
                     coords[(size_t)ti * 2], coords[(size_t)ti * 2 + 1], hypo[(hi * vn + vi) * 2],
                     hypo[(hi * vn + vi) * 2 + 1], thresh))
        inliers[((size_t)hi * vn + vi) * tn + ti] = 1;
}

// block per (hypothesis, keypoint): exact predicate, block-summed
__global__ void __launch_bounds__(256)
    k_compat_counts(const float *__restrict__ direct, const float *__restrict__ coords,
                    const float *__restrict__ hypo, int *__restrict__ counts, int tn, int vn, float thresh)
{
    __shared__ int scratch[96];
    const int vi = blockIdx.x, hi = blockIdx.y;
    const float hx = hypo[(hi * vn + vi) * 2], hy = hypo[(hi * vn + vi) * 2 + 1];
    int c = 0, z0 = 0, z1 = 0;
    for (int ti = threadIdx.x; ti < tn; ti += blockDim.x)
        c += exact_inlier(direct[((size_t)ti * vn + vi) * 2], direct[((size_t)ti * vn + vi) * 2 + 1],
                          coords[(size_t)ti * 2], coords[(size_t)ti * 2 + 1], hx, hy, thresh)
                 ? 1
                 : 0;
    block_sum3(c, z0, z1, scratch);
    if (threadIdx.x == 0) counts[hi * vn + vi] = c;
}

// ------------------------------------------------------------------ vanishing-point pair
// 1:1 stand-ins for generate_hypothesis_vanishing_point / voting_for_hypothesis_vanishing_point
// (src/ransac_voting_kernel.cu:170-230, :263-305): homogeneous intersections [hn,vn,3] of the two pixels'
// lines and the |cos| test against them.  Rounding sequence read off the SASS nvcc 12.9 emits for the
// reference file (default -fmad): every fma below is one the compiler contracted, every
// __fmul_rn a product it kept separate because the value is used twice.
__device__ __forceinline__ void exact_vp_hypothesis(float dx0, float dy0, float cx0, float cy0, float dx1, float dy1,
                                                    float cx1, float cy1, float &ox, float &oy, float &oz)
{
    const float lz0 = __fmaf_rn(dx0, cy0, -__fmul_rn(dy0, cx0));      // cy0*dx0 - cx0*dy0   (:197)
    const float lz1 = __fmaf_rn(dx1, cy1, -__fmul_rn(dy1, cx1));      //                     (:201)
    float z = __fmaf_rn(dx0, dy1, -__fmul_rn(dy0, dx1));              // lx0*ly1 - ly0*lx1   (:206)
    float x = __fmaf_rn(dx1, lz0, -__fmul_rn(dx0, lz1));              // ly0*lz1 - lz0*ly1   (:204)
    float y = __fmaf_rn(dy1, lz0, -__fmul_rn(dy0, lz1));              // lz0*lx1 - lx0*lz1   (:205)
    const float vx0 = __fmul_rn(dx0, __fmaf_rn(-cx0, z, x)), vx1 = __fmul_rn(dx1, __fmaf_rn(-cx1, z, x));   // :209-210
    const float vy0 = __fmul_rn(dy0, __fmaf_rn(-cy0, z, y)), vy1 = __fmul_rn(dy1, __fmaf_rn(-cy1, z, y));   // :211-212
    if (vx0 < 0.f && vx1 < 0.f && vy0 < 0.f && vy1 < 0.f) {            // :214-215
        x = -x;
        y = -y;
        z = -z;
    }
    // :217-218 `val_x0*val_x1<0 || val_y0*val_y1<0` as the compiler evaluates it: min of the two products
    // (FMNMX returns the non-NaN operand), zeroed unless it is >= 0 or unordered
    const float m = fminf(__fmul_rn(vx0, vx1), __fmul_rn(vy0, vy1));
    if (m < 0.f) x = y = z = 0.f;
    ox = x;
    oy = y;
    oz = z;
}

__device__ __forceinline__ bool exact_vp_inlier(float dx, float dy, float cx, float cy, float hx, float hy, float hz,
                                                float thresh)
{
    const float fx = __fmaf_rn(-cx, hz, hx), fy = __fmaf_rn(-cy, hz, hy);              // :287-288
    const float norm1 = __fsqrt_rn(__fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
    const float norm2 = __fsqrt_rn(__fmaf_rn(fx, fx, __fmul_rn(fy, fy)));
    if (fmin((double)norm1, (double)norm2) < 1e-6) return false;                       // :292
    const float vx = __fmul_rn(fx, dx), vy = __fmul_rn(fy, dy);                        // :295-296 (reused by :294)
    const float ang = __fdiv_rn(__fadd_rn(vx, vy), __fmul_rn(norm2, norm1));
    if (fminf(vx, vy) < 0.f) return false;                                             // :297
    return fabsf(ang) > thresh;                                                        // :298
}

__global__ void k_compat_vp_gen_hyp(const float *__restrict__ direct, const float *__restrict__ coords,
                                    const int *__restrict__ idxs, float *__restrict__ hypo, int vn, int hn)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hn * vn) return;
    const int vi = i % vn;
    const int t0 = idxs[i * 2], t1 = idxs[i * 2 + 1];
    float x, y, z;
    exact_vp_hypothesis(direct[((size_t)t0 * vn + vi) * 2], direct[((size_t)t0 * vn + vi) * 2 + 1],
                        coords[(size_t)t0 * 2], coords[(size_t)t0 * 2 + 1], direct[((size_t)t1 * vn + vi) * 2],
                        direct[((size_t)t1 * vn + vi) * 2 + 1], coords[(size_t)t1 * 2], coords[(size_t)t1 * 2 + 1], x, y,
                        z);
    hypo[i * 3] = x;
    hypo[i * 3 + 1] = y;
    hypo[i * 3 + 2] = z;
}

// block per (keypoint, hypothesis): optional u8 inlier rows [hn,vn,tn] (only SET, like the reference)
// and/or the row sums [hn,vn]
__global__ void __launch_bounds__(256)
    k_compat_vp_vote(const float *__restrict__ direct, const float *__restrict__ coords, const float *__restrict__ hypo,
                     unsigned char *__restrict__ inliers, int *__restrict__ counts, int tn, int vn, float thresh)
{
    __shared__ int scratch[96];
    const int vi = blockIdx.x, hi = blockIdx.y;
    const float hx = hypo[(hi * vn + vi) * 3], hy = hypo[(hi * vn + vi) * 3 + 1], hz = hypo[(hi * vn + vi) * 3 + 2];
    int c = 0, z0 = 0, z1 = 0;
    for (int ti = threadIdx.x; ti < tn; ti += blockDim.x) {
        const bool in = exact_vp_inlier(direct[((size_t)ti * vn + vi) * 2], direct[((size_t)ti * vn + vi) * 2 + 1],
                                        coords[(size_t)ti * 2], coords[(size_t)ti * 2 + 1], hx, hy, hz, thresh);
        if (in && inliers) inliers[((size_t)hi * vn + vi) * tn + ti] = 1;
        c += in ? 1 : 0;
    }
    if (counts) {
        block_sum3(c, z0, z1, scratch);
        if (threadIdx.x == 0) counts[hi * vn + vi] = c;
    }
}

// ------------------------------------------------------------------ host side
struct VoteWs {
    unsigned *pix;
    int *chunk_fg, *chunk_kept, *tn, *fg, *status, *counts;
    float2 *hyp, *win, *direct;
    unsigned *ticket;
    double *part;
    int cap, ntile;      // per-image capacity of the compact lists (pixels, multiple of VT_TILE) and tiles
    size_t bytes;
};

VoteWs carve(void *ws, int b, int h, int w, int vn, int hn_total)
{
    const size_t npx = (size_t)h * w;
    const int nchunk = (int)((npx + CH_PX - 1) / CH_PX);
    Carver c(ws);
    VoteWs v;
    v.ntile = (int)((npx + VT_TILE - 1) / VT_TILE);
    v.cap = v.ntile * VT_TILE;
    v.pix = c.take<unsigned>((size_t)b * npx);
    v.chunk_fg = c.take<int>((size_t)b * nchunk);
    v.chunk_kept = c.take<int>((size_t)b * nchunk);
    v.tn = c.take<int>(b);
    v.fg = c.take<int>(b);
    v.status = c.take<int>(b);
    v.ticket = c.take<unsigned>(1);
    v.counts = c.take<int>((size_t)b * vn * hn_total);
    v.hyp = c.take<float2>((size_t)b * vn * hn_total);
    v.win = c.take<float2>((size_t)b * vn);
    v.part = c.take<double>((size_t)b * vn * RF_CHUNKS * 5);
    v.direct = c.take<float2>((size_t)b * vn * v.cap);
    v.bytes = pvnet::align_up(c.off, 256);
    return v;
}

int check_common(const void *mask, int mask_elem_size, const float *vertex, const long long *strides, int b, int h,
                 int w, int vn, int hn)
{
    PV_CHECK_ARG(mask && vertex && strides, "null mask/vertex/strides pointer");
    PV_CHECK_ARG(mask_elem_size == 1 || mask_elem_size == 2 || mask_elem_size == 4 || mask_elem_size == 8,
                 "mask element size %d not in {1,2,4,8}", mask_elem_size);
    PV_CHECK_ARG(b >= 1 && b <= VT_MAX_B, "batch %d outside [1,%d]", b, VT_MAX_B);
    PV_CHECK_ARG(h >= 1 && w >= 1 && h <= 65535 && w <= 65535, "image size %dx%d unsupported", h, w);
    PV_CHECK_ARG(vn >= 1 && vn <= 65535, "keypoint count %d unsupported", vn);
    PV_CHECK_ARG(hn >= 1 && hn <= (1 << 24), "hypothesis count %d unsupported", hn);
    return PVNET_OK;
}

// Where the samples come from: the caller's tensors (parity tests, rng="reference") or the device
// generator.  idxs == nullptr needs rng_state; selection == nullptr && rng_state == nullptr means
// "never subsample".
struct Samples {
    const int32_t *idxs;
    const float *selection;
    const unsigned long long *rng_state;
};

template <typename T>
int launch_compaction_t(const T *mask, int mode, const Samples &sm, int b, int h, int w, int min_num, int max_num,
                        const VoteWs &ws, cudaStream_t s)
{
    const int npx = h * w;
    const int nchunk = (npx + CH_PX - 1) / CH_PX;
    dim3 grid(nchunk, b);
    k_chunk_count<T><<<grid, CH_THREADS, 0, s>>>(mask, mode, npx, nchunk, ws.chunk_fg);
    PV_LAUNCHED("k_chunk_count");
    // the kept-count pass is only needed when an image could be subsampled
    const bool may_sub = (sm.selection != nullptr || sm.rng_state != nullptr) && max_num < npx;
    if (may_sub) {
        k_chunk_kept<T><<<grid, CH_THREADS, 0, s>>>(mask, mode, sm.selection, sm.rng_state, npx, nchunk, min_num, max_num,
                                                    ws.chunk_fg, ws.chunk_kept, ws.status);
        PV_LAUNCHED("k_chunk_kept");
    }
    k_compact_write<T><<<grid, CH_THREADS, 0, s>>>(mask, mode, sm.selection, sm.rng_state, npx, w, nchunk, min_num,
                                                   max_num, ws.chunk_fg, may_sub ? ws.chunk_kept : nullptr, ws.pix,
                                                   ws.tn, ws.fg);
    PV_LAUNCHED("k_compact_write");
    return PVNET_OK;
}

// mask -> stable pixel list -> compact direct lists + tile boxes (everything the scoring passes read)
int launch_pixels(const void *mask, int esz, int mode, const float *vertex, const Strides &st, const Samples &sm,
                  int b, int h, int w, int vn, int min_num, int max_num, const VoteWs &ws, cudaStream_t s)
{
    int rc;
    switch (esz) {
    case 1: rc = launch_compaction_t((const unsigned char *)mask, mode, sm, b, h, w, min_num, max_num, ws, s); break;
    case 2: rc = launch_compaction_t((const short *)mask, mode, sm, b, h, w, min_num, max_num, ws, s); break;
    case 4: rc = launch_compaction_t((const int *)mask, mode, sm, b, h, w, min_num, max_num, ws, s); break;
    default: rc = launch_compaction_t((const long long *)mask, mode, sm, b, h, w, min_num, max_num, ws, s); break;
    }
    if (rc) return rc;
    dim3 grid(ws.ntile, b);
    k_gather<<<grid, 256, 0, s>>>(vertex, st, ws.pix, ws.tn, h * w, ws.cap, vn, ws.direct);
    PV_LAUNCHED("k_gather");
    return PVNET_OK;
}

// hypotheses of one sample set into columns [h_off, h_off + hn) of the [b][vn][HT] tables
int launch_gen_hyp(const Samples &sm, int rng_stream, int b, int h, int w, int vn, int hn, int HT, int h_off,
                   const VoteWs &ws, cudaStream_t s)
{
    PV_CHECK_ARG(sm.idxs || sm.rng_state, "neither idxs nor an rng state given");
    dim3 ghyp((hn * vn + 255) / 256, b);
    k_gen_hyp<<<ghyp, 256, 0, s>>>(ws.direct, sm.idxs, sm.rng_state, rng_stream, ws.pix, ws.tn, h * w, ws.cap, vn, hn, HT,
                                   h_off, ws.hyp);
    PV_LAUNCHED("k_gen_hyp");
    return PVNET_OK;
}

// Guard-band constants of k_vote3 for a threshold T (DESIGN.md section 3).  With u = 2^-24:
//   reference: fl(cos) = cos (1 + delta), |delta| <= eta = (7 + 1/T) u  (two sqrt of an fma, the fma of
//   the numerator with its inner product, one multiply, one division) plus u rad from rounding d;
//   in m = |d| sin(theta_T - |theta|) that is a band of (eta T / sin(theta_T) + u) |d|;
//   ours: unit vector, functionals, centring and the two fma chains: < 8 u (|h'|_1 + r1).
// beta = 1.25 (1.1 eta T / s + u) + 16 u; b0 = 1e-5 covers |d| < 1e-6 (norm test of the reference).
// Outside T in [0.05, 1 - 1e-6] (and for NaN) beta is NaN: every test takes the exact path.
struct VoteConsts {
    float sn, cs, beta, b0;
};
VoteConsts vote_consts(float thresh)
{
    VoteConsts c;
    const double T = (double)thresh, u = 5.9604644775390625e-8;
    if (T >= 0.05 && T <= 1.0 - 1e-6) {
        const double sn = sqrt(1.0 - T * T);
        const double eta = (7.0 + 1.0 / T) * u * 1.05;
        c.sn = (float)sn;
        c.cs = (float)T;
        c.beta = (float)(1.25 * (1.1 * eta * T / sn + u) + 16.0 * u);
    } else {
        c.sn = 0.f;
        c.cs = 1.f;
        c.beta = nanf("");
    }
    c.b0 = 1e-5f;
    return c;
}

// score columns [h0, h0 + hn) of the hypothesis tables (counts must be zero there)
int launch_vote(const float *vertex, const Strides &st, int b, int h, int w, int vn, int hn, int HT, int h0, float thresh,
                const VoteWs &ws, cudaStream_t s)
{
    const int npx = h * w;
    static const int impl = [] {
        const char *e = getenv("PVNET_VOTE_IMPL");     // tuning knob: 0 = round-1 kernel (k_vote, A/B), 3 = k_vote3 (default)
        return e ? atoi(e) : 3;
    }();
    static const int hpl_env = [] {
        const char *e = getenv("PVNET_VOTE_HPL");      // tuning knob: hypotheses per lane of k_vote3 (4 or 8)
        return e ? atoi(e) : 8;
    }();
    const int HPL = (impl != 0 && hpl_env == 8 && hn > 128) ? 8 : 4;
    static const int ctas_per_sm = [] {
        const char *e = getenv("PVNET_VOTE_CTAS");     // tuning knob: resident vote CTAs per SM
        return e ? atoi(e) : 0;
    }();
    if (impl == 0) {
        int wh = 1;                                    // hypothesis warps per CTA: 128 hypotheses per warp
        while (wh < VT_WARPS && wh * 32 * 4 < hn) wh <<= 1;
        const int HC = wh * 32 * 4;
        const long long max_items = (long long)b * ((npx + VT_TILE - 1) / VT_TILE) * vn * ((hn + HC - 1) / HC);
        long long grid = (long long)pvnet::sm_count() * (ctas_per_sm > 0 ? ctas_per_sm : 4);
        if (grid > max_items) grid = max_items;
        if (grid < 1) grid = 1;
        // thresh <= 0 (or NaN) has no squared form: NaN makes every test take the exact path
        const float t2 = (thresh > 0.f && thresh < 1e18f) ? thresh * thresh : nanf("");
        const float band = GUARD_EPS * (thresh > 0.f ? thresh * thresh : 1.f);
        k_vote<4, VT_TILE><<<(unsigned)grid, VT_THREADS, 0, s>>>(vertex, st, ws.pix, ws.tn, npx, b, vn, hn, HT, h0, wh,
                                                                 ws.hyp, ws.counts, thresh, t2, band);
        PV_LAUNCHED("k_vote");
        return PVNET_OK;
    }
    const VoteConsts vc = vote_consts(thresh);
    const int per_sm = ctas_per_sm > 0 ? ctas_per_sm : (HPL > 4 ? 2 : 3);
    const unsigned grid = (unsigned)(pvnet::sm_count() * per_sm);
    PV_CUDA(cudaMemsetAsync(ws.ticket, 0, sizeof(unsigned), s));
    static const int grp = [] {
        const char *e = getenv("PVNET_VOTE_GROUP");    // tuning knob: pixels per unrolled step of the sweep (4 or 8)
        return e ? atoi(e) : 4;
    }();
    static const int items_pw = [] {
        const char *e = getenv("PVNET_VOTE_ITEMS");    // tuning knob: work items per resident warp the segment length aims at
        return e ? atoi(e) : 16;                       // (config-4 layer: 3.96 / 3.81 / 3.73 / 3.73 ms at 6 / 10 / 16 / 24)
    }();
#define VOTE3(H_, G_)                                                                                                  \
    k_vote3<H_, G_><<<grid, VT_THREADS, 0, s>>>(ws.pix, ws.direct, ws.tn, npx, ws.cap, b, vn, hn, HT, h0, ws.hyp, ws.counts, \
                                                ws.ticket, thresh, vc.sn, vc.cs, vc.beta, vc.b0, items_pw)
    if (HPL == 8 && grp == 8) VOTE3(8, 8);
    else if (HPL == 8) VOTE3(8, 4);
    else if (grp == 8) VOTE3(4, 8);
    else VOTE3(4, 4);
#undef VOTE3
    PV_LAUNCHED("k_vote3");
    return PVNET_OK;
}

int launch_refit(int b, int h, int w, int vn, int hn, int HT, float thresh, const VoteWs &ws, float *out_pts,
                 cudaStream_t s, const float2 *win_in = nullptr)
{
    dim3 grf(RF_CHUNKS, b * vn);
    k_refit<<<grf, RF_THREADS, 0, s>>>(ws.direct, ws.cap, ws.pix, ws.tn, h * w, vn, hn, HT, ws.hyp, ws.counts, thresh,
                                       ws.part, ws.win, win_in);
    PV_LAUNCHED("k_refit");
    k_refit_final<<<(b * vn + 127) / 128, 128, 0, s>>>(ws.part, ws.tn, b, vn, out_pts);
    PV_LAUNCHED("k_refit_final");
    return PVNET_OK;
}

int launch_export(const VoteWs &ws, int b, int vn, int hn, int HT, int h_off, float *out_hyp, int32_t *out_counts,
                  int32_t *out_tn, cudaStream_t s)
{
    if (!out_hyp && !out_counts && !out_tn) return PVNET_OK;
    const long long n = (long long)b * vn * hn;
    int grid = (int)((n + 255) / 256);
    if (grid > 4096) grid = 4096;
    if (grid < 1) grid = 1;
    k_export<<<grid, 256, 0, s>>>(ws.hyp, ws.counts, ws.tn, b, vn, hn, HT, h_off, out_hyp, out_counts, out_tn);
    PV_LAUNCHED("k_export");
    return PVNET_OK;
}

int finish_rng(const Samples &sm, cudaStream_t s)
{
    if (!sm.rng_state) return PVNET_OK;
    k_rng_bump<<<1, 1, 0, s>>>(const_cast<unsigned long long *>(sm.rng_state));
    PV_LAUNCHED("k_rng_bump");
    return PVNET_OK;
}

int ws_check(const VoteWs &ws, void *workspace, size_t workspace_bytes)
{
    PV_CHECK_ARG(workspace, "null workspace");
    if (workspace_bytes < ws.bytes) {
        pvnet::set_error("workspace %zu < %zu bytes", workspace_bytes, ws.bytes);
        return PVNET_E_WORKSPACE;
    }
    return PVNET_OK;
}

Strides to_strides(const int64_t *vs)
{
    Strides st;
    for (int i = 0; i < 5; ++i) st.s[i] = vs ? vs[i] : 0;
    return st;
}

}  // namespace

// ====================================================================== C ABI
extern "C" {

int pvnet_vote_workspace_bytes(int b, int h, int w, int vn, int hn_total, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "null bytes pointer");
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && vn >= 1 && hn_total >= 1, "non-positive dimension");
    *bytes = carve(nullptr, b, h, w, vn, hn_total).bytes + 256;
    return PVNET_OK;
}

int pvnet_mask_foreground_count(const void *mask, int mask_elem_size, int mask_mode, int b, int h, int w,
                                int32_t *fg_out, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(mask && fg_out && workspace, "null pointer");
    PV_CHECK_ARG(b >= 1 && b <= VT_MAX_B && h >= 1 && w >= 1 && h <= 65535 && w <= 65535, "bad shape");
    const int npx = h * w, nchunk = (npx + CH_PX - 1) / CH_PX;
    if (workspace_bytes < sizeof(int) * (size_t)b * nchunk) {
        pvnet::set_error("workspace %zu < %zu bytes", workspace_bytes, sizeof(int) * (size_t)b * nchunk);
        return PVNET_E_WORKSPACE;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int *chunk_fg = (int *)workspace;
    dim3 grid(nchunk, b);
    switch (mask_elem_size) {
    case 1: k_chunk_count<unsigned char><<<grid, CH_THREADS, 0, s>>>((const unsigned char *)mask, mask_mode, npx, nchunk, chunk_fg); break;
    case 2: k_chunk_count<short><<<grid, CH_THREADS, 0, s>>>((const short *)mask, mask_mode, npx, nchunk, chunk_fg); break;
    case 4: k_chunk_count<int><<<grid, CH_THREADS, 0, s>>>((const int *)mask, mask_mode, npx, nchunk, chunk_fg); break;
    case 8: k_chunk_count<long long><<<grid, CH_THREADS, 0, s>>>((const long long *)mask, mask_mode, npx, nchunk, chunk_fg); break;
    default: pvnet::set_error("mask element size %d not in {1,2,4,8}", mask_elem_size); return PVNET_E_INVALID;
    }
    PV_LAUNCHED("k_chunk_count");
    k_sum_chunks<<<b, 128, 0, s>>>(chunk_fg, nchunk, fg_out);
    PV_LAUNCHED("k_sum_chunks");
    return PVNET_OK;
}

int pvnet_ransac_voting_v3(const void *mask, int mask_elem_size, const float *vertex,
                           const int64_t vertex_strides[5], const int32_t *idxs, const float *selection, int b,
                           int h, int w, int vn, int hn, float inlier_thresh, int min_num, int max_num,
                           float *out_pts, int32_t *out_counts, float *out_hyp, int32_t *out_tn, void *workspace,
                           size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(idxs, "null idxs (use pvnet_ransac_voting_pipeline for device-side sampling)");
    int rc = check_common(mask, mask_elem_size, vertex, (const long long *)vertex_strides, b, h, w, vn, hn);
    if (rc) return rc;
    PV_CHECK_ARG(out_pts, "null out_pts");
    const Strides st = to_strides(vertex_strides);
    VoteWs ws = carve(workspace, b, h, w, vn, hn);
    if ((rc = ws_check(ws, workspace, workspace_bytes))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const Samples sm{idxs, selection, nullptr};
    if ((rc = launch_pixels(mask, mask_elem_size, PVNET_MASK_NONZERO_BYTE, vertex, st, sm, b, h, w, vn, min_num, max_num, ws, s))) return rc;
    PV_CUDA(cudaMemsetAsync(ws.counts, 0, sizeof(int) * (size_t)b * vn * hn, s));
    if ((rc = launch_gen_hyp(sm, RNG_IDXS_V3, b, h, w, vn, hn, hn, 0, ws, s))) return rc;
    if ((rc = launch_vote(vertex, st, b, h, w, vn, hn, hn, 0, inlier_thresh, ws, s))) return rc;
    if ((rc = launch_refit(b, h, w, vn, hn, hn, inlier_thresh, ws, out_pts, s))) return rc;
    return launch_export(ws, b, vn, hn, hn, 0, out_hyp, out_counts, out_tn, s);
}

int pvnet_refit_at_points(const void *mask, int mask_elem_size, const float *vertex, const int64_t vertex_strides[5],
                          const float *selection, const float *points, int b, int h, int w, int vn,
                          float inlier_thresh, int min_num, int max_num, float *out_pts, void *workspace,
                          size_t workspace_bytes, pvnet_stream_t stream)
{
    int rc = check_common(mask, mask_elem_size, vertex, (const long long *)vertex_strides, b, h, w, vn, 1);
    if (rc) return rc;
    PV_CHECK_ARG(points && out_pts, "null points/out_pts");
    const Strides st = to_strides(vertex_strides);
    VoteWs ws = carve(workspace, b, h, w, vn, 1);
    if ((rc = ws_check(ws, workspace, workspace_bytes))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const Samples sm{nullptr, selection, nullptr};
    if ((rc = launch_pixels(mask, mask_elem_size, PVNET_MASK_NONZERO_BYTE, vertex, st, sm, b, h, w, vn, min_num, max_num, ws, s))) return rc;
    return launch_refit(b, h, w, vn, 1, 1, inlier_thresh, ws, out_pts, s, reinterpret_cast<const float2 *>(points));
}

int pvnet_ransac_voting_v5(const void *mask, int mask_elem_size, const float *vertex,
                           const int64_t vertex_strides[5], const int32_t *idxs, const float *selection, int b,
                           int h, int w, int vn, int hn, float inlier_thresh, float conf_thresh, int min_num,
                           int max_num, float *out_pts, float *out_conf, int32_t *out_counts, float *out_hyp,
                           int32_t *out_tn, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(out_conf, "null out_conf");
    int rc = pvnet_ransac_voting_v3(mask, mask_elem_size, vertex, vertex_strides, idxs, selection, b, h, w, vn, hn,
                                    inlier_thresh, min_num, max_num, out_pts, out_counts, out_hyp, out_tn, workspace,
                                    workspace_bytes, stream);
    if (rc) return rc;
    VoteWs ws = carve(workspace, b, h, w, vn, hn);
    cudaStream_t s = (cudaStream_t)stream;
    int *conf_cnt = reinterpret_cast<int *>(ws.part);      // the refit partials are consumed by now
    PV_CUDA(cudaMemsetAsync(conf_cnt, 0, sizeof(int) * (size_t)b * vn, s));
    dim3 grid(RF_CHUNKS, b * vn);
    k_conf_count<<<grid, RF_THREADS, 0, s>>>(ws.direct, ws.cap, ws.pix, ws.tn, h * w, vn, out_pts, conf_thresh, conf_cnt);
    PV_LAUNCHED("k_conf_count");
    k_conf_final<<<(b * vn + 127) / 128, 128, 0, s>>>(conf_cnt, ws.tn, b, vn, out_conf);
    PV_LAUNCHED("k_conf_final");
    return PVNET_OK;
}

int pvnet_ransac_voting_v4(const void *mask, int mask_elem_size, const float *vertex,
                           const int64_t vertex_strides[5], const int32_t *idxs, const float *selection, int b,
                           int h, int w, int vn, int hn, float inlier_thresh, int min_num, int max_num,
                           float *out_pts, float *out_var, int32_t *out_counts, float *out_hyp, int32_t *out_tn,
                           void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(out_var, "null out_var");
    int rc = pvnet_ransac_voting_v3(mask, mask_elem_size, vertex, vertex_strides, idxs, selection, b, h, w, vn, hn,
                                    inlier_thresh, min_num, max_num, out_pts, out_counts, out_hyp, out_tn, workspace,
                                    workspace_bytes, stream);
    if (rc) return rc;
    VoteWs ws = carve(workspace, b, h, w, vn, hn);
    cudaStream_t s = (cudaStream_t)stream;
    dim3 grid(RF_CHUNKS, b * vn);                          // the refit partials are consumed by now
    k_resid_sum<<<grid, RF_THREADS, 0, s>>>(ws.direct, ws.cap, ws.pix, ws.tn, h * w, vn, ws.win, out_pts, inlier_thresh,
                                            ws.part);
    PV_LAUNCHED("k_resid_sum");
    k_resid_final<<<(b * vn + 127) / 128, 128, 0, s>>>(ws.part, ws.tn, b, vn, out_var);
    PV_LAUNCHED("k_resid_final");
    return PVNET_OK;
}

int pvnet_ransac_motion_voting(const void *mask, int mask_elem_size, const float *vertex,
                               const int64_t vertex_strides[5], int b, int h, int w, int vn, float *out_pts,
                               void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    int rc = check_common(mask, mask_elem_size, vertex, (const long long *)vertex_strides, b, h, w, vn, 1);
    if (rc) return rc;
    PV_CHECK_ARG(out_pts, "null out_pts");
    const Strides st = to_strides(vertex_strides);
    VoteWs ws = carve(workspace, b, h, w, vn, 1);
    if ((rc = ws_check(ws, workspace, workspace_bytes))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    // every foreground pixel takes part: min_num 1, no subsampling
    const Samples sm{nullptr, nullptr, nullptr};
    if ((rc = launch_pixels(mask, mask_elem_size, PVNET_MASK_NONZERO_BYTE, vertex, st, sm, b, h, w, vn, 1, 0x7fffffff, ws, s))) return rc;
    dim3 grid(RF_CHUNKS, b * vn);
    k_motion_sum<<<grid, RF_THREADS, 0, s>>>(ws.direct, ws.cap, ws.pix, ws.tn, h * w, vn, ws.part);
    PV_LAUNCHED("k_motion_sum");
    k_motion_final<<<(b * vn + 127) / 128, 128, 0, s>>>(ws.part, ws.tn, b, vn, out_pts);
    PV_LAUNCHED("k_motion_final");
    return PVNET_OK;
}

int pvnet_vote_cov_with_mean(const void *mask, int mask_elem_size, const float *vertex,
                             const int64_t vertex_strides[5], const int32_t *idxs, const float *selection,
                             const float *mean, int b, int h, int w, int vn, int hn, int rounds, int min_hyp_num,
                             float inlier_thresh, int min_num, int max_num, float *out_cov, int32_t *out_counts,
                             float *out_hyp, int32_t *out_tn, void *workspace, size_t workspace_bytes,
                             pvnet_stream_t stream)
{
    PV_CHECK_ARG(idxs, "null idxs (use pvnet_ransac_voting_pipeline for device-side sampling)");
    PV_CHECK_ARG(rounds >= 1 && min_hyp_num >= 1, "rounds/min_hyp_num must be positive");
    const long long hnt_ll = (long long)hn * rounds;
    PV_CHECK_ARG(hnt_ll <= (1 << 24), "too many hypotheses");
    const int hnt = (int)hnt_ll;
    int rc = check_common(mask, mask_elem_size, vertex, (const long long *)vertex_strides, b, h, w, vn, hnt);
    if (rc) return rc;
    PV_CHECK_ARG(out_cov && mean, "null out_cov/mean");
    const Strides st = to_strides(vertex_strides);
    VoteWs ws = carve(workspace, b, h, w, vn, hnt);
    if ((rc = ws_check(ws, workspace, workspace_bytes))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const Samples sm{idxs, selection, nullptr};
    if ((rc = launch_pixels(mask, mask_elem_size, PVNET_MASK_EQUALS_ONE, vertex, st, sm, b, h, w, vn, min_num, max_num, ws, s))) return rc;
    PV_CUDA(cudaMemsetAsync(ws.counts, 0, sizeof(int) * (size_t)b * vn * hnt, s));
    if ((rc = launch_gen_hyp(sm, RNG_IDXS_COV, b, h, w, vn, hnt, hnt, 0, ws, s))) return rc;
    if ((rc = launch_vote(vertex, st, b, h, w, vn, hnt, hnt, 0, inlier_thresh, ws, s))) return rc;
    k_cov<<<b * vn, 256, 0, s>>>(ws.hyp, ws.counts, ws.tn, mean, vn, hnt, hnt, 0, min_hyp_num, out_cov);
    PV_LAUNCHED("k_cov");
    return launch_export(ws, b, vn, hnt, hnt, 0, out_hyp, out_counts, out_tn, s);
}

// ransac_voting_layer_v3 followed by estimate_voting_distribution_with_mean on its result, the
// sequence of tools/train_linemod.py:119-130 (UncertaintyEvalWrapper), as ONE launch sequence: the
// mask is compacted and the field gathered once, and when both thresholds agree one k_vote3 launch
// scores the v3 and the covariance hypotheses together.  See include/pvnet_b200.h.
int pvnet_ransac_voting_pipeline(const void *mask, int mask_elem_size, int mask_mode, const float *vertex,
                                 const int64_t vertex_strides[5], const int32_t *idxs, const int32_t *cov_idxs,
                                 const float *selection, const unsigned long long *rng_state, int b, int h, int w,
                                 int vn, int hn, float inlier_thresh, int cov_hn, int cov_rounds, int cov_min_hyp_num,
                                 float cov_inlier_thresh, int min_num, int max_num, float *out_pts, float *out_cov,
                                 int32_t *out_counts, float *out_hyp, int32_t *out_cov_counts, float *out_cov_hyp,
                                 int32_t *out_tn, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    const bool with_cov = out_cov != nullptr;
    PV_CHECK_ARG(mask_mode == PVNET_MASK_NONZERO_BYTE || mask_mode == PVNET_MASK_EQUALS_ONE, "bad mask mode");
    PV_CHECK_ARG(idxs || rng_state, "neither idxs nor rng_state given");
    PV_CHECK_ARG(!with_cov || cov_idxs || rng_state, "neither cov_idxs nor rng_state given");
    PV_CHECK_ARG(!with_cov || (cov_hn >= 1 && cov_rounds >= 1 && cov_min_hyp_num >= 1), "bad covariance sizes");
    const long long hnt_ll = with_cov ? (long long)cov_hn * cov_rounds : 0;
    PV_CHECK_ARG(hnt_ll + hn <= (1 << 24), "too many hypotheses");
    const int hnt = (int)hnt_ll, HT = hn + hnt;
    int rc = check_common(mask, mask_elem_size, vertex, (const long long *)vertex_strides, b, h, w, vn, hn);
    if (rc) return rc;
    PV_CHECK_ARG(out_pts, "null out_pts");
    const Strides st = to_strides(vertex_strides);
    VoteWs ws = carve(workspace, b, h, w, vn, HT);
    if ((rc = ws_check(ws, workspace, workspace_bytes))) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const Samples sm{idxs, selection, idxs ? nullptr : rng_state};
    const Samples sel_src{nullptr, selection, selection ? nullptr : rng_state};
    if ((rc = launch_pixels(mask, mask_elem_size, mask_mode, vertex, st, sel_src, b, h, w, vn, min_num, max_num, ws, s))) return rc;
    PV_CUDA(cudaMemsetAsync(ws.counts, 0, sizeof(int) * (size_t)b * vn * HT, s));
    if ((rc = launch_gen_hyp(sm, RNG_IDXS_V3, b, h, w, vn, hn, HT, 0, ws, s))) return rc;
    if (with_cov) {
        const Samples smc{cov_idxs, selection, cov_idxs ? nullptr : rng_state};
        if ((rc = launch_gen_hyp(smc, RNG_IDXS_COV, b, h, w, vn, hnt, HT, hn, ws, s))) return rc;
    }
    if (with_cov && cov_inlier_thresh == inlier_thresh) {
        if ((rc = launch_vote(vertex, st, b, h, w, vn, HT, HT, 0, inlier_thresh, ws, s))) return rc;
    } else {
        if ((rc = launch_vote(vertex, st, b, h, w, vn, hn, HT, 0, inlier_thresh, ws, s))) return rc;
        if (with_cov && (rc = launch_vote(vertex, st, b, h, w, vn, hnt, HT, hn, cov_inlier_thresh, ws, s))) return rc;
    }
    if ((rc = launch_refit(b, h, w, vn, hn, HT, inlier_thresh, ws, out_pts, s))) return rc;
    if (with_cov) {
        k_cov<<<b * vn, 256, 0, s>>>(ws.hyp, ws.counts, ws.tn, out_pts, vn, hnt, HT, hn, cov_min_hyp_num, out_cov);
        PV_LAUNCHED("k_cov");
    }
    if ((rc = launch_export(ws, b, vn, hn, HT, 0, out_hyp, out_counts, out_tn, s))) return rc;
    if (with_cov && (rc = launch_export(ws, b, vn, hnt, HT, hn, out_cov_hyp, out_cov_counts, nullptr, s))) return rc;
    if (rng_state && (!idxs || (with_cov && !cov_idxs) || !selection)) return finish_rng(Samples{nullptr, nullptr, rng_state}, s);
    return PVNET_OK;
}

int pvnet_generate_hypothesis(const float *direct, const float *coords, const int32_t *idxs, float *hypo, int tn,
                              int vn, int hn, pvnet_stream_t stream)
{
    PV_CHECK_ARG(direct && coords && idxs && hypo, "null pointer");
    PV_CHECK_ARG(tn >= 1 && vn >= 1 && hn >= 1, "non-positive dimension");
    k_compat_gen_hyp<<<(hn * vn + 255) / 256, 256, 0, (cudaStream_t)stream>>>(direct, coords, idxs, hypo, tn, vn, hn);
    PV_LAUNCHED("k_compat_gen_hyp");
    return PVNET_OK;
}

int pvnet_voting_for_hypothesis(const float *direct, const float *coords, const float *hypo, uint8_t *inliers,
                                int tn, int vn, int hn, float inlier_thresh, pvnet_stream_t stream)
{
    PV_CHECK_ARG(direct && coords && hypo && inliers, "null pointer");
    PV_CHECK_ARG(tn >= 1 && vn >= 1 && hn >= 1 && vn <= 65535 && hn <= 65535, "dimension out of range");
    dim3 grid((tn + 255) / 256, vn, hn);
    k_compat_vote<<<grid, 256, 0, (cudaStream_t)stream>>>(direct, coords, hypo, inliers, tn, vn, hn, inlier_thresh);
    PV_LAUNCHED("k_compat_vote");
    return PVNET_OK;
}

int pvnet_generate_hypothesis_vanishing_point(const float *direct, const float *coords, const int32_t *idxs,
                                              float *hypo, int tn, int vn, int hn, pvnet_stream_t stream)
{
    PV_CHECK_ARG(direct && coords && idxs && hypo, "null pointer");
    PV_CHECK_ARG(tn >= 1 && vn >= 1 && hn >= 1, "non-positive dimension");
    k_compat_vp_gen_hyp<<<(hn * vn + 255) / 256, 256, 0, (cudaStream_t)stream>>>(direct, coords, idxs, hypo, vn, hn);
    PV_LAUNCHED("k_compat_vp_gen_hyp");
    return PVNET_OK;
}

int pvnet_voting_for_hypothesis_vanishing_point(const float *direct, const float *coords, const float *hypo,
                                                uint8_t *inliers, int32_t *counts, int tn, int vn, int hn,
                                                float inlier_thresh, pvnet_stream_t stream)
{
    PV_CHECK_ARG(direct && coords && hypo && (inliers || counts), "null pointer");
    PV_CHECK_ARG(tn >= 1 && vn >= 1 && hn >= 1 && hn <= 65535, "dimension out of range");
    dim3 grid(vn, hn);
    k_compat_vp_vote<<<grid, 256, 0, (cudaStream_t)stream>>>(direct, coords, hypo, inliers, counts, tn, vn, inlier_thresh);
    PV_LAUNCHED("k_compat_vp_vote");
    return PVNET_OK;
}

int pvnet_vote_counts(const float *direct, const float *coords, const float *hypo, int32_t *counts, int tn, int vn,
                      int hn, float inlier_thresh, pvnet_stream_t stream)
{
    PV_CHECK_ARG(direct && coords && hypo && counts, "null pointer");
    PV_CHECK_ARG(tn >= 1 && vn >= 1 && hn >= 1 && hn <= 65535, "dimension out of range");
    dim3 grid(vn, hn);
    k_compat_counts<<<grid, 256, 0, (cudaStream_t)stream>>>(direct, coords, hypo, counts, tn, vn, inlier_thresh);
    PV_LAUNCHED("k_compat_counts");
    return PVNET_OK;
}

}  // extern "C"
