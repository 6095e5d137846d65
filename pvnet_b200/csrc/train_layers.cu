// train_layers.cu -- the two layers of Resnet18_8s's training step that have no eval-path kernel to reuse: the stem
// conv1's weight gradient (lib/networks/resnet.py:201, 7x7 stride 2, pad 3, no bias) on the Hopper tensor cores, and
// the head convraw.3 (model_repository.py:57, 1x1 with bias) forward and backward in plain fp32 / fp64.
//
// Stem.  The forward runs as a 4x4 stride-1 convolution on the 2x2 space-to-depth image S [b,H/2,W/2,16]
// (pvnet_stem_s2d_nhwc, backbone_aux.cu), so its weight gradient is the 4x4 one on S, folded back:
//   dW_s2d[co][ty][tx][ch] = sum_p dY[p][co] * S[p + (ty-2, tx-2)][ch]
//   dW[co][c][kh][kw]      = dW_s2d[co][ty][tx][(py*2+px)*3+c],  kh = 2ty+py-1, kw = 2tx+px-1
// (147 of the 256 entries per output channel; the rest are gradients of weights fixed at zero, dropped).
// k_stem_wgrad is the GEMM M = 64 output channels, N = 256 (all 16 taps x 16 channels), K = pixels: one CTA reads
// each dY tile once for all taps.  As in k_conv_wgrad (conv_grad.cu) A = dY^T comes from registers (the [32 px][64]
// tile stored as loaded, read transposed through padded fragment loads) and B = S^T is scattered by the loader into
// 128-byte-swizzled K-major rows; the two warpgroups own taps 0-7 and 8-15 (m64n128 each).  CTAs split the pixels;
// k_stem_wgrad_reduce adds the partial tiles in split order and writes the 147 folded entries.  No atomics.
//
// Head.  Forward: out[n][o][p] = fmaf chain over c ascending from bias[o] (exact fp32, no TF32), written straight to
// NCHW.  Backward: dy[p][c] = fmaf chain over o ascending from 0; dW[o][c] = sum_p dOut[p][o]*y[p][c] and
// db[o] = sum_p dOut[p][o] in fp64 (the fp32 x fp32 products are exact) over a fixed partition of the pixels into
// HEAD_CHUNK-pixel partials, merged in a fixed lane-then-tree order and rounded once to fp32 -- nothing depends on
// the grid or the SM count.
#include "common.cuh"
#include "ptx.cuh"

#include <algorithm>

namespace pvnet {

// ------------------------------------------------------------------ stem weight gradient
constexpr int SW_KP = 32;                       // pixels per K-block: one 128-byte row of the K-major S^T tile
constexpr int SW_LDA = 64 + 8;                  // floats per pixel row of the dY tile (conflict-free fragment loads)
constexpr int SW_THREADS = 256;
constexpr size_t SW_SMEM = 1024 + 256 * 128 + (size_t)SW_KP * SW_LDA * 4;
constexpr int SW_TILE = 64 * 256;               // one partial tile [co][tap][ch]

struct StemWgradGeom {
    const float *s2d, *dy;
    float *part;
    long long P;                                 // b*H2*W2 pixels
    int H2, W2;
    int kb_total, kb_per_split, splits;
};

__global__ void __launch_bounds__(SW_THREADS, 1) k_stem_wgrad(const __grid_constant__ StemWgradGeom g)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sb = ptx::smem_u32(smem);                  // S^T: 256 rows (tap*16 + ch) of 128 bytes, swizzled
    const uint32_t sa = sb + 256u * 128u;                     // dY: [32 px][SW_LDA]
    const int split = blockIdx.x;
    const int kb0 = split * g.kb_per_split;
    const int kb1 = min(kb0 + g.kb_per_split, g.kb_total);
    const int HW = g.H2 * g.W2;

    // S loader: thread = (channel quad x_q, pixel x_p, tap half x_h), 8 taps of one pixel
    const int x_q = threadIdx.x & 3, x_p = (threadIdx.x >> 2) & 31, x_h = threadIdx.x >> 7;
    // dY loader: item = pixel * 16 + channel quad; the thread's pixels are d_p and d_p + 16
    const int d_q = threadIdx.x & 15, d_p = threadIdx.x >> 4;

    float4 xr[8], dr[2];
    auto load = [&](int kb) {
        const long long pix = (long long)kb * SW_KP + x_p;
        const bool in = pix < g.P;
        long long n = 0;
        int y = 0, x = 0;
        if (in) {
            n = pix / HW;
            const int rem = (int)(pix - n * HW);
            y = rem / g.W2;
            x = rem - y * g.W2;
        }
        const float *img = g.s2d + n * HW * 16 + 4 * x_q;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int tap = x_h * 8 + j;
            const int yy = y + (tap >> 2) - 2, xx = x + (tap & 3) - 2;
            xr[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (in && yy >= 0 && yy < g.H2 && xx >= 0 && xx < g.W2)
                xr[j] = __ldg(reinterpret_cast<const float4 *>(img + ((long long)yy * g.W2 + xx) * 16));
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long p = (long long)kb * SW_KP + d_p + 16 * j;
            dr[j] = p < g.P ? __ldg(reinterpret_cast<const float4 *>(g.dy + p * 64 + 4 * d_q))
                            : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2, wq = warp & 3;
    const int g8 = lane >> 2, t4 = lane & 3;
    const int mrow = wq * 16 + g8;                            // this thread's A rows (output channels) mrow, mrow + 8
    const uint64_t bdesc = ptx::make_kmajor_desc(sb + (uint32_t)wg * 128u * 128u, 128);

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;

    if (kb0 < kb1) load(kb0);
    for (int kb = kb0; kb < kb1; ++kb) {
        __syncthreads();                                      // both warpgroups' MMAs on the previous tiles are done
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = (x_h * 8 + j) * 16 + 4 * x_q;
            const float v[4] = {xr[j].x, xr[j].y, xr[j].z, xr[j].w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                ptx::sts32(sb + ptx::swizzle_off((uint32_t)((r + e) * 128 + x_p * 4), 128), v[e]);
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) ptx::sts128(sa + (uint32_t)(((d_p + 16 * j) * SW_LDA + 4 * d_q) * 4), dr[j]);
        ptx::fence_proxy_async();                             // generic-proxy stores -> visible to wgmma
        __syncthreads();
        if (kb + 1 < kb1) load(kb + 1);                       // in flight during this K-block's MMAs
        uint32_t a[SW_KP / 8][4];
#pragma unroll
        for (int k = 0; k < SW_KP / 8; ++k) {
            const uint32_t r0 = sa + (uint32_t)(((8 * k + t4) * SW_LDA + mrow) * 4);
            const uint32_t r1 = r0 + (uint32_t)(4 * SW_LDA * 4);
            a[k][0] = __float_as_uint(ptx::lds32(r0));
            a[k][1] = __float_as_uint(ptx::lds32(r0 + 32));
            a[k][2] = __float_as_uint(ptx::lds32(r1));
            a[k][3] = __float_as_uint(ptx::lds32(r1 + 32));
        }
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < SW_KP / 8; ++k) ptx::Wgmma<128>::rs(acc, a[k], bdesc + (uint64_t)(2 * k), 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
    }

    // partial tile -> part[split][co][tap*16 + ch]; warpgroup wg holds columns [128 wg, 128 wg + 128)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float *dst = g.part + ((long long)split * 64 + mrow + 8 * h) * 256 + wg * 128;
#pragma unroll
        for (int j = 0; j < 16; ++j)
            *reinterpret_cast<float2 *>(dst + 8 * j + 2 * t4) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
}

// dW[co][c][kh][kw] = sum over splits (in split order) of part[.][co][tap][ch] for the 147 (tap, ch) that carry a
// weight of the 7x7 kernel.  Threads walk the partials in their own order (coalesced reads).
__global__ void __launch_bounds__(256) k_stem_wgrad_reduce(const float *__restrict__ part, float *__restrict__ dw,
                                                           int splits)
{
    const int o = blockIdx.x * 256 + threadIdx.x;            // co*256 + tap*16 + ch
    if (o >= SW_TILE) return;
    const int co = o >> 8, tap = (o >> 4) & 15, ch = o & 15;
    const int par = ch / 3, c = ch - 3 * par;
    const int kh = 2 * (tap >> 2) + (par >> 1) - 1, kw = 2 * (tap & 3) + (par & 1) - 1;
    if (ch >= 12 || kh < 0 || kh > 6 || kw < 0 || kw > 6) return;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s = __fadd_rn(s, __ldg(part + o + (long long)k * SW_TILE));
    dw[((co * 3 + c) * 7 + kh) * 7 + kw] = s;
}

static int stem_wgrad_plan(int b, int H, int W, StemWgradGeom *g)
{
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "stem wgrad: b, H, W must be positive, H and W even");
    *g = StemWgradGeom{};
    g->H2 = H / 2;
    g->W2 = W / 2;
    g->P = (long long)b * g->H2 * g->W2;
    const long long kbt = (g->P + SW_KP - 1) / SW_KP;
    PV_CHECK_ARG(kbt < (1ll << 31), "stem wgrad: %lld pixels is too many", g->P);
    int occ = 0;
    PV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_stem_wgrad, SW_THREADS, SW_SMEM));
    const long long slots = (long long)std::max(1, sm_count()) * std::max(1, occ);
    // one wave of CTAs, each with at least 16 K-blocks
    const long long s = std::max(1ll, std::min(slots, kbt / 16));
    g->kb_per_split = (int)((kbt + s - 1) / s);
    g->kb_total = (int)kbt;
    g->splits = (int)((kbt + g->kb_per_split - 1) / g->kb_per_split);
    return PVNET_OK;
}

// ------------------------------------------------------------------ head convraw.3 (1x1 + bias)
constexpr int HEAD_CHUNK = 4096;                // pixels per fp64 partial of dW / db (fixed partition)
constexpr int HB_TP = 64;                       // pixels per shared-memory tile of the backward
constexpr int HB_ITEMS = 2;                     // quads of sums per thread and pass
constexpr int HEAD_LANES = 256;                 // merge: lanes, then a halving tree
constexpr size_t HEAD_SMEM_LIMIT = 227 * 1024;  // the kernels' dynamic shared-memory limit, set once per device

static size_t head_fwd_smem(int Cin, int Cout) { return ((size_t)Cout * Cin + Cout) * sizeof(float); }
static size_t head_bwd_smem(int Cin, int Cout)
{
    return (size_t)HB_TP * (Cout + Cin) * sizeof(double) + ((size_t)HB_TP * Cout + (size_t)Cout * Cin) * sizeof(float);
}

// y NHWC [P][Cin] (Cin a multiple of 32) -> out NCHW [b][Cout][HW]; one thread = one pixel, 16 outputs at a time
__global__ void __launch_bounds__(256)
    k_head_train(const float *__restrict__ y, const float *__restrict__ w, const float *__restrict__ bias,
                 float *__restrict__ out, long long P, int HW, int Cin, int Cout)
{
    extern __shared__ float hsm[];
    float *sw = hsm, *sbias = hsm + (size_t)Cout * Cin;
    for (int i = threadIdx.x; i < Cout * Cin; i += blockDim.x) sw[i] = w[i];
    for (int i = threadIdx.x; i < Cout; i += blockDim.x) sbias[i] = bias[i];
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const long long n = i / HW, p = i - n * HW;
    const float *yr = y + i * Cin;
    float *o = out + n * Cout * (long long)HW + p;
    for (int o0 = 0; o0 < Cout; o0 += 16) {
        float acc[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) acc[u] = sbias[min(o0 + u, Cout - 1)];
        for (int c0 = 0; c0 < Cin; c0 += 32) {
            float v[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 t = __ldg(reinterpret_cast<const float4 *>(yr + c0) + j);
                v[4 * j] = t.x;
                v[4 * j + 1] = t.y;
                v[4 * j + 2] = t.z;
                v[4 * j + 3] = t.w;
            }
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const float4 *wr = reinterpret_cast<const float4 *>(sw + (size_t)min(o0 + u, Cout - 1) * Cin + c0);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float4 ww = wr[j];
                    acc[u] = __fmaf_rn(ww.x, v[4 * j], acc[u]);
                    acc[u] = __fmaf_rn(ww.y, v[4 * j + 1], acc[u]);
                    acc[u] = __fmaf_rn(ww.z, v[4 * j + 2], acc[u]);
                    acc[u] = __fmaf_rn(ww.w, v[4 * j + 3], acc[u]);
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 16; ++u)
            if (o0 + u < Cout) o[(long long)(o0 + u) * HW] = acc[u];
    }
}

// One CTA = one HEAD_CHUNK-pixel partial.  Tiles of HB_TP pixels of dOut (NCHW) and y (NHWC) are staged in shared
// memory; dy for the tile (first pass only), then the fp64 sums: item q < Cout*Cin/4 is (o, channel quad) of dW, the
// rest are quads of db.  Pixels ascend within the chunk; the partial goes to part[item][chunk].
template <bool SUMS>
__global__ void __launch_bounds__(256)
    k_head_train_backward(const float *__restrict__ dout, const float *__restrict__ y, const float *__restrict__ w,
                          float *__restrict__ dy, double *__restrict__ part, long long P, int HW, int Cin, int Cout,
                          int nparts)
{
    extern __shared__ double hsd[];
    double *gs = hsd;                                        // [HB_TP][Cout]
    double *ys = gs + HB_TP * Cout;                          // [HB_TP][Cin]
    float *gf = reinterpret_cast<float *>(ys + HB_TP * Cin); // [HB_TP][Cout]
    float *sw = gf + HB_TP * Cout;                           // [Cout][Cin]
    for (int i = threadIdx.x; i < Cout * Cin; i += blockDim.x) sw[i] = w[i];
    const long long p0 = (long long)blockIdx.x * HEAD_CHUNK;
    const long long p1 = min(p0 + HEAD_CHUNK, P);
    const int cq = Cin >> 2;
    const int nq = Cout * cq, nitems = nq + (Cout + 3) / 4;
    const int passes = SUMS ? (nitems + HB_ITEMS * 256 - 1) / (HB_ITEMS * 256) : 1;
    for (int pass = 0; pass < passes; ++pass) {
        double acc[HB_ITEMS][4];
#pragma unroll
        for (int k = 0; k < HB_ITEMS; ++k)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[k][e] = 0.0;
        for (long long t0 = p0; t0 < p1; t0 += HB_TP) {
            __syncthreads();
            const long long n0 = t0 / HW;                    // the tile's first image and its pixel offset there
            const int q0 = (int)(t0 - n0 * HW);
            for (int i = threadIdx.x; i < Cout * HB_TP; i += blockDim.x) {
                const int o = i / HB_TP, pp = i - o * HB_TP;
                float v = 0.f;
                if (t0 + pp < p1) {
                    long long n = n0;
                    int q = q0 + pp;
                    while (q >= HW) {                            // the tile runs into the next image(s)
                        q -= HW;
                        ++n;
                    }
                    v = __ldg(dout + (n * Cout + o) * HW + q);
                }
                gf[pp * Cout + o] = v;
                gs[pp * Cout + o] = (double)v;
            }
            for (int i = threadIdx.x; i < HB_TP * cq; i += blockDim.x) {
                const int pp = i / cq, c4 = i - pp * cq;
                const long long pix = t0 + pp;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (pix < p1) v = __ldg(reinterpret_cast<const float4 *>(y + pix * Cin) + c4);
                double *d = ys + pp * Cin + 4 * c4;
                d[0] = v.x;
                d[1] = v.y;
                d[2] = v.z;
                d[3] = v.w;
            }
            __syncthreads();
            if (pass == 0 && dy) {
                for (int i = threadIdx.x; i < HB_TP * cq; i += blockDim.x) {
                    const int pp = i / cq, c4 = i - pp * cq;
                    const long long pix = t0 + pp;
                    if (pix >= p1) continue;
                    float a[4] = {0.f, 0.f, 0.f, 0.f};
                    for (int o = 0; o < Cout; ++o) {
                        const float g = gf[pp * Cout + o];
                        const float4 ww = *reinterpret_cast<const float4 *>(sw + o * Cin + 4 * c4);
                        a[0] = __fmaf_rn(ww.x, g, a[0]);
                        a[1] = __fmaf_rn(ww.y, g, a[1]);
                        a[2] = __fmaf_rn(ww.z, g, a[2]);
                        a[3] = __fmaf_rn(ww.w, g, a[3]);
                    }
                    reinterpret_cast<float4 *>(dy + pix * Cin)[c4] = make_float4(a[0], a[1], a[2], a[3]);
                }
            }
            if (SUMS) {
#pragma unroll
                for (int k = 0; k < HB_ITEMS; ++k) {
                    const int it = (pass * HB_ITEMS + k) * 256 + threadIdx.x;
                    if (it < nq) {
                        const int o = it / cq, c4 = it - o * cq;
#pragma unroll 8
                        for (int pp = 0; pp < HB_TP; ++pp) {
                            const double g = gs[pp * Cout + o];
                            const double *yv = ys + pp * Cin + 4 * c4;
#pragma unroll
                            for (int e = 0; e < 4; ++e) acc[k][e] = __fma_rn(g, yv[e], acc[k][e]);
                        }
                    } else if (it < nitems) {
                        const int oq = 4 * (it - nq);
                        for (int pp = 0; pp < HB_TP; ++pp)
#pragma unroll
                            for (int e = 0; e < 4; ++e)
                                if (oq + e < Cout) acc[k][e] = __dadd_rn(acc[k][e], gs[pp * Cout + oq + e]);
                    }
                }
            }
        }
        if (SUMS) {
#pragma unroll
            for (int k = 0; k < HB_ITEMS; ++k) {
                const int it = (pass * HB_ITEMS + k) * 256 + threadIdx.x;
                if (it < nq) {
                    const int o = it / cq, c4 = it - o * cq;
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        part[((long long)o * Cin + 4 * c4 + e) * nparts + blockIdx.x] = acc[k][e];
                } else if (it < nitems) {
                    const int oq = 4 * (it - nq);
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (oq + e < Cout) part[((long long)Cout * Cin + oq + e) * nparts + blockIdx.x] = acc[k][e];
                }
            }
        }
    }
}

// one block per item (dW entries o*Cin + c, then db entries): lane t adds partials t, t+256, ... in order, then a
// halving tree; rounded once to fp32
__global__ void __launch_bounds__(HEAD_LANES)
    k_head_train_reduce(const double *__restrict__ part, int nparts, int ndw, float *__restrict__ dw,
                        float *__restrict__ db)
{
    __shared__ double red[HEAD_LANES];
    const int item = blockIdx.x;
    const double *src = part + (long long)item * nparts;
    double s = 0.0;
    for (int j = threadIdx.x; j < nparts; j += HEAD_LANES) s = __dadd_rn(s, __ldg(src + j));
    red[threadIdx.x] = s;
    __syncthreads();
    for (int h = HEAD_LANES / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (item < ndw) {
            if (dw) dw[item] = __double2float_rn(red[0]);
        } else if (db) {
            db[item - ndw] = __double2float_rn(red[0]);
        }
    }
}

static int check_head_args(const char *what, int b, int H, int W, int Cin, int Cout)
{
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0, "%s: b, H, W must be positive", what);
    PV_CHECK_ARG(Cin > 0 && Cin % 32 == 0, "%s: Cin %d must be a positive multiple of 32", what, Cin);
    PV_CHECK_ARG(Cout >= 1, "%s: Cout %d must be at least 1", what, Cout);
    PV_CHECK_ARG((long long)H * W < (1ll << 31), "%s: H*W must fit in 31 bits", what);
    PV_CHECK_ARG(head_bwd_smem(Cin, Cout) <= HEAD_SMEM_LIMIT, "%s: Cin %d x Cout %d does not fit in shared memory", what,
                 Cin, Cout);
    return PVNET_OK;
}

static long long head_nparts(int b, int H, int W)
{
    return ((long long)b * H * W + HEAD_CHUNK - 1) / HEAD_CHUNK;
}

}  // namespace pvnet

extern "C" {

int pvnet_stem_s2d_wgrad_workspace_bytes(int b, int H, int W, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "stem wgrad: null bytes");
    pvnet::StemWgradGeom g;
    if (int rc = pvnet::stem_wgrad_plan(b, H, W, &g)) return rc;
    *bytes = (size_t)g.splits * pvnet::SW_TILE * sizeof(float);
    return PVNET_OK;
}

int pvnet_stem_s2d_wgrad(const float *s2d, const float *dout, float *dw, int b, int H, int W, void *workspace,
                         size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(s2d && dout && dw, "stem wgrad: null pointer");
    PV_CHECK_ARG((uintptr_t)s2d % 16 == 0 && (uintptr_t)dout % 16 == 0, "stem wgrad: pointers must be 16-byte aligned");
    pvnet::StemWgradGeom g;
    if (int rc = pvnet::stem_wgrad_plan(b, H, W, &g)) return rc;
    const size_t need = (size_t)g.splits * pvnet::SW_TILE * sizeof(float);
    PV_CHECK_ARG(workspace && workspace_bytes >= need, "stem wgrad: workspace of %zu bytes, %zu needed",
                 workspace_bytes, need);
    PV_CHECK_ARG((uintptr_t)workspace % 16 == 0, "stem wgrad: workspace must be 16-byte aligned");
    g.s2d = s2d;
    g.dy = dout;
    g.part = static_cast<float *>(workspace);
    cudaStream_t s = (cudaStream_t)stream;
    pvnet::k_stem_wgrad<<<(unsigned)g.splits, pvnet::SW_THREADS, pvnet::SW_SMEM, s>>>(g);
    PV_LAUNCHED("k_stem_wgrad");
    pvnet::k_stem_wgrad_reduce<<<pvnet::SW_TILE / 256, 256, 0, s>>>(g.part, dw, g.splits);
    PV_LAUNCHED("k_stem_wgrad_reduce");
    return PVNET_OK;
}

int pvnet_head1x1_nchw(const float *y, const float *w, const float *bias, float *out, int b, int H, int W, int Cin,
                       int Cout, pvnet_stream_t stream)
{
    if (int rc = pvnet::check_head_args("head", b, H, W, Cin, Cout)) return rc;
    PV_CHECK_ARG(y && w && bias && out, "head: null pointer");
    PV_CHECK_ARG((uintptr_t)y % 16 == 0 && (uintptr_t)w % 16 == 0, "head: y and w must be 16-byte aligned");
    const size_t smem = pvnet::head_fwd_smem(Cin, Cout);
    PV_CHECK_ARG(smem <= pvnet::HEAD_SMEM_LIMIT, "head: Cin %d x Cout %d does not fit in shared memory", Cin, Cout);
    PV_CUDA(pvnet::ensure_max_smem((const void *)pvnet::k_head_train, (int)pvnet::HEAD_SMEM_LIMIT));
    const long long P = (long long)b * H * W;
    pvnet::k_head_train<<<(unsigned)((P + 255) / 256), 256, smem, (cudaStream_t)stream>>>(y, w, bias, out, P, H * W,
                                                                                        Cin, Cout);
    PV_LAUNCHED("k_head_train");
    return PVNET_OK;
}

int pvnet_head1x1_backward_workspace_bytes(int b, int H, int W, int Cin, int Cout, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "head backward: null bytes");
    if (int rc = pvnet::check_head_args("head backward", b, H, W, Cin, Cout)) return rc;
    *bytes = (size_t)Cout * (Cin + 1) * (size_t)pvnet::head_nparts(b, H, W) * sizeof(double);
    return PVNET_OK;
}

int pvnet_head1x1_backward(const float *dout, const float *y, const float *w, float *dy, float *dw, float *db, int b,
                           int H, int W, int Cin, int Cout, void *workspace, size_t workspace_bytes,
                           pvnet_stream_t stream)
{
    if (int rc = pvnet::check_head_args("head backward", b, H, W, Cin, Cout)) return rc;
    PV_CHECK_ARG(dout && y && w, "head backward: null pointer");
    PV_CHECK_ARG((uintptr_t)y % 16 == 0 && (uintptr_t)w % 16 == 0 && (uintptr_t)dy % 16 == 0,
                 "head backward: y, w and dy must be 16-byte aligned");
    const bool sums = dw || db;
    const long long nparts = pvnet::head_nparts(b, H, W);
    PV_CHECK_ARG(nparts < (1ll << 31), "head backward: too many pixels");
    const size_t need = (size_t)Cout * (Cin + 1) * (size_t)nparts * sizeof(double);
    PV_CHECK_ARG(!sums || (workspace && workspace_bytes >= need), "head backward: workspace of %zu bytes, %zu needed",
                 workspace_bytes, need);
    PV_CHECK_ARG(!sums || (uintptr_t)workspace % 16 == 0, "head backward: workspace must be 16-byte aligned");
    if (!dy && !sums) return PVNET_OK;
    cudaStream_t s = (cudaStream_t)stream;
    const size_t smem = pvnet::head_bwd_smem(Cin, Cout);
    const long long P = (long long)b * H * W;
    double *part = static_cast<double *>(workspace);
    if (sums) {
        PV_CUDA(pvnet::ensure_max_smem((const void *)pvnet::k_head_train_backward<true>, (int)pvnet::HEAD_SMEM_LIMIT));
        pvnet::k_head_train_backward<true><<<(unsigned)nparts, 256, smem, s>>>(dout, y, w, dy, part, P, H * W, Cin,
                                                                              Cout, (int)nparts);
    } else {
        PV_CUDA(pvnet::ensure_max_smem((const void *)pvnet::k_head_train_backward<false>, (int)pvnet::HEAD_SMEM_LIMIT));
        pvnet::k_head_train_backward<false><<<(unsigned)nparts, 256, smem, s>>>(dout, y, w, dy, part, P, H * W, Cin,
                                                                               Cout, (int)nparts);
    }
    PV_LAUNCHED("k_head_train_backward");
    if (sums) {
        pvnet::k_head_train_reduce<<<(unsigned)(Cout * (Cin + 1)), pvnet::HEAD_LANES, 0, s>>>(part, (int)nparts,
                                                                                             Cout * Cin, dw, db);
        PV_LAUNCHED("k_head_train_reduce");
    }
    return PVNET_OK;
}

}  // extern "C"
