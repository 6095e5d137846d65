// conv_grad.cu -- the weight gradient of an NHWC convolution on the Hopper tensor cores (wgmma, sm_90a), and the
// zero insertion that turns the two stride-2 layers' gradients into stride-1 problems.  Together with
// pvnet_conv2d_nhwc (which runs every data gradient as a forward convolution of dY with the flipped, transposed
// weights) this is the backward of the 24 trunk/decoder convolutions of Resnet18_8s under autograd
// (lib/networks/resnet.py:28-35,54-70, model_repository.py:22-58).
//
//   dW[co][ci][kh][kw] = sum_{n,y,x} dY[n,y,x,co] * X[n, y+(kh-c)*d, x+(kw-c)*d, ci]      c = (k-1)/2
//
// As a GEMM: M = Cout, N = Cin (per tap), K = pixels.  In NHWC both operands have the channels contiguous, i.e.
// they are MN-major, and wgmma takes tf32 shared-memory operands only K-major, so one transpose per tile is
// unavoidable.  k_conv_wgrad puts it on the loader:
//   A = dY^T  from registers (register-A wgmma): the dY tile [32 px][BM co] is stored as loaded (one 16-byte
//             store per float4) with a padded row, and each thread reads its m16n8k8-style fragments with
//             4-byte loads -- the transpose is the fragment addressing, and the padding makes it conflict-free.
//   B = X^T   K-major: the loader scatters each float4 of 4 channels of one pixel into 4 rows of a 128-byte
//             swizzled [BN ci][32 px] tile (what TMA would have written for a K-major operand).
// Nothing transposed ever goes to HBM.  One CTA owns one (tap, Cout tile, Cin tile) and a contiguous range of
// K-blocks of 32 flattened pixels (the split over pixels: M x N is small, K is up to 9.8 M).  Out-of-image X
// pixels (the padding) and pixels past the end are zeros from the loader.  Each CTA writes its fp32 partial tile
// to the workspace; k_conv_wgrad_reduce adds the partials in split order and writes dW in torch's layout.  No
// atomics: the result is identical run to run.
#include "common.cuh"
#include "ptx.cuh"

#include <algorithm>

namespace pvnet {

constexpr int WG_KP = 32;     // pixels per K-block: one 128-byte row of the K-major X tile

struct WgradGeom {
    const float *x, *dy;
    float *part;
    long long P;               // b*H*W pixels (the K extent)
    int H, W;
    int x_cs, x_co, Cin;
    int dy_cs, dy_co, Cout;
    int ksize, dil, taps;
    int n_ci_tiles, n_co_tiles;
    int kb_total, kb_per_split, splits;
};

// NWG consumer warpgroups, 64 output channels each (BM = 64 NWG); BN input channels per tile (64 or 128).
template <int NWG, int BN>
__global__ void __launch_bounds__(NWG * 128, 2) k_conv_wgrad(const __grid_constant__ WgradGeom g)
{
    constexpr int NT = NWG * 128;
    constexpr int BM = 64 * NWG;
    constexpr int LDA = BM + 8;                  // floats per pixel row of the dY tile: 8 t + g hits 32 banks
    constexpr int XI = WG_KP * BN / 4 / NT;      // float4 loads of X per thread and K-block
    constexpr int DI = WG_KP * BM / 4 / NT;      // float4 loads of dY per thread and K-block
    static_assert(XI * NT * 4 == WG_KP * BN && DI * NT * 4 == WG_KP * BM, "tile / thread mismatch");
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const uint32_t sb = ptx::smem_u32(smem);                       // X^T: BN rows of 128 bytes, swizzled
    const uint32_t sa = sb + (uint32_t)(BN * 128);                 // dY:  [32 px][LDA]

    // grid order: Cin tile fastest, then Cout tile, tap, split -- the CTAs resident together read the same pixels
    long long id = blockIdx.x;
    const int ci_t = (int)(id % g.n_ci_tiles);
    id /= g.n_ci_tiles;
    const int co_t = (int)(id % g.n_co_tiles);
    id /= g.n_co_tiles;
    const int tap = (int)(id % g.taps);
    const int split = (int)(id / g.taps);
    const int ci0 = ci_t * BN, co0 = co_t * BM;
    const int c = g.ksize >> 1;
    const int oy = (tap / g.ksize - c) * g.dil, ox = (tap % g.ksize - c) * g.dil;
    const int kb0 = split * g.kb_per_split;
    const int kb1 = min(kb0 + g.kb_per_split, g.kb_total);
    const int HW = g.H * g.W;

    // X loader: bits [0,2) of the item = channel quad within a group of 4, [2,7) = pixel, the rest = quad group.
    // NT >= 128, so a thread's pixel is the same for all its XI items.
    const int x_q = threadIdx.x & 3, x_p = (threadIdx.x >> 2) & 31, x_grp = threadIdx.x >> 7;
    // dY loader: item = pixel * (BM/4) + channel quad; a thread's pixels are 8 apart (NT / (BM/4) = 8)
    const int d_q = threadIdx.x % (BM / 4), d_p = threadIdx.x / (BM / 4);

    float4 xr[XI], dr[DI];
    auto load = [&](int kb) {
        const long long pix = (long long)kb * WG_KP + x_p;
        bool ok = pix < g.P;
        const float *src = g.x;
        if (ok) {
            const int n = (int)(pix / HW);
            const int rem = (int)(pix - (long long)n * HW);
            const int y = rem / g.W + oy, xx = rem % g.W + ox;
            ok = y >= 0 && y < g.H && xx >= 0 && xx < g.W;
            src = g.x + ((long long)n * HW + (long long)y * g.W + xx) * g.x_cs + g.x_co;
        }
#pragma unroll
        for (int j = 0; j < XI; ++j) {
            const int ci = ci0 + 4 * ((x_grp + j * (NT / 128)) * 4 + x_q);
            xr[j] = ok && ci < g.Cin ? __ldg(reinterpret_cast<const float4 *>(src + ci)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < DI; ++j) {
            const long long p = (long long)kb * WG_KP + d_p + 8 * j;
            const int co = co0 + 4 * d_q;
            dr[j] = p < g.P && co < g.Cout
                        ? __ldg(reinterpret_cast<const float4 *>(g.dy + p * g.dy_cs + g.dy_co + co))
                        : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = warp >> 2, wq = warp & 3;
    const int g8 = lane >> 2, t4 = lane & 3;
    const int mrow = wg * 64 + wq * 16 + g8;          // this thread's A rows (output channels) mrow, mrow + 8
    const uint64_t bdesc = ptx::make_kmajor_desc(sb, 128);

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

    load(kb0);
    for (int kb = kb0; kb < kb1; ++kb) {
        __syncthreads();                               // every warpgroup's MMAs on the previous tiles have completed
#pragma unroll
        for (int j = 0; j < XI; ++j) {
            const int r = 4 * ((x_grp + j * (NT / 128)) * 4 + x_q);
            const float v[4] = {xr[j].x, xr[j].y, xr[j].z, xr[j].w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                ptx::sts32(sb + ptx::swizzle_off((uint32_t)((r + e) * 128 + x_p * 4), 128), v[e]);
        }
#pragma unroll
        for (int j = 0; j < DI; ++j)
            ptx::sts128(sa + (uint32_t)(((d_p + 8 * j) * LDA + 4 * d_q) * 4), dr[j]);
        ptx::fence_proxy_async();                      // generic-proxy stores -> visible to wgmma's operand reads
        __syncthreads();
        if (kb + 1 < kb1) load(kb + 1);                // in flight during this K-block's MMAs
        uint32_t a[WG_KP / 8][4];
#pragma unroll
        for (int k = 0; k < WG_KP / 8; ++k) {
            const uint32_t r0 = sa + (uint32_t)(((8 * k + t4) * LDA + mrow) * 4);
            const uint32_t r1 = r0 + (uint32_t)(4 * LDA * 4);
            a[k][0] = __float_as_uint(ptx::lds32(r0));
            a[k][1] = __float_as_uint(ptx::lds32(r0 + 32));
            a[k][2] = __float_as_uint(ptx::lds32(r1));
            a[k][3] = __float_as_uint(ptx::lds32(r1 + 32));
        }
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_KP / 8; ++k)            // 8 tf32 = 32 bytes along K: +2 in 16-byte units
            ptx::Wgmma<BN>::rs(acc, a[k], bdesc + (uint64_t)(2 * k), 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();                          // the A registers and the tiles are reused next K-block
        ptx::fence_regs(acc);
    }

    // partial tile -> part[split][co][tap][ci]
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int co = co0 + mrow + 8 * h;
        if (co >= g.Cout) continue;
        float *dst = g.part + (((long long)split * g.Cout + co) * g.taps + tap) * g.Cin;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            const int ci = ci0 + 8 * j + 2 * t4;
            if (ci < g.Cin)
                *reinterpret_cast<float2 *>(dst + ci) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

// dW[co][ci][tap] (torch's [Cout][Cin][kh][kw]) = sum over splits, in split order.  Threads walk the partials in
// their own [co][tap][ci] order, so the reads (splits x the size of dW) are coalesced; the write of dW is strided.
__global__ void k_conv_wgrad_reduce(const float *__restrict__ part, float *__restrict__ dw, int Cout, int Cin, int taps,
                                    int splits)
{
    const long long n = (long long)Cout * taps * Cin;
    for (long long o = blockIdx.x * (long long)blockDim.x + threadIdx.x; o < n; o += (long long)gridDim.x * blockDim.x) {
        const long long ct = o / Cin;                  // co * taps + tap
        const int ci = (int)(o - ct * Cin);
        const int co = (int)(ct / taps), tap = (int)(ct - (long long)co * taps);
        float s = 0.f;
        for (int k = 0; k < splits; ++k) s += __ldg(part + o + k * n);
        dw[((long long)co * Cin + ci) * taps + tap] = s;
    }
}

// out[n,y,x,c] = (y, x both even) ? in[n,y/2,x/2,c] : 0, over the full-resolution H x W grid
__global__ void k_zero_insert2x(const float *__restrict__ in, int in_cs, int in_co, float *__restrict__ out, int out_cs,
                                int out_co, int C, long long npix, int H, int W)
{
    const int cq = C / 4;
    const long long n = npix * cq;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long pix = i / cq;
        const int q = (int)(i - pix * cq);
        const int x = (int)(pix % W);
        const long long ny = pix / W;
        const int y = (int)(ny % H);
        const long long img = ny / H;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (((x | y) & 1) == 0)
            v = __ldg(reinterpret_cast<const float4 *>(in + ((img * (H / 2) + y / 2) * (W / 2) + x / 2) * in_cs + in_co +
                                                       4 * q));
        *reinterpret_cast<float4 *>(out + pix * out_cs + out_co + 4 * q) = v;
    }
}

// ------------------------------------------------------------------ host side
struct WgradPlan {
    WgradGeom g;
    int nwg, bn;
    long long grid;
    size_t smem, part_bytes;
};

template <int NWG, int BN>
static size_t wgrad_smem() { return 1024 + (size_t)BN * 128 + (size_t)WG_KP * (64 * NWG + 8) * 4; }

template <int NWG, int BN>
static int wgrad_occupancy(int *blocks)
{
    PV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, k_conv_wgrad<NWG, BN>, NWG * 128,
                                                          wgrad_smem<NWG, BN>()));
    return PVNET_OK;
}

static int wgrad_plan(int Cin, int Cout, int b, int H, int W, int ksize, WgradPlan *p)
{
    PV_CHECK_ARG(ksize == 1 || ksize == 3, "wgrad: kernel size %d unsupported", ksize);
    PV_CHECK_ARG(Cin > 0 && Cout > 0 && Cin % 4 == 0 && Cout % 4 == 0, "wgrad: Cin %d, Cout %d must be positive multiples of 4",
                 Cin, Cout);
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0, "wgrad: empty pixel grid");
    WgradGeom &g = p->g;
    g = WgradGeom{};
    g.P = (long long)b * H * W;
    g.H = H;
    g.W = W;
    g.Cin = Cin;
    g.Cout = Cout;
    g.ksize = ksize;
    g.taps = ksize * ksize;
    // 128 output channels share each X^T tile across two warpgroups when the layer has them; the Cin tile is
    // 128 where it divides Cin, 64 otherwise (64, 192 and convraw.0's 40)
    p->nwg = Cout >= 128 ? 2 : 1;
    p->bn = Cin % 128 == 0 ? 128 : 64;
    g.n_co_tiles = (Cout + 64 * p->nwg - 1) / (64 * p->nwg);
    g.n_ci_tiles = (Cin + p->bn - 1) / p->bn;
    const long long kbt = (g.P + WG_KP - 1) / WG_KP;
    PV_CHECK_ARG(kbt < (1ll << 31), "wgrad: %lld pixels is too many", g.P);
    g.kb_total = (int)kbt;
    int occ = 0;
    int rc = p->nwg == 2 ? (p->bn == 128 ? wgrad_occupancy<2, 128>(&occ) : wgrad_occupancy<2, 64>(&occ))
                         : (p->bn == 128 ? wgrad_occupancy<1, 128>(&occ) : wgrad_occupancy<1, 64>(&occ));
    if (rc) return rc;
    const long long slots = (long long)(sm_count() > 0 ? sm_count() : 1) * (occ > 0 ? occ : 1);
    const long long tiles = (long long)g.taps * g.n_co_tiles * g.n_ci_tiles;
    // split count: the one whose waves x (K-blocks per CTA + WGRAD_CTA_COST) is least (ties to fewer splits).  The
    // per-CTA term, in K-block units, stands for the prologue's exposed load latency, the partial-tile store and its
    // read in the reduction; without it the count runs into the hundreds for a gain of a fraction of a wave.  At
    // least 16 K-blocks per split, and at most WGRAD_MAX_PART_BYTES of partial tiles.
    constexpr long long WGRAD_CTA_COST = 8;
    constexpr long long WGRAD_MAX_PART_BYTES = 128ll << 20;
    const long long tile_bytes = (long long)Cout * g.taps * Cin * (long long)sizeof(float);
    long long best = -1;
    int best_s = 1;
    const int max_s = (int)std::max(1ll, std::min({4096ll, kbt / 16, WGRAD_MAX_PART_BYTES / tile_bytes}));
    for (int s = 1; s <= max_s; ++s) {
        const long long per = (kbt + s - 1) / s;
        const long long used = (kbt + per - 1) / per;
        if (used != s) continue;                    // the same split as a smaller s
        const long long cost = (tiles * s + slots - 1) / slots * (per + WGRAD_CTA_COST);
        if (best < 0 || cost < best) {
            best = cost;
            best_s = s;
        }
    }
    g.kb_per_split = (int)((kbt + best_s - 1) / best_s);
    g.splits = best_s;
    p->grid = tiles * best_s;
    p->smem = p->nwg == 2 ? (p->bn == 128 ? wgrad_smem<2, 128>() : wgrad_smem<2, 64>())
                          : (p->bn == 128 ? wgrad_smem<1, 128>() : wgrad_smem<1, 64>());
    p->part_bytes = (size_t)best_s * Cout * g.taps * Cin * sizeof(float);
    return PVNET_OK;
}

template <int NWG, int BN>
static int wgrad_launch_t(const WgradPlan &p, cudaStream_t s)
{
    k_conv_wgrad<NWG, BN><<<(unsigned)p.grid, NWG * 128, p.smem, s>>>(p.g);
    PV_LAUNCHED("k_conv_wgrad");
    return PVNET_OK;
}

}  // namespace pvnet

extern "C" {

int pvnet_conv2d_nhwc_wgrad_workspace_bytes(int Cin, int Cout, int b, int H, int W, int ksize, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "wgrad: null bytes");
    pvnet::WgradPlan p;
    int rc = pvnet::wgrad_plan(Cin, Cout, b, H, W, ksize, &p);
    if (rc) return rc;
    *bytes = p.part_bytes;
    return PVNET_OK;
}

int pvnet_conv2d_nhwc_wgrad(const float *in, int in_cs, int in_co, int Cin, const float *dout, int dout_cs, int dout_co,
                            int Cout, float *dw, int b, int H, int W, int ksize, int dilation, void *workspace,
                            size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(in && dout && dw, "wgrad: null pointer");
    PV_CHECK_ARG(dilation >= 1, "wgrad: dilation %d must be >= 1", dilation);
    PV_CHECK_ARG(in_cs % 4 == 0 && in_co % 4 == 0 && dout_cs % 4 == 0 && dout_co % 4 == 0,
                 "wgrad: channel strides/offsets must be multiples of 4 floats");
    PV_CHECK_ARG(in_co + Cin <= in_cs && dout_co + Cout <= dout_cs, "wgrad: channel slice exceeds its buffer");
    PV_CHECK_ARG((uintptr_t)in % 16 == 0 && (uintptr_t)dout % 16 == 0, "wgrad: pointers must be 16-byte aligned");
    pvnet::WgradPlan p;
    int rc = pvnet::wgrad_plan(Cin, Cout, b, H, W, ksize, &p);
    if (rc) return rc;
    PV_CHECK_ARG(workspace && workspace_bytes >= p.part_bytes, "wgrad: workspace of %zu bytes, %zu needed",
                 workspace_bytes, p.part_bytes);
    PV_CHECK_ARG((uintptr_t)workspace % 16 == 0, "wgrad: workspace must be 16-byte aligned");
    pvnet::WgradGeom &g = p.g;
    g.x = in;
    g.dy = dout;
    g.part = static_cast<float *>(workspace);
    g.x_cs = in_cs;
    g.x_co = in_co;
    g.dy_cs = dout_cs;
    g.dy_co = dout_co;
    g.dil = dilation;
    cudaStream_t s = (cudaStream_t)stream;
    if (p.nwg == 2)
        rc = p.bn == 128 ? pvnet::wgrad_launch_t<2, 128>(p, s) : pvnet::wgrad_launch_t<2, 64>(p, s);
    else
        rc = p.bn == 128 ? pvnet::wgrad_launch_t<1, 128>(p, s) : pvnet::wgrad_launch_t<1, 64>(p, s);
    if (rc) return rc;
    const long long n = (long long)Cout * Cin * g.taps;
    const int blocks = (int)std::min<long long>((n + 255) / 256, 4096);
    pvnet::k_conv_wgrad_reduce<<<blocks, 256, 0, s>>>(g.part, dw, Cout, Cin, g.taps, g.splits);
    PV_LAUNCHED("k_conv_wgrad_reduce");
    return PVNET_OK;
}

int pvnet_zero_insert2x_nhwc(const float *in, int in_cs, int in_co, int C, float *out, int out_cs, int out_co, int b,
                             int H, int W, pvnet_stream_t stream)
{
    PV_CHECK_ARG(in && out, "zero insertion: null pointer");
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "zero insertion: H,W must be positive and even");
    PV_CHECK_ARG(C > 0 && C % 4 == 0 && in_cs % 4 == 0 && in_co % 4 == 0 && out_cs % 4 == 0 && out_co % 4 == 0,
                 "zero insertion: channels, strides and offsets must be multiples of 4 floats");
    PV_CHECK_ARG(in_co + C <= in_cs && out_co + C <= out_cs, "zero insertion: channel slice exceeds its buffer");
    PV_CHECK_ARG((uintptr_t)in % 16 == 0 && (uintptr_t)out % 16 == 0, "zero insertion: pointers must be 16-byte aligned");
    const long long npix = (long long)b * H * W;
    const long long n = npix * (C / 4);
    const int blocks = (int)std::min<long long>((n + 255) / 256, 8 * 1024);
    pvnet::k_zero_insert2x<<<blocks, 256, 0, (cudaStream_t)stream>>>(in, in_cs, in_co, out, out_cs, out_co, C, npix, H, W);
    PV_LAUNCHED("k_zero_insert2x");
    return PVNET_OK;
}

}  // extern "C"
