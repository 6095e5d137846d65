// conv_col.cu -- persistent, weights-resident 3x3 convolution for the narrow layers
// (Cout <= 64: layer1.*, conv2s.0, convraw.0 of lib/networks/model_repository.py:22-58, and the stem in its
// space-to-depth 4x4 form), on the Hopper tensor cores (wgmma, sm_90a).
//
// Why a second kernel: with N <= 64 output channels a 128-pixel tile does too little math per byte
// for the per-tap kernel (conv_tc.cu), which re-reads the 128-pixel A tile for each of the 9 taps
// and the weights in every CTA.  Here:
//   * ALL weights of the layer (<= 147 KB) are loaded into shared memory once per CTA, and the
//     CTA is persistent over output tiles (grid = one CTA per SM, static round-robin);
//   * "halo box": for each channel chunk ONE TMA box of (TH+KH-1) x (TW+KH-1) pixels is loaded and
//     all KH x KW taps read from it: A traffic is (TH+2)(TW+2)/(TH*TW) = 1.41x the tile instead of 9x.
//     A tap's operand is the box shifted by the tap offset: a descriptor starting at that pixel, with
//     8-row groups one box row apart, addresses it in place (the swizzle follows the absolute address).
//     Both operands are shared-memory descriptors, and one chunk's MMAs stay in flight while the
//     previous chunk's stage is released;
//   * optional fused head (convraw.3 1x1 + bias + argmax) in the epilogue: the activated 128 x 32 tile
//     is already in the register layout of a wgmma A operand, so the head is one more MMA, and the
//     reference's NCHW output is written directly -- the [b,H,W,32] intermediate never exists;
//   * optional fused bilinear x2 upsampling of convraw.0's first input (the producer warps interpolate
//     it into the operand stages instead of TMA loading it).
#include "conv_tc.cuh"
#include "ptx.cuh"

#include <cstdlib>
#include <mutex>
#include <new>

namespace pvnet {

int g_conv_mode = 0;

namespace {

constexpr int COL_TH = 16, COL_TW = 8;
constexpr int COL_THREADS = 384;       // consumer warpgroups 0 and 1 (64 tile pixels each), producer warpgroup 2
constexpr int HEAD_MAX = 64;

struct ColGeom {
    int Ho, Wo, tiles_x, tiles_y, total_tiles;
    int cin_chunks, cin_pad;
    int split_chunk;        // chunks >= split_chunk are read through the second source map (== cin_chunks: none)
    int pad_l, pad_t;       // how many taps lie left of / above the output pixel
    int stages;
    int resident;           // 1: all weights loaded once per CTA; 0: the KH*KH weight tiles ride in each stage
    int out_cs, out_co, res_cs, res_co;
    int act, round_out;
    // fused head
    int head_cout, head_seg, mask_esz;
    int head_nhwc;          // fused head writes pixel-major [b,H,W,cout] instead of the reference's NCHW
};

// fused bilinear x2 upsampling of the first split_chunk channel chunks (UP variant of the kernel)
struct ColUp {
    const float *src;       // half-resolution source [b,h,w,cs], dense
    int h, w, cs;
    float sy, sx;           // ATen's align_corners scale (in-1)/(out-1)
    unsigned zero;          // always 0; opaque to the compiler (see up_fill_rows)
};

// Fused upsampling (UP variant of the kernel): producer warp q interpolates channel chunk q (8 channels)
// of one tile's halo box -- (COL_TH+2) x (COL_TW+2) full-resolution pixels, zero outside the image like
// the TMA box it replaces -- straight into the operand stage, in the 32-byte-swizzled layout TMA would
// have written (16-byte half `hf` of box row rr sits at rr*32 + ((hf ^ (rr>>2 & 1)) << 4): address bit 4
// XOR bit 7).  Arithmetic is k_upsample2x's (backbone_aux.cu), i.e. ATen's upsample_bilinear2d with
// align_corners: src = scale*dst, out = h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11), rounded to tf32.
// Lane = (box column, half): it walks its column top to bottom, keeping the horizontally interpolated
// source rows in registers (10 rows x 2 loads for 18 outputs instead of 4 loads per output).  With
// scale 2 the source row pair of output row y0-1+i is (E, E+1), E = y0/2 - 1 + i/2, except in the
// last image row when scale*y rounds below E (then it is (E-1, E)): a three-row window with one zero
// weight covers both, as in k_upsample2x.
__device__ __forceinline__ float4 ldg_nc_v4_volatile(const float *p)
{
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
// Box rows [I0, I1) of one lane's column: loads the window slots these rows need (slot 0 never: it only ever
// carries the zero weight, see above), interpolates horizontally, then vertically row by row.
template <int I0, int I1>
__device__ __forceinline__ void up_fill_rows(const float *base, unsigned rstride, unsigned olo, unsigned ohi, int R0, int uh,
                                             bool act, bool vx, float w1x_, unsigned zero, float wa_l, float wb_l, float wc_l,
                                             uint32_t sbase, int c, int hf)
{
    constexpr int PITCH = COL_TW + 2;
    constexpr int S0 = I0 >> 1, S1 = ((I1 - 1) >> 1) + 2;      // window slots of these rows
    constexpr int L0 = S0 < 1 ? 1 : S0, NL = S1 - L0 + 1;      // slots actually loaded
    // All source loads are issued before anything consumes them (volatile asm keeps them together) ...
    float4 a[NL], b[NL];
#pragma unroll
    for (int j = L0; j <= S1; ++j) {
        a[j - L0] = b[j - L0] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (act) {
            const unsigned ro = (unsigned)min(max(R0 + j, 0), uh - 1) * rstride;
            a[j - L0] = ldg_nc_v4_volatile(base + (ro + olo));
            b[j - L0] = ldg_nc_v4_volatile(base + (ro + ohi));
        }
    }
    // ... and nothing may consume them before the last one has landed: ptxas otherwise starts on the first
    // output rows as soon as their three source rows are there and parks the remaining loads behind those
    // stores (3-4 exposed L2 round trips per tile instead of one).  The interpolation weight is made to
    // depend on every load through an AND with a kernel parameter that is always zero.
    unsigned dep = 0;
#pragma unroll
    for (int j = 0; j < NL; ++j) dep |= __float_as_uint(a[j].x) | __float_as_uint(b[j].x);
    float w1x = __uint_as_float(__float_as_uint(w1x_) | (dep & zero)), w0x = 1.f - w1x_;
    if (!vx) w0x = w1x = 0.f;
    float4 t[S1 - S0 + 1];
    if (S0 == 0) t[0] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = L0; j <= S1; ++j) {
        t[j - S0].x = __fmaf_rn(w1x, b[j - L0].x, __fmul_rn(w0x, a[j - L0].x));   // lerp3 with a zero third weight
        t[j - S0].y = __fmaf_rn(w1x, b[j - L0].y, __fmul_rn(w0x, a[j - L0].y));
        t[j - S0].z = __fmaf_rn(w1x, b[j - L0].z, __fmul_rn(w0x, a[j - L0].z));
        t[j - S0].w = __fmaf_rn(w1x, b[j - L0].w, __fmul_rn(w0x, a[j - L0].w));
    }
#pragma unroll
    for (int i = I0; i < I1; ++i) {
        const float wa = __shfl_sync(0xffffffffu, wa_l, i), wb = __shfl_sync(0xffffffffu, wb_l, i),
                    wc = __shfl_sync(0xffffffffu, wc_l, i);
        const int e = (i >> 1) - S0;
        // Rounding to tf32 (nearest, ties away -- cvt.rna.tf32, what k_upsample2x stores): add half an ulp of
        // the 10-bit mantissa and clear the 13 low bits, so the MMA reads exactly the values the separate
        // launch stores.
        float4 o;
        o.x = __uint_as_float((__float_as_uint(lerp3(wa, t[e].x, wb, t[e + 1].x, wc, t[e + 2].x)) + 0x1000u) & 0xFFFFE000u);
        o.y = __uint_as_float((__float_as_uint(lerp3(wa, t[e].y, wb, t[e + 1].y, wc, t[e + 2].y)) + 0x1000u) & 0xFFFFE000u);
        o.z = __uint_as_float((__float_as_uint(lerp3(wa, t[e].z, wb, t[e + 1].z, wc, t[e + 2].z)) + 0x1000u) & 0xFFFFE000u);
        o.w = __uint_as_float((__float_as_uint(lerp3(wa, t[e].w, wb, t[e + 1].w, wc, t[e + 2].w)) + 0x1000u) & 0xFFFFE000u);
        const int rr = i * PITCH + c;
        if (act) ptx::sts128(sbase + (uint32_t)(i * PITCH * 32) + (uint32_t)((hf ^ ((rr >> 2) & 1)) << 4), o);
    }
}

// The whole column at once (20 loads in flight).
__device__ __forceinline__ void up_fill_chunk(const ColUp &u, const ColGeom &g, int img, int y0, int x0, int q, int lane,
                                              uint32_t stage_addr)
{
    constexpr int PITCH = COL_TW + 2, ROWS = COL_TH + 2;
    const bool act = lane < 2 * PITCH;                 // lanes 20..31 only take part in the shuffles
    const int c = act ? lane >> 1 : 0, hf = lane & 1;
    const int x = x0 - 1 + c;
    const bool vx = act && x >= 0 && x < g.Wo;
    const int xc = min(max(x, 0), g.Wo - 1);
    const float fx = u.sx * (float)xc;
    const int xlo = (int)fx;
    const int xhi = min(xlo + 1, u.w - 1);
    const float w1x_ = fx - (float)xlo;
    const int R0 = (y0 >> 1) - 2;
    // Vertical weights: lane r works out box row r's window weights once; the row loop fetches them with
    // three shuffles (the weights are the same for the whole warp: ~20 instructions per row otherwise).
    // Rows outside the image get zero weights -- the conv's zero padding -- and columns outside get zero
    // horizontal weights, so no output needs a select.
    float wa_l = 0.f, wb_l = 0.f, wc_l = 0.f;
    {
        const int y = y0 - 1 + lane;
        if (lane < ROWS && y >= 0 && y < g.Ho) {
            const float fy = u.sy * (float)y;
            const int ylo = (int)fy;
            const float h1 = fy - (float)ylo, h0 = 1.f - h1;
            const bool low = ylo < R0 + 1 + (lane >> 1);   // source pair is rows (E-1, E) rather than (E, E+1)
            wa_l = low ? h0 : 0.f;
            wb_l = low ? h1 : h0;
            wc_l = low ? 0.f : h1;
        }
    }
    const float *base = u.src + (size_t)img * u.h * u.w * u.cs + q * 8 + hf * 4;
    const unsigned rstride = (unsigned)u.w * (unsigned)u.cs;      // 32-bit element offsets inside one image
    const unsigned olo = (unsigned)xlo * (unsigned)u.cs, ohi = (unsigned)xhi * (unsigned)u.cs;
    const uint32_t sbase = stage_addr + (uint32_t)(c * 32);   // box row rr = i*PITCH + c sits at rr*32 + ((hf ^ bit 2 of rr) << 4)
    up_fill_rows<0, ROWS>(base, rstride, olo, ohi, R0, u.h, act, vx, w1x_, u.zero, wa_l, wb_l, wc_l, sbase, c, hf);
}



// BN = Cout (32 or 64); KC channels per chunk (rows of KC*4 bytes, swizzled by the same amount).
template <int KC, bool HEAD, int KH, bool UP, int BN>
__global__ void __launch_bounds__(COL_THREADS, 1)
    k_conv_col(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ColGeom g,
               const float *__restrict__ bias, const float *__restrict__ res, float *__restrict__ out,
               const float *__restrict__ head_w, const float *__restrict__ head_b, float *__restrict__ head_out,
               void *__restrict__ mask, const ColUp up)
{
    static_assert(!UP || (HEAD && KC == 8 && KH == 3), "fused upsampling: convraw.0 form only");
    static_assert(!HEAD || BN == 32, "fused head: 32 input channels");
    constexpr int ROWB = KC * 4;                       // bytes per K-major row
    constexpr int B_TILE = BN * ROWB;                  // one [BN][KC] weight tile (a multiple of 1024 bytes)
    constexpr int PITCH = COL_TW + KH - 1;             // box pitch in pixels (= shared-memory rows)
    constexpr int A_BOX = (COL_TH + KH - 1) * PITCH * ROWB;
    constexpr int A_BYTES = (A_BOX + 1023) & ~1023;    // stages stay 1024-byte aligned
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int n_btiles = KH * KH * g.cin_chunks;
    const int stage_bytes = A_BYTES + (g.resident ? 0 : KH * KH * B_TILE);
    uint8_t *sB = smem;
    uint8_t *sA = smem + (g.resident ? (size_t)n_btiles * B_TILE : 0);
    uint8_t *sH = sA + (size_t)g.stages * stage_bytes;            // HEAD: head weights, 32 x 32, 128-byte swizzle
    uint64_t *wfull = reinterpret_cast<uint64_t *>(sH + (HEAD ? 4096 : 0));
    uint64_t *full = wfull + 1;
    uint64_t *empty = full + g.stages;
    float *s_bias = reinterpret_cast<float *>(empty + g.stages);  // [BN]
    float *s_head = s_bias + 64;                                  // [32]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        ptx::mbar_init(wfull, 1);
        for (int s = 0; s < g.stages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], 8);              // one arrive per consumer warp
        }
        ptx::fence_barrier_init();
    }
    for (int i = threadIdx.x; i < BN; i += blockDim.x) s_bias[i] = bias[i];
    if (HEAD) {
        for (int i = threadIdx.x; i < 32; i += blockDim.x) s_head[i] = i < g.head_cout ? head_b[i] : 0.f;
        // convraw.3 weights [cout][32] as the B operand of the head MMA, rows >= cout zero.  K is stored permuted
        // within each group of 8 (position p < 4 holds channel 2p, position p >= 4 channel 2(p-4)+1): the order in
        // which the accumulator fragment of the 3x3 conv hands its channels to the A fragment of the head MMA.
        for (int i = threadIdx.x; i < 32 * 32; i += blockDim.x) {
            const int n = i >> 5, p = i & 31, q = p & 7;
            const int k = (p & ~7) + (q < 4 ? 2 * q : 2 * (q - 4) + 1);
            const float v = n < g.head_cout ? head_w[n * 32 + k] : 0.f;
            *reinterpret_cast<float *>(sH + ptx::swizzle_off((uint32_t)(n * 128 + p * 4), 128)) = v;
        }
        ptx::fence_proxy_async();                      // generic stores -> read by the MMA (async proxy)
    }
    __syncthreads();
    const int tiles_per_img = g.tiles_x * g.tiles_y;

    if (warp >= 8) {
        // producer warpgroup: warp 8 lane 0 issues the TMA loads; with UP, warp 8 + q also interpolates chunk q
        const int pw = warp - 8;
        if (pw == 0 && lane == 0 && g.resident) {
            // all weights, once: tile t = cc*KH*KH + kh*KH + kw <- packed [Cout][kh][kw][cin]
            ptx::mbar_arrive_expect_tx(wfull, (uint32_t)(n_btiles * B_TILE));
            for (int cc = 0; cc < g.cin_chunks; ++cc)
                for (int t = 0; t < KH * KH; ++t)
                    ptx::tma_load_2d(sB + (size_t)(cc * KH * KH + t) * B_TILE, &tmB, wfull, t * g.cin_pad + cc * KC, 0);
        }
        if (!UP && pw != 0) return;
        int s = 0;
        uint32_t ph = 0;
        const uint32_t tx_bytes = (uint32_t)(A_BOX + (g.resident ? 0 : KH * KH * B_TILE));
        for (int tile = blockIdx.x; tile < g.total_tiles; tile += gridDim.x) {
            const int img = tile / tiles_per_img;
            const int trem = tile - img * tiles_per_img;
            const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
            const int y0 = tyi * COL_TH, x0 = txi * COL_TW;
            for (int cc = 0; cc < g.cin_chunks; ++cc) {
                uint8_t *st = sA + (size_t)s * stage_bytes;
                if (UP && cc < g.split_chunk) {
                    if (pw == cc) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        up_fill_chunk(up, g, img, y0, x0, cc, lane, ptx::smem_u32(st));
                        // generic-proxy stores into a stage that a later round refills by TMA (async proxy)
                        ptx::fence_proxy_async();
                        __syncwarp();
                        if (lane == 0) ptx::mbar_arrive(&full[s]);
                    }
                } else if (pw == 0) {
                    if (lane == 0) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        ptx::mbar_arrive_expect_tx(&full[s], tx_bytes);
                        if (cc < g.split_chunk)
                            ptx::tma_load_4d(st, &tmA, &full[s], cc * KC, x0 - g.pad_l, y0 - g.pad_t, img);
                        else
                            ptx::tma_load_4d(st, &tmA2, &full[s], (cc - g.split_chunk) * KC, x0 - g.pad_l, y0 - g.pad_t, img);
                        if (!g.resident)
                            for (int t = 0; t < KH * KH; ++t)
                                ptx::tma_load_2d(st + A_BYTES + (size_t)t * B_TILE, &tmB, &full[s], t * g.cin_pad + cc * KC, 0);
                    }
                    __syncwarp();
                }
                if (++s == g.stages) {
                    s = 0;
                    ph ^= 1u;
                }
            }
        }
        return;
    }

    // consumer warpgroup wg: tile rows [8 wg, 8 wg + 8).  At tap (kh, kw) its 64 A rows are 8 core-matrix groups
    // of 8 consecutive box pixels, group i at box row 8 wg + i + kh from column kw: a K-major operand whose groups
    // are PITCH box pixels apart, addressed by a descriptor that starts at that pixel (see make_kmajor_desc).
    // Thread (wq, lane) holds the accumulator rows of tile pixels (8 wg + 2 wq, g8) and (8 wg + 2 wq + 1, g8).
    const int wg = warp >> 2, wq = warp & 3;
    const int g8 = lane >> 2, t4 = lane & 3;
    const uint32_t sA_u = ptx::smem_u32(sA), sB_u = ptx::smem_u32(sB);
    if (g.resident) ptx::mbar_wait(wfull, 0);
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < g.total_tiles; tile += gridDim.x) {
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int cc = 0; cc < g.cin_chunks; ++cc) {
            ptx::mbar_wait(&full[s], ph);
            const uint32_t a0 = sA_u + (uint32_t)s * (uint32_t)stage_bytes;
            const uint32_t b0 = g.resident ? sB_u + (uint32_t)(cc * KH * KH * B_TILE) : a0 + (uint32_t)A_BYTES;
            const uint64_t ad0 = ptx::make_kmajor_desc(a0 + (uint32_t)(8 * wg * PITCH * ROWB), ROWB, PITCH * ROWB);
            const uint64_t bd0 = ptx::make_kmajor_desc(b0, ROWB);
            // the chunk's taps, then 8-channel K steps, into one accumulator; descriptor start addresses count
            // 16-byte units
            ptx::wgmma_fence();
#pragma unroll
            for (int t = 0; t < KH * KH; ++t) {
                const uint64_t ad = ad0 + (uint64_t)(((t / KH) * PITCH + t % KH) * ROWB / 16);
                const uint64_t bd = bd0 + (uint64_t)(t * B_TILE / 16);
#pragma unroll
                for (int ks = 0; ks < KC / 8; ++ks)
                    ptx::Wgmma<BN>::ss(acc, ad + (uint64_t)(2 * ks), bd + (uint64_t)(2 * ks), (cc | t | ks) != 0 ? 1u : 0u);
            }
            ptx::wgmma_commit();
            // the previous chunk's MMAs have finished reading their stage: hand it back
            ptx::wgmma_wait<1>();
            ptx::fence_regs(acc);
            if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
            prev = s;
            if (++s == g.stages) {
                s = 0;
                ph ^= 1u;
            }
        }
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
        if (lane == 0) ptx::mbar_arrive(&empty[prev]);

        const int img = tile / tiles_per_img;
        const int trem = tile - img * tiles_per_img;
        const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
        const int ty = 8 * wg + 2 * wq;
        if constexpr (!HEAD) {
            bool ok[2];
            size_t pix[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int y = tyi * COL_TH + ty + h, x = txi * COL_TW + g8;
                ok[h] = y < g.Ho && x < g.Wo;
                pix[h] = ok[h] ? ((size_t)img * g.Ho + y) * g.Wo + x : 0;
            }
            // every residual load of the thread's two pixels is issued before any arithmetic: the epilogue waits
            // for one load latency rather than one per 8-channel block
            float2 rv[2][BN / 8];
            if (res) {
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int j = 0; j < BN / 8; ++j)
                        rv[h][j] = ok[h] ? __ldg(reinterpret_cast<const float2 *>(res + pix[h] * g.res_cs + g.res_co + 8 * j + 2 * t4))
                                         : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!ok[h]) continue;
                float *optr = out + pix[h] * g.out_cs + g.out_co;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = 8 * j + 2 * t4;
                    float2 v = make_float2(acc[4 * j + 2 * h] + s_bias[c], acc[4 * j + 2 * h + 1] + s_bias[c + 1]);
                    if (res) {
                        v.x += rv[h][j].x;
                        v.y += rv[h][j].y;
                    }
                    v.x = epi_act(v.x, g.act, g.round_out);
                    v.y = epi_act(v.y, g.act, g.round_out);
                    *reinterpret_cast<float2 *>(optr + c) = v;
                }
            }
        } else {
            // convraw.3 (model_repository.py:57): the activated, tf32-rounded tile is the A operand of a
            // 128 x 32 x 32 MMA against the head weights; accumulator entry (row, 8j+2t+e) is K position
            // 8j+t+4e of step j, matching the permuted B rows written above.
            uint32_t a2[4][4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int f = 0; f < 4; ++f) {
                    const int r = 4 * j + ((f & 1) << 1) + (f >> 1);      // f: (row g, k t), (g+8, t), (g, t+4), (g+8, t+4)
                    const int c = 8 * j + 2 * t4 + (f >> 1);
                    a2[j][f] = __float_as_uint(ptx::round_tf32(epi_act(acc[r] + s_bias[c], g.act, g.round_out)));
                }
            float hacc[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) hacc[i] = 0.f;
            const uint64_t hd = ptx::make_kmajor_desc(ptx::smem_u32(sH), 128);
            ptx::wgmma_fence();
#pragma unroll
            for (int j = 0; j < 4; ++j) ptx::Wgmma<32>::rs(hacc, a2[j], hd + (uint64_t)(2 * j), j != 0 ? 1u : 0u);
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::fence_regs(hacc);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int y = tyi * COL_TH + ty + h, x = txi * COL_TW + g8;
                const bool valid = y < g.Ho && x < g.Wo;
                const size_t pix = ((size_t)img * g.Ho + y) * g.Wo + x;
                const size_t npix = (size_t)g.Ho * g.Wo;
                float best = -INFINITY;
                int best_c = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int co = 8 * j + 2 * t4 + e;
                        const float val = hacc[4 * j + 2 * h + e] + s_head[co];
                        if (co < g.head_seg && val > best) {
                            best = val;
                            best_c = co;
                        }
                        if (valid && co < g.head_cout) {
                            if (g.head_nhwc) head_out[pix * (size_t)g.head_cout + co] = val;
                            else head_out[((size_t)img * g.head_cout + co) * npix + (size_t)y * g.Wo + x] = val;
                        }
                    }
                // torch.argmax over the four lanes of the pixel: the largest value, the lowest channel among equals
#pragma unroll
                for (int o = 1; o < 4; o <<= 1) {
                    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                    const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
                    if (ob > best || (ob == best && oc < best_c)) {
                        best = ob;
                        best_c = oc;
                    }
                }
                if (valid && mask && t4 == 0) {
                    if (g.mask_esz == 8) reinterpret_cast<long long *>(mask)[pix] = best_c;
                    else reinterpret_cast<unsigned char *>(mask)[pix] = (unsigned char)best_c;
                }
            }
        }
    }
}

struct ColPlan {
    CUtensorMap tmA, tmA2, tmB;
    ColGeom g;
    int kc, ksize, head, up, bn;
    ColUp cup;
    unsigned grid;
    size_t smem;
    const float *bias, *res;
    float *out;
    HeadDesc hd;
};

constexpr size_t SMEM_LIMIT = 227 * 1024;

// K-chunk: 128-byte rows when Cin is a multiple of 32, 64-byte rows for the 16-channel stem, else
// 32-byte rows (Cin=40: 8-channel chunks instead of zero-padded 32-channel ones).
int col_kc(int Cin) { return Cin % 32 == 0 ? 32 : (Cin == 16 ? 16 : 8); }
int col_cin_pad(int Cin) { return Cin == 16 ? 16 : (Cin + 31) / 32 * 32; }   // packing of the weights

size_t col_smem(int kc, int ksize, int cin_chunks, int bn, int stages, bool head, bool resident)
{
    const size_t rowb = (size_t)kc * 4;
    const size_t a_box = (size_t)(COL_TH + ksize - 1) * (COL_TW + ksize - 1) * rowb;
    const size_t a = (a_box + 1023) & ~(size_t)1023, bt = (size_t)bn * rowb;
    return 1024 + (resident ? (size_t)ksize * ksize * cin_chunks * bt : 0) +
           (size_t)stages * (a + (resident ? 0 : (size_t)ksize * ksize * bt)) + (head ? 4096 : 0) +
           (size_t)(1 + 2 * stages) * 8 + (64 + 32) * 4;
}

template <int KC, bool HEAD, int KH, bool UP, int BN>
int col_launch(const ColPlan &p, cudaStream_t s)
{
    // the instantiation must be the plan's: weight boxes, barrier byte counts and stores are sized by BN
    if (p.bn != BN || p.kc != KC || p.ksize != KH || p.head != (HEAD ? 1 : 0) || p.up != (UP ? 1 : 0)) {
        set_error("conv(col): no kernel instantiation for this plan (Cout %d, chunk %d, ksize %d)", p.bn, p.kc, p.ksize);
        return PVNET_E_STATE;
    }
    auto fn = k_conv_col<KC, HEAD, KH, UP, BN>;
    const cudaError_t attr_err = ensure_max_smem((const void *)fn, (int)SMEM_LIMIT);
    PV_CUDA(attr_err);
    const HeadDesc &h = p.hd;
    fn<<<p.grid, COL_THREADS, p.smem, s>>>(p.tmA, p.tmA2, p.tmB, p.g, p.bias, p.res, p.out, p.head ? h.w : nullptr,
                                           p.head ? h.bias : nullptr, p.head ? h.out_nchw : nullptr,
                                           p.head ? h.mask : nullptr, p.cup);
    PV_LAUNCHED("k_conv_col");
    return PVNET_OK;
}

}  // namespace

bool conv_col_eligible(const ConvDesc &d)
{
    // ksize 4 = the space-to-depth form of the 7x7/2 stem: taps at offsets {-2,-1,0,1}
    if ((d.ksize != 3 && d.ksize != 4) || d.stride != 1 || d.dilation != 1 || d.Cout > 64 || d.Cout % 32 != 0)
        return false;
    const int cin = d.Cin + d.Cin2;
    const int kc = col_kc(cin);
    if (d.Cin % kc != 0 || d.Cin2 % kc != 0) return false;
    if ((d.ksize == 4) != (kc == 16)) return false;   // instantiated: 4x4 taps with 16 channels, 3x3 otherwise
    return col_smem(kc, d.ksize, (cin + kc - 1) / kc, d.Cout, 2, true, false) <= SMEM_LIMIT;
}

size_t conv_col_plan_size() { return sizeof(ColPlan); }

int conv_col_plan_at(const ConvDesc &d, const HeadDesc *head, void *storage)
{
    ColPlan *p = new (storage) ColPlan();
    PV_CHECK_ARG(conv_col_eligible(d), "conv(col): layer not eligible for the column kernel");
    PV_CHECK_ARG((d.in || d.up_src) && d.w && d.bias && (d.out || head), "conv(col): null pointer");
    PV_CHECK_ARG(!d.up_src || (head && d.in2 && col_kc(d.Cin + d.Cin2) == 8 && d.Cin == 32 && d.Cin2 == 8 && d.ksize == 3 &&
                               d.H % 2 == 0 && d.W % 2 == 0 && (uintptr_t)d.up_src % 16 == 0),
                 "conv(col): fused upsampling needs the convraw.0 form (32 upsampled + 8 direct channels, fused head)");
    PV_CHECK_ARG(d.in_cs % 4 == 0 && d.in_co % 4 == 0 && d.out_cs % 4 == 0 && d.out_co % 4 == 0,
                 "conv(col): channel strides/offsets must be multiples of 4 floats");
    PV_CHECK_ARG(!d.res || (d.res_cs % 4 == 0 && d.res_co % 4 == 0), "conv(col): residual stride/offset alignment");
    PV_CHECK_ARG(!head || (d.Cout == 32 && col_kc(d.Cin + d.Cin2) != 16 && head->cout >= 1 && head->cout <= 32 && head->w && head->bias &&
                           head->out_nchw && (!head->mask || head->mask_esz == 1 || head->mask_esz == 8)),
                 "conv(col): bad fused-head description");
    const int kc = col_kc(d.Cin + d.Cin2);
    ColGeom &g = p->g;
    g.pad_l = g.pad_t = d.ksize == 4 ? 2 : 1;
    g.Ho = d.H;
    g.Wo = d.W;
    g.tiles_x = (d.W + COL_TW - 1) / COL_TW;
    g.tiles_y = (d.H + COL_TH - 1) / COL_TH;
    g.total_tiles = g.tiles_x * g.tiles_y * d.b;
    g.cin_chunks = (d.Cin + d.Cin2) / kc;
    g.split_chunk = d.in2 ? d.Cin / kc : g.cin_chunks;
    g.cin_pad = col_cin_pad(d.Cin + d.Cin2);   // weights are packed [Cout][KH][KW][cin_pad], zero padded
    g.out_cs = d.out_cs;
    g.out_co = d.out_co;
    g.res_cs = d.res_cs;
    g.res_co = d.res_co;
    g.act = d.act;
    g.round_out = d.round_out;
    g.head_cout = head ? head->cout : 0;
    g.head_seg = head ? head->seg_dim : 0;
    g.mask_esz = head ? head->mask_esz : 0;
    g.head_nhwc = 0;
    p->cup.src = d.up_src;
    p->cup.h = d.H / 2;
    p->cup.w = d.W / 2;
    p->cup.cs = d.Cin;
    p->cup.sy = (float)(p->cup.h - 1) / (float)(2 * p->cup.h - 1);   // launch_upsample2x's scales
    p->cup.sx = (float)(p->cup.w - 1) / (float)(2 * p->cup.w - 1);
    p->cup.zero = 0;
    // Resident weights whenever at least 2 A stages (one channel chunk with all its taps each) still
    // fit next to them; otherwise the KH*KW weight tiles of a chunk travel with its A box.
    const bool hd = head != nullptr;
    int stages = 8;
    bool resident = true;
    while (stages > 2 && col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, true) > SMEM_LIMIT) --stages;
    if (col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, true) > SMEM_LIMIT) {
        resident = false;
        stages = 8;
        while (stages > 2 && col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, false) > SMEM_LIMIT) --stages;
    }
    PV_CHECK_ARG(!d.up_src || resident, "conv(col): fused upsampling needs resident weights");
    g.stages = stages;
    g.resident = resident ? 1 : 0;
    p->smem = col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, resident);
    p->kc = kc;
    p->ksize = d.ksize;
    p->bn = d.Cout;
    p->head = hd ? 1 : 0;
    p->up = d.up_src ? 1 : 0;
    if (head) p->hd = *head;
    if (!d.up_src) {
        const float *base = d.in + d.in_co;
        cuuint64_t dims[4] = {(cuuint64_t)d.Cin, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.b};
        cuuint64_t strides[3] = {(cuuint64_t)d.in_cs * 4, (cuuint64_t)d.W * d.in_cs * 4,
                                 (cuuint64_t)d.H * d.W * d.in_cs * 4};
        cuuint32_t box[4] = {(cuuint32_t)kc, (cuuint32_t)(COL_TW + d.ksize - 1), (cuuint32_t)(COL_TH + d.ksize - 1), 1};
        int rc = tma_encode(&p->tmA, base, 4, dims, strides, box, kc * 4);
        if (rc) return rc;
        p->tmA2 = p->tmA;
    }
    if (d.in2) {
        PV_CHECK_ARG(d.in2_cs % 4 == 0 && d.in2_co % 4 == 0 && d.Cin2 > 0, "conv(col): second source stride/offset alignment");
        cuuint64_t dims[4] = {(cuuint64_t)d.Cin2, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.b};
        cuuint64_t strides[3] = {(cuuint64_t)d.in2_cs * 4, (cuuint64_t)d.W * d.in2_cs * 4,
                                 (cuuint64_t)d.H * d.W * d.in2_cs * 4};
        cuuint32_t box[4] = {(cuuint32_t)kc, (cuuint32_t)(COL_TW + d.ksize - 1), (cuuint32_t)(COL_TH + d.ksize - 1), 1};
        int rc = tma_encode(&p->tmA2, d.in2 + d.in2_co, 4, dims, strides, box, kc * 4);
        if (rc) return rc;
        if (d.up_src) p->tmA = p->tmA2;     // the first source is interpolated in the kernel, not read by TMA
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)d.ksize * d.ksize * g.cin_pad, (cuuint64_t)d.Cout};
        cuuint64_t strides[1] = {(cuuint64_t)d.ksize * d.ksize * g.cin_pad * 4};
        cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)d.Cout};
        int rc = tma_encode(&p->tmB, d.w, 2, dims, strides, box, kc * 4);
        if (rc) return rc;
    }
    PV_CHECK_ARG(!head || (uintptr_t)head->w % 16 == 0, "conv(col): head weights must be 16-byte aligned");
    long long grid = (long long)sm_count();
    if (grid > g.total_tiles) grid = g.total_tiles;
    p->grid = (unsigned)grid;
    p->bias = d.bias;
    p->res = d.res;
    p->out = d.out;
    return PVNET_OK;
}

void conv_col_set_head_ptrs(void *storage, float *out_nchw, void *mask, int mask_esz, int nhwc)
{
    ColPlan *p = static_cast<ColPlan *>(storage);
    p->g.head_nhwc = nhwc;
    p->hd.out_nchw = out_nchw;
    p->hd.mask = mask;
    p->hd.mask_esz = mask_esz;
    p->g.mask_esz = mask_esz;
}

int conv_col_launch_at(const void *storage, cudaStream_t s)
{
    const ColPlan &p = *static_cast<const ColPlan *>(storage);
    if (p.up) return col_launch<8, true, 3, true, 32>(p, s);
    if (p.head) return p.kc == 32 ? col_launch<32, true, 3, false, 32>(p, s) : col_launch<8, true, 3, false, 32>(p, s);
    const bool n64 = p.bn == 64;
    if (p.ksize == 4) return n64 ? col_launch<16, false, 4, false, 64>(p, s) : col_launch<16, false, 4, false, 32>(p, s);
    if (p.kc == 32) return n64 ? col_launch<32, false, 3, false, 64>(p, s) : col_launch<32, false, 3, false, 32>(p, s);
    if (p.kc == 16) return n64 ? col_launch<16, false, 3, false, 64>(p, s) : col_launch<16, false, 3, false, 32>(p, s);
    return n64 ? col_launch<8, false, 3, false, 64>(p, s) : col_launch<8, false, 3, false, 32>(p, s);
}

}  // namespace pvnet

extern "C" {
// test hook: 0 auto, 1 force the per-tap kernel, 2 force the column kernel
int pvnet_conv_set_mode(int mode)
{
    PV_CHECK_ARG(mode >= 0 && mode <= 2, "mode must be 0, 1 or 2");
    pvnet::g_conv_mode = mode;
    return PVNET_OK;
}
}
