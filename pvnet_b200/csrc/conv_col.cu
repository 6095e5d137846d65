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
//     is already in the register layout of a wgmma A operand, so the head is one more MMA; its output is staged
//     in shared memory and stored by the producer warpgroup's otherwise idle warps while the next tile's MMAs
//     run -- the [b,H,W,32] intermediate never exists.
//
// k_conv_col<KC, HEAD, KH, BN, WIDE, SPLIT8> is instantiated per layer form, nine in all: 3x3 taps with 32- or
// 8-channel chunks and BN = Cout 32 or 64; the stem's 4x4 taps with 16-channel chunks, BN 32 or 64; convraw.0's fused
// head (HEAD, 8-channel chunks, BN 32), with or without WIDE, its two-source input with the 32-channel first source
// loaded as one 128-byte-swizzled box; and SPLIT8 (32-channel chunks, BN 64): Resnet50_8s_2o's conv2s.0, whose first
// source runs in 32-channel chunks and whose 8-channel second source is one more chunk.  conv_col_launch_at picks the
// instantiation a plan was made for.
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

// Fused head: one tile's output (128 pixels x head_cout fp32, then 128 argmax bytes) is staged in shared memory,
// double-buffered, and copied to global memory by warps that issue no MMAs.  Pixel-major staging keeps a pixel's
// channels at a pitch of 8 mod 16 floats, so the consumers' float2 writes (lane = pixel g8, channel pair t4) hit
// four disjoint 8-bank windows per half-warp; NCHW staging is [cout][16][8] with a channel pitch of 4 mod 16
// floats, so the scalar writes of channels 2t4 and 2t4+1 spread the four t4 lanes 8 banks apart.
__host__ __device__ constexpr int head_pitch(int hc) { return hc <= 8 ? 8 : (hc <= 24 ? 24 : 40); }
constexpr int HEAD_CPITCH = COL_TH * COL_TW + 4;
__host__ __device__ constexpr int head_stage_floats(int hc)
{
    return COL_TH * COL_TW * head_pitch(hc) > hc * HEAD_CPITCH ? COL_TH * COL_TW * head_pitch(hc) : hc * HEAD_CPITCH;
}
__host__ __device__ constexpr int head_stage_bytes(int hc) { return (head_stage_floats(hc) * 4 + COL_TH * COL_TW + 127) & ~127; }

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

// Copies one staged head tile (see head_pitch) to head_out and mask; thread `tid` of `nthr`.  The tile is 32*hc
// units of four floats: pixel-major, 2*hc of them cover one tile row's contiguous run of 8*hc floats; NCHW, two
// cover one channel's 8 pixels of a tile row.  A unit is one 16-byte store when the layout keeps it aligned and
// inside one pixel (pixel-major) or inside the image (NCHW), otherwise four scalar stores.  sv and sm are the
// shared-memory addresses of the staged values and argmax bytes.
__device__ __forceinline__ void head_store_tile(const ColGeom &g, uint32_t sv, uint32_t sm, float *head_out, void *mask,
                                                int img, int y0, int x0, int tid, int nthr)
{
    const int hc = g.head_cout, pp = head_pitch(hc);
    const int nx = min(COL_TW, g.Wo - x0), ny = min(COL_TH, g.Ho - y0);
    const size_t npix = (size_t)g.Ho * g.Wo;
    const bool vec = (reinterpret_cast<uintptr_t>(head_out) & 15) == 0 && (g.head_nhwc ? hc % 4 == 0 : g.Wo % 4 == 0);
    for (int u = tid; u < 32 * hc; u += nthr) {
        if (g.head_nhwc) {
            const int r = u / (2 * hc), e0 = 4 * (u - r * 2 * hc);
            if (r >= ny) continue;
            float *dst = head_out + (((size_t)img * g.Ho + y0 + r) * g.Wo + x0) * hc + e0;
            if (vec) {
                const int col = e0 / hc;
                if (col < nx)
                    *reinterpret_cast<float4 *>(dst) = ptx::lds128(sv + 4u * (uint32_t)((r * COL_TW + col) * pp + e0 - col * hc));
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int col = (e0 + i) / hc;
                    if (col < nx) dst[i] = ptx::lds32(sv + 4u * (uint32_t)((r * COL_TW + col) * pp + e0 + i - col * hc));
                }
            }
        } else {
            const int co = u >> 5, r = (u >> 1) & 15, xo = 4 * (u & 1);
            if (r >= ny) continue;
            float *dst = head_out + ((size_t)img * hc + co) * npix + (size_t)(y0 + r) * g.Wo + x0 + xo;
            const uint32_t src = sv + 4u * (uint32_t)(co * HEAD_CPITCH + r * COL_TW + xo);
            if (vec) {
                if (xo < nx) *reinterpret_cast<float4 *>(dst) = ptx::lds128(src);
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (xo + i < nx) dst[i] = ptx::lds32(src + 4u * i);
            }
        }
    }
    if (!mask) return;
    for (int p = tid; p < COL_TH * COL_TW; p += nthr) {
        const int r = p / COL_TW, c = p % COL_TW;
        if (r >= ny || c >= nx) continue;
        const size_t pix = ((size_t)img * g.Ho + y0 + r) * g.Wo + x0 + c;
        const uint32_t v = ptx::lds8(sm + (uint32_t)p);
        if (g.mask_esz == 8) reinterpret_cast<long long *>(mask)[pix] = v;
        else reinterpret_cast<unsigned char *>(mask)[pix] = (unsigned char)v;
    }
}

// BN = Cout (32 or 64); KC channels per chunk (rows of KC*4 bytes, swizzled by the same amount).
// WIDE (convraw.0 with a 32-channel first source): the four 8-channel chunks of the first source are loaded as one
// 128-byte-swizzled box, with their weights as 128-byte-swizzled [32][32] tiles, and the MMAs still run chunk by
// chunk, tap by tap, so every output sums the same products in the same order as with 8-channel boxes.  The
// 32-byte-swizzled operands of 8-channel chunks ran the same MMAs at about half the rate (DESIGN.md section 6).
// SPLIT8 (KC = 32, weights not resident): chunk split_chunk, the last, is the second source's 8 channels: a box of
// 32-byte rows from tmA2 with its KH*KH [BN][8] weight tiles (32-byte swizzle, tmBw) in the same stage.  The first
// source keeps 128-byte rows, so a 192 + 8 channel input does not fall back to 8-channel chunks (DESIGN.md §21).
template <int KC, bool HEAD, int KH, int BN, bool WIDE = false, bool SPLIT8 = false>
__global__ void __launch_bounds__(COL_THREADS, 1)
    k_conv_col(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmBw, const __grid_constant__ ColGeom g,
               const float *__restrict__ bias, const float *__restrict__ res, float *__restrict__ out,
               const float *__restrict__ head_w, const float *__restrict__ head_b, float *__restrict__ head_out,
               void *__restrict__ mask)
{
    static_assert(!HEAD || BN == 32, "fused head: 32 input channels");
    static_assert(!HEAD || KC == 8, "fused head: convraw.0's 8-channel chunks");
    static_assert((KC == 16) == (KH == 4), "16-channel chunks are the 4x4 stem's, and only its");
    static_assert(!WIDE || (HEAD && KC == 8 && KH == 3), "wide first source: convraw.0 form only");
    static_assert(!SPLIT8 || (!HEAD && !WIDE && KC == 32 && KH == 3), "split chunks: 32-channel first source, 3x3");
    constexpr int ROWB = KC * 4;                       // bytes per K-major row
    constexpr int B_TILE = BN * ROWB;                  // one [BN][KC] weight tile (a multiple of 1024 bytes)
    constexpr int PITCH = COL_TW + KH - 1;             // box pitch in pixels (= shared-memory rows)
    constexpr int A_BOX = (COL_TH + KH - 1) * PITCH * ROWB;
    constexpr int A_BYTES = (A_BOX + 1023) & ~1023;    // stages stay 1024-byte aligned
    // WIDE: the first source's 32 channels arrive as one box of 128-byte rows (WIDE_BOX), the second source's 8 as
    // a box of 32-byte rows; a stage is sized for the wide box
    constexpr int WIDE_BOX = (COL_TH + KH - 1) * PITCH * 128;
    constexpr int WIDE_BYTES = (WIDE_BOX + 1023) & ~1023;
    // SPLIT8: the 8-channel chunk's box and weight tile (32-byte rows)
    constexpr int T_A_BOX = (COL_TH + KH - 1) * PITCH * 32, T_B_TILE = BN * 32;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int n_btiles = KH * KH * g.cin_chunks;
    const int n_loads = WIDE ? 2 : g.cin_chunks;         // operand boxes per tile (one ring stage each)
    const int stage_bytes = WIDE ? WIDE_BYTES : A_BYTES + (g.resident ? 0 : KH * KH * B_TILE);
    uint8_t *sB = smem;
    uint8_t *sA = smem + (g.resident ? (size_t)n_btiles * B_TILE : 0);
    uint8_t *sH = sA + (size_t)g.stages * stage_bytes;            // HEAD: head weights, 32 x 32, 128-byte swizzle
    uint8_t *sHS = sH + (HEAD ? 4096 : 0);                        // HEAD: two head output staging buffers
    const int hs_bytes = HEAD ? head_stage_bytes(g.head_cout) : 0;
    uint64_t *wfull = reinterpret_cast<uint64_t *>(sHS + 2 * hs_bytes);
    uint64_t *full = wfull + 1;
    uint64_t *empty = full + g.stages;
    uint64_t *hstaged = empty + g.stages;                         // HEAD: [2] staging buffer written by the consumers
    uint64_t *hfree = hstaged + 2;                                // HEAD: [2] staging buffer copied out by the store warps
    float *s_bias = reinterpret_cast<float *>(empty + g.stages + (HEAD ? 4 : 0));  // [BN]
    float *s_head = s_bias + 64;                                  // [32]
    constexpr int STORE_THREADS = 96;                             // HEAD: producer warps 9-11 store the head output

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        ptx::mbar_init(wfull, 1);
        for (int s = 0; s < g.stages; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], 8);              // one arrive per consumer warp
        }
        if (HEAD)
            for (int b = 0; b < 2; ++b) {
                ptx::mbar_init(&hstaged[b], 256);      // every consumer thread, after its own shared-memory writes
                ptx::mbar_init(&hfree[b], STORE_THREADS);
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
        // producer warpgroup: warp 8 lane 0 issues the TMA loads; with HEAD, warps 9-11 store the head output
        const int pw = warp - 8;
        if (pw == 0 && lane == 0 && g.resident) {
            // all weights, once: tile t = cc*KH*KH + kh*KH + kw <- packed [Cout][kh][kw][cin]; WIDE: the first
            // source's chunks as KH*KH [BN][32] tiles of 128-byte rows, in the same bytes
            ptx::mbar_arrive_expect_tx(wfull, (uint32_t)(n_btiles * B_TILE));
            for (int cc = WIDE ? g.split_chunk : 0; cc < g.cin_chunks; ++cc)
                for (int t = 0; t < KH * KH; ++t)
                    ptx::tma_load_2d(sB + (size_t)(cc * KH * KH + t) * B_TILE, &tmB, wfull, t * g.cin_pad + cc * KC, 0);
            if (WIDE)
                for (int t = 0; t < KH * KH; ++t) ptx::tma_load_2d(sB + (size_t)t * BN * 128, &tmBw, wfull, t * g.cin_pad, 0);
        }
        if (HEAD && pw != 0) {
            // store warps: the CTA's tiles in the consumers' order, buffer it & 1, the ring's parity discipline
            const int tid = threadIdx.x - 9 * 32;
            int it = 0;
            for (int tile = blockIdx.x; tile < g.total_tiles; tile += gridDim.x, ++it) {
                const int b = it & 1;
                const int img = tile / tiles_per_img;
                const int trem = tile - img * tiles_per_img;
                const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
                const uint32_t buf = ptx::smem_u32(sHS) + (uint32_t)(b * hs_bytes);
                ptx::mbar_wait(&hstaged[b], (uint32_t)(it >> 1) & 1u);
                head_store_tile(g, buf, buf + 4u * (uint32_t)head_stage_floats(g.head_cout), head_out, mask, img, tyi * COL_TH,
                                txi * COL_TW, tid, STORE_THREADS);
                ptx::mbar_arrive(&hfree[b]);
            }
            return;
        }
        if (pw != 0) return;
        int s = 0;
        uint32_t ph = 0;
        const uint32_t tx_bytes = (uint32_t)(A_BOX + (g.resident ? 0 : KH * KH * B_TILE));
        for (int tile = blockIdx.x; tile < g.total_tiles; tile += gridDim.x) {
            const int img = tile / tiles_per_img;
            const int trem = tile - img * tiles_per_img;
            const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
            const int y0 = tyi * COL_TH, x0 = txi * COL_TW;
            for (int cc = 0; cc < n_loads; ++cc) {
                uint8_t *st = sA + (size_t)s * stage_bytes;
                if (WIDE) {
                    if (pw == 0 && lane == 0) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)(cc == 0 ? WIDE_BOX : A_BOX));
                        ptx::tma_load_4d(st, cc == 0 ? &tmA : &tmA2, &full[s], 0, x0 - g.pad_l, y0 - g.pad_t, img);
                    }
                    __syncwarp();
                } else if (SPLIT8 && cc == g.split_chunk) {
                    if (lane == 0) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)(T_A_BOX + KH * KH * T_B_TILE));
                        ptx::tma_load_4d(st, &tmA2, &full[s], 0, x0 - g.pad_l, y0 - g.pad_t, img);
                        for (int t = 0; t < KH * KH; ++t)
                            ptx::tma_load_2d(st + A_BYTES + (size_t)t * T_B_TILE, &tmBw, &full[s], t * g.cin_pad + cc * KC, 0);
                    }
                    __syncwarp();
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
    int it = 0;
    for (int tile = blockIdx.x; tile < g.total_tiles; tile += gridDim.x, ++it) {
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int cc = 0; cc < n_loads; ++cc) {
            ptx::mbar_wait(&full[s], ph);
            const uint32_t a0 = sA_u + (uint32_t)s * (uint32_t)stage_bytes;
            ptx::wgmma_fence();
            if (WIDE && cc == 0) {
                // the first source's four 8-channel chunks (32-byte K steps inside the 128-byte rows), each over
                // all taps: the order of the 8-channel-box form
                const uint64_t ad0 = ptx::make_kmajor_desc(a0 + (uint32_t)(8 * wg * PITCH * 128), 128, PITCH * 128);
                const uint64_t bd0 = ptx::make_kmajor_desc(sB_u, 128);
#pragma unroll
                for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                    for (int t = 0; t < KH * KH; ++t)
                        ptx::Wgmma<BN>::ss(acc, ad0 + (uint64_t)(((t / KH) * PITCH + t % KH) * 128 / 16 + 2 * ks),
                                           bd0 + (uint64_t)(t * (BN * 128) / 16 + 2 * ks), (t | ks) != 0 ? 1u : 0u);
            } else if (SPLIT8 && cc == g.split_chunk) {
                // the second source's 8 channels, tap by tap, after every chunk of the first
                const uint64_t ad0 = ptx::make_kmajor_desc(a0 + (uint32_t)(8 * wg * PITCH * 32), 32, PITCH * 32);
                const uint64_t bd0 = ptx::make_kmajor_desc(a0 + (uint32_t)A_BYTES, 32);
#pragma unroll
                for (int t = 0; t < KH * KH; ++t)
                    ptx::Wgmma<BN>::ss(acc, ad0 + (uint64_t)(((t / KH) * PITCH + t % KH) * 32 / 16),
                                       bd0 + (uint64_t)(t * T_B_TILE / 16), 1u);
            } else {
                const int c8 = WIDE ? g.split_chunk : cc;      // the chunk's index in 8-channel units
                const uint32_t b0 = g.resident ? sB_u + (uint32_t)(c8 * KH * KH * B_TILE) : a0 + (uint32_t)A_BYTES;
                const uint64_t ad0 = ptx::make_kmajor_desc(a0 + (uint32_t)(8 * wg * PITCH * ROWB), ROWB, PITCH * ROWB);
                const uint64_t bd0 = ptx::make_kmajor_desc(b0, ROWB);
                // the chunk's taps, then 8-channel K steps, into one accumulator; descriptor start addresses count
                // 16-byte units
#pragma unroll
                for (int t = 0; t < KH * KH; ++t) {
                    const uint64_t ad = ad0 + (uint64_t)(((t / KH) * PITCH + t % KH) * ROWB / 16);
                    const uint64_t bd = bd0 + (uint64_t)(t * B_TILE / 16);
#pragma unroll
                    for (int ks = 0; ks < KC / 8; ++ks)
                        ptx::Wgmma<BN>::ss(acc, ad + (uint64_t)(2 * ks), bd + (uint64_t)(2 * ks), (c8 | t | ks) != 0 ? 1u : 0u);
                }
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
            // into staging buffer it & 1 (head_pitch), once the store side has copied out what it held two tiles ago
            const int hc = g.head_cout, pp = head_pitch(hc);
            const uint32_t sv = ptx::smem_u32(sHS) + (uint32_t)((it & 1) * hs_bytes);
            const uint32_t sm = sv + 4u * (uint32_t)head_stage_floats(hc);
            ptx::mbar_wait(&hfree[it & 1], ((uint32_t)(it >> 1) & 1u) ^ 1u);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint32_t p = (uint32_t)((ty + h) * COL_TW + g8);
                float best = -INFINITY;
                int best_c = 0;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int co = 8 * j + 2 * t4;
                    float val[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        val[e] = hacc[4 * j + 2 * h + e] + s_head[co + e];
                        if (co + e < g.head_seg && val[e] > best) {
                            best = val[e];
                            best_c = co + e;
                        }
                    }
                    // channel co + 1 == hc (odd hc) lands in the pixel's padding
                    if (co < hc) {
                        if (g.head_nhwc) {
                            ptx::sts64(sv + 4u * (p * pp + co), make_float2(val[0], val[1]));
                        } else {
                            ptx::sts32(sv + 4u * (co * HEAD_CPITCH + p), val[0]);
                            if (co + 1 < hc) ptx::sts32(sv + 4u * ((co + 1) * HEAD_CPITCH + p), val[1]);
                        }
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
                if (t4 == 0) ptx::sts8(sm + p, (uint32_t)best_c);
            }
            ptx::mbar_arrive(&hstaged[it & 1]);
        }
    }
}

struct ColPlan {
    CUtensorMap tmA, tmA2, tmB, tmBw;
    ColGeom g;
    int kc, ksize, head, bn, wide, split8;
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

template <int KC, bool HEAD, int KH, int BN, bool WIDE = false, bool SPLIT8 = false>
int col_launch(const ColPlan &p, cudaStream_t s)
{
    // the instantiation must be the plan's: weight boxes, barrier byte counts and stores are sized by BN
    if (p.bn != BN || p.kc != KC || p.ksize != KH || p.head != (HEAD ? 1 : 0) || p.wide != (WIDE ? 1 : 0) ||
        p.split8 != (SPLIT8 ? 1 : 0)) {
        set_error("conv(col): no kernel instantiation for this plan (Cout %d, chunk %d, ksize %d)", p.bn, p.kc, p.ksize);
        return PVNET_E_STATE;
    }
    auto fn = k_conv_col<KC, HEAD, KH, BN, WIDE, SPLIT8>;
    const cudaError_t attr_err = ensure_max_smem((const void *)fn, (int)SMEM_LIMIT);
    PV_CUDA(attr_err);
    const HeadDesc &h = p.hd;
    fn<<<p.grid, COL_THREADS, p.smem, s>>>(p.tmA, p.tmA2, p.tmB, p.tmBw, p.g, p.bias, p.res, p.out, p.head ? h.w : nullptr,
                                           p.head ? h.bias : nullptr, p.head ? h.out_nchw : nullptr,
                                           p.head ? h.mask : nullptr);
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

namespace {

int plan_at(const ConvDesc &d, const HeadDesc *head, bool split8, void *storage)
{
    ColPlan *p = new (storage) ColPlan();
    PV_CHECK_ARG(conv_col_eligible(d), "conv(col): layer not eligible for the column kernel");
    PV_CHECK_ARG(d.in && d.w && d.bias && (d.out || head), "conv(col): null pointer");
    PV_CHECK_ARG(d.in_cs % 4 == 0 && d.in_co % 4 == 0 && d.out_cs % 4 == 0 && d.out_co % 4 == 0,
                 "conv(col): channel strides/offsets must be multiples of 4 floats");
    PV_CHECK_ARG(!d.res || (d.res_cs % 4 == 0 && d.res_co % 4 == 0), "conv(col): residual stride/offset alignment");
    PV_CHECK_ARG(!head || (d.Cout == 32 && col_kc(d.Cin + d.Cin2) == 8 && head->cout >= 1 && head->cout <= 32 && head->w && head->bias &&
                           head->out_nchw && (!head->mask || head->mask_esz == 1 || head->mask_esz == 8)),
                 "conv(col): bad fused-head description");
    // split chunks: the first source in 32-channel chunks, the 8-channel second source as one more chunk, weights
    // streamed with each stage (their [Cout][taps][cin_pad] packing is the single-chunk-size one: cin_pad rounds
    // Cin + 8 up to 32, the second source's weights start at column Cin of each tap)
    PV_CHECK_ARG(!split8 || (!head && d.in2 && d.Cin % 32 == 0 && d.Cin2 == 8 && d.Cout == 64 && d.ksize == 3),
                 "conv(col): split chunks need a 32-channel-multiple first source, an 8-channel second, Cout 64, 3x3");
    const int kc = split8 ? 32 : col_kc(d.Cin + d.Cin2);
    ColGeom &g = p->g;
    g.pad_l = g.pad_t = d.ksize == 4 ? 2 : 1;
    g.Ho = d.H;
    g.Wo = d.W;
    g.tiles_x = (d.W + COL_TW - 1) / COL_TW;
    g.tiles_y = (d.H + COL_TH - 1) / COL_TH;
    g.total_tiles = g.tiles_x * g.tiles_y * d.b;
    g.cin_chunks = split8 ? d.Cin / kc + 1 : (d.Cin + d.Cin2) / kc;
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
    // Resident weights whenever at least 2 A stages (one channel chunk with all its taps each) still
    // fit next to them; otherwise the KH*KW weight tiles of a chunk travel with its A box.
    const bool hd = head != nullptr;
    // the head's two output staging buffers and their four barriers
    const size_t hs = hd ? 2 * (size_t)head_stage_bytes(head->cout) + 4 * 8 : 0;
    // convraw.0's 32 + 8 channel form loads its first source as one box of 128-byte rows (WIDE in k_conv_col);
    // its stages then hold that box instead of an 8-channel one
    bool wide = hd && d.in2 && d.Cin == 32 && d.Cin2 == 8 && kc == 8 && d.ksize == 3;
    const size_t wx = col_smem(32, 3, 0, 0, 1, false, false) - col_smem(8, 3, 0, 0, 1, false, false);
    int stages = 8;
    bool resident = true;
    while (stages > 2 && col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, true) + hs + (wide ? stages * wx : 0) > SMEM_LIMIT)
        --stages;
    if (split8 || col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, true) + hs + (wide ? stages * wx : 0) > SMEM_LIMIT) {
        wide = false;
        resident = false;
        stages = 8;
        while (stages > 2 && col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, false) + hs > SMEM_LIMIT) --stages;
    }
    g.stages = stages;
    g.resident = resident ? 1 : 0;
    p->smem = col_smem(kc, d.ksize, g.cin_chunks, d.Cout, stages, hd, resident) + hs + (wide ? stages * wx : 0);
    p->wide = wide ? 1 : 0;
    p->split8 = split8 ? 1 : 0;
    PV_CHECK_ARG(p->smem <= SMEM_LIMIT, "conv(col): layer does not fit in shared memory");
    p->kc = kc;
    p->ksize = d.ksize;
    p->bn = d.Cout;
    p->head = hd ? 1 : 0;
    if (head) p->hd = *head;
    {
        const float *base = d.in + d.in_co;
        cuuint64_t dims[4] = {(cuuint64_t)d.Cin, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.b};
        cuuint64_t strides[3] = {(cuuint64_t)d.in_cs * 4, (cuuint64_t)d.W * d.in_cs * 4,
                                 (cuuint64_t)d.H * d.W * d.in_cs * 4};
        const int akc = wide ? 32 : kc;
        cuuint32_t box[4] = {(cuuint32_t)akc, (cuuint32_t)(COL_TW + d.ksize - 1), (cuuint32_t)(COL_TH + d.ksize - 1), 1};
        int rc = tma_encode(&p->tmA, base, 4, dims, strides, box, akc * 4);
        if (rc) return rc;
        p->tmA2 = p->tmA;
    }
    if (d.in2) {
        PV_CHECK_ARG(d.in2_cs % 4 == 0 && d.in2_co % 4 == 0 && d.Cin2 > 0, "conv(col): second source stride/offset alignment");
        cuuint64_t dims[4] = {(cuuint64_t)d.Cin2, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.b};
        cuuint64_t strides[3] = {(cuuint64_t)d.in2_cs * 4, (cuuint64_t)d.W * d.in2_cs * 4,
                                 (cuuint64_t)d.H * d.W * d.in2_cs * 4};
        const int kc2 = split8 ? 8 : kc;
        cuuint32_t box[4] = {(cuuint32_t)kc2, (cuuint32_t)(COL_TW + d.ksize - 1), (cuuint32_t)(COL_TH + d.ksize - 1), 1};
        int rc = tma_encode(&p->tmA2, d.in2 + d.in2_co, 4, dims, strides, box, kc2 * 4);
        if (rc) return rc;
    }
    {
        cuuint64_t dims[2] = {(cuuint64_t)d.ksize * d.ksize * g.cin_pad, (cuuint64_t)d.Cout};
        cuuint64_t strides[1] = {(cuuint64_t)d.ksize * d.ksize * g.cin_pad * 4};
        cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)d.Cout};
        int rc = tma_encode(&p->tmB, d.w, 2, dims, strides, box, kc * 4);
        if (rc) return rc;
        p->tmBw = p->tmB;
        if (wide) {
            box[0] = 32;
            if ((rc = tma_encode(&p->tmBw, d.w, 2, dims, strides, box, 128))) return rc;
        }
        if (split8) {
            box[0] = 8;
            if ((rc = tma_encode(&p->tmBw, d.w, 2, dims, strides, box, 32))) return rc;
        }
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

}  // namespace

int conv_col_plan_at(const ConvDesc &d, const HeadDesc *head, void *storage) { return plan_at(d, head, false, storage); }

int conv_col_plan_split_at(const ConvDesc &d, void *storage) { return plan_at(d, nullptr, true, storage); }

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
    if (p.wide) return col_launch<8, true, 3, 32, true>(p, s);
    if (p.split8) return col_launch<32, false, 3, 64, false, true>(p, s);
    if (p.head) return col_launch<8, true, 3, 32>(p, s);
    const bool n64 = p.bn == 64;
    if (p.ksize == 4) return n64 ? col_launch<16, false, 4, 64>(p, s) : col_launch<16, false, 4, 32>(p, s);
    if (p.kc == 32) return n64 ? col_launch<32, false, 3, 64>(p, s) : col_launch<32, false, 3, 32>(p, s);
    return n64 ? col_launch<8, false, 3, 64>(p, s) : col_launch<8, false, 3, 32>(p, s);
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
