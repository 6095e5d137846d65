// conv_tc.cu -- implicit-GEMM 2-D convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// One CTA computes 128-pixel x BN-channel output tiles of an NHWC convolution
// (lib/networks/resnet.py:28-35 `conv3x3`, the 1x1 downsample convs, and the decoder convs
// of lib/networks/model_repository.py:22-58), with BatchNorm folded into weights/bias and
// the activation / residual add fused into the epilogue:
//
//   M = 128 output pixels (a TH x TW = 8 x 16 patch of one image)
//   N = BN output channels (32, 64, 128 or 256: conv_plan picks the one its model says finishes first)
//   K = taps x Cin, walked tap by tap in chunks of 32 input channels
//
//   warp 8       TMA producer: per K-block one 4-D box {32 ch, TW, TH, 1 image} of the NHWC input,
//                shifted by the tap's (dy,dx)*dilation -- out-of-bounds coordinates are zero-filled
//                by TMA, which IS the conv padding -- plus one 2-D box {32, BN} of the packed weights
//                [Cout][tap][Cin]; 128-byte-swizzled K-major tiles in a ring of mbarrier-guarded stages.
//                With a residual it also loads the residual's {32 ch, TW, TH, 1} boxes into the epilogue's
//                staging buffers, as the consumers hand them back.
//   warps 0-7    two consumer warpgroups, 64 pixel rows each: wgmma.m64nBNk8 (tf32 in, fp32
//                accumulate in registers) straight from the stage, then the epilogue: +bias (+residual)
//                -> ReLU / LeakyReLU(0.1) -> optional round-to-tf32, written 32 channels at a time into
//                one of two swizzled [128 pixels][32 channels] staging buffers and stored from there by
//                TMA into the channel slice of a (possibly wider) NHWC destination buffer, so torch.cat
//                never happens. TMA clips partial tiles. The consumers do not wait for a store to reach
//                memory: the last slabs of a tile drain under the next tile's MMAs.
//
// CTAs are persistent over (M tile, N tile) items (static round-robin; the ring runs on across items,
// so the producer fetches the next item's operands during the current epilogue).
//
// Stride-2 convolutions read the input through four "parity plane" tensor maps (even/odd
// rows x even/odd columns); each tap then is a stride-1 box in one plane.
#include "conv_tc.cuh"
#include "ptx.cuh"

#include <cstdlib>
#include <mutex>
#include <new>

namespace pvnet {

struct ConvGeom {
    int Ho, Wo;
    int tiles_x, tiles_y, total_m_tiles;
    int TH, TW;
    int taps, cin_chunks, cin_pad;
    int Cout, BN;
    int out_cs, out_co;
    int res_cs, res_co;
    int act;        // 0 none, 1 ReLU, 2 LeakyReLU(0.1)
    int round_out;  // round stored values to tf32 (they feed another tensor-core conv)
    signed char tap_map[9];
    short tap_ox[9], tap_oy[9];
    int n_items;    // M tiles x N tiles, N tile fastest
    int stages;     // depth of the TMA ring
};

struct AMaps {
    CUtensorMap m[4];
};

constexpr int CONV_THREADS = 288;      // two consumer warpgroups + one producer warp
constexpr int CONV_KC = 32;            // input channels per K-block: one 128-byte swizzled row per pixel
constexpr int CONV_A_BYTES = 128 * CONV_KC * 4;
constexpr int CONV_SLAB = 32;          // output channels per epilogue slab: one 128-byte swizzled row per pixel
constexpr int CONV_SLAB_BYTES = 128 * CONV_SLAB * 4;
constexpr int CONV_EPI_BAR = 1;        // named barrier of the 256 consumer threads

template <int BN>
__global__ void __launch_bounds__(CONV_THREADS, 1)
    k_conv_tap(const __grid_constant__ AMaps amaps, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmRes,
               const __grid_constant__ ConvGeom g, const float *__restrict__ bias, const int has_res)
{
    constexpr int B_BYTES = BN * CONV_KC * 4;
    constexpr int STAGE_BYTES = CONV_A_BYTES + B_BYTES;
    constexpr int SLABS = BN / CONV_SLAB;
    const int STAGES = g.stages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    // two slab staging buffers behind the ring (a stage is a multiple of 1024 bytes, so they are 1024-byte aligned,
    // what the 128-byte swizzle needs), then the barriers
    uint8_t *slab = smem + (size_t)STAGES * STAGE_BYTES;
    uint64_t *full = reinterpret_cast<uint64_t *>(slab + 2 * CONV_SLAB_BYTES);
    uint64_t *empty = full + STAGES;
    uint64_t *res_full = empty + STAGES;   // [2] the residual slab has landed in staging buffer i
    uint64_t *res_free = res_full + 2;     // [2] the last store out of staging buffer i has finished reading it

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_img = g.tiles_x * g.tiles_y;
    const int n_tiles_n = g.Cout / BN;
    const int nkb = g.taps * g.cin_chunks;
    const int unit = (int)blockIdx.x, nunits = (int)gridDim.x;
    auto item_tile = [&](int item, int &m_tile, int &n0) {
        m_tile = item / n_tiles_n;
        n0 = (item - m_tile * n_tiles_n) * BN;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], 8);    // one arrive per consumer warp
        }
        for (int i = 0; i < 2; ++i) {
            ptx::mbar_init(&res_full[i], 1);
            ptx::mbar_init(&res_free[i], 1);
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // Residual slabs ride into the staging buffers on the same thread, between operand loads: slab q of
            // this CTA's slab sequence goes to buffer q & 1 once the consumers handed that buffer back (res_free),
            // never blocking the ring. The buffers are free when an item's epilogue ends, so an item's first two
            // residual slabs are fetched under its K loop and the later ones as its slabs are stored.
            int r_item = has_res ? unit : g.n_items, r_slab = 0;
            uint32_t rq = 0;
            auto poll_res = [&]() {
                if (r_item >= g.n_items) return;
                const uint32_t b = rq & 1u;
                if (!ptx::mbar_test_wait(&res_free[b], ((rq >> 1) & 1u) ^ 1u)) return;
                int m_tile, n0;
                item_tile(r_item, m_tile, n0);
                const int img = m_tile / tiles_per_img;
                const int trem = m_tile - img * tiles_per_img;
                const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
                ptx::mbar_arrive_expect_tx(&res_full[b], (uint32_t)CONV_SLAB_BYTES);
                ptx::tma_load_4d(slab + b * CONV_SLAB_BYTES, &tmRes, &res_full[b], n0 + r_slab * CONV_SLAB, txi * g.TW,
                                 tyi * g.TH, img);
                ++rq;
                if (++r_slab == SLABS) {
                    r_slab = 0;
                    r_item += nunits;
                }
            };
            int s = 0;
            uint32_t ph = 0;
            for (int item = unit; item < g.n_items; item += nunits) {
                int m_tile, n0;
                item_tile(item, m_tile, n0);
                const int img = m_tile / tiles_per_img;
                const int trem = m_tile - img * tiles_per_img;
                const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
                const int y0 = tyi * g.TH, x0 = txi * g.TW;
                for (int tap = 0; tap < g.taps; ++tap)
                    for (int cc = 0; cc < g.cin_chunks; ++cc) {
                        poll_res();
                        // with residual slabs pending, look at the ring without being parked in try_wait
                        while (!(has_res ? ptx::mbar_test_wait(&empty[s], ph ^ 1u) : ptx::mbar_try_wait(&empty[s], ph ^ 1u)))
                            poll_res();
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)STAGE_BYTES);
                        uint8_t *sa = smem + (size_t)s * STAGE_BYTES;
                        ptx::tma_load_4d(sa, &amaps.m[g.tap_map[tap]], &full[s], cc * CONV_KC, x0 + g.tap_ox[tap],
                                         y0 + g.tap_oy[tap], img);
                        ptx::tma_load_2d(sa + CONV_A_BYTES, &tmB, &full[s], tap * g.cin_pad + cc * CONV_KC, n0);
                        if (++s == STAGES) {
                            s = 0;
                            ph ^= 1u;
                        }
                    }
            }
            while (r_item < g.n_items) poll_res();
        }
    } else {
        // consumer warpgroup wg: pixel rows [64 wg, 64 wg + 64) of the tile
        const int wg = warp >> 2, wq = warp & 3;
        const int g8 = lane >> 2, t4 = lane & 3;
        const uint32_t smem_u = ptx::smem_u32(smem);
        int s = 0;
        uint32_t ph = 0, sq = 0;            // sq: slabs this CTA has stored so far
        for (int item = unit; item < g.n_items; item += nunits) {
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
            int prev = -1;
            for (int kb = 0; kb < nkb; ++kb) {
                ptx::mbar_wait(&full[s], ph);
                const uint32_t sa = smem_u + (uint32_t)s * (uint32_t)STAGE_BYTES;
                const uint64_t adesc = ptx::make_kmajor_desc(sa + (uint32_t)(wg * 64 * 128), 128);
                const uint64_t bdesc = ptx::make_kmajor_desc(sa + (uint32_t)CONV_A_BYTES, 128);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < CONV_KC / 8; ++k)   // 8 tf32 = 32 bytes along K: +2 in 16-byte units
                    ptx::Wgmma<BN>::ss(acc, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
                ptx::wgmma_commit();
                // the previous K-block's MMAs have finished reading their stage: hand it back
                ptx::wgmma_wait<1>();
                ptx::fence_regs(acc);
                if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
                prev = s;
                if (++s == STAGES) {
                    s = 0;
                    ph ^= 1u;
                }
            }
            ptx::wgmma_wait<0>();
            ptx::fence_regs(acc);
            if (lane == 0) ptx::mbar_arrive(&empty[prev]);

            // Epilogue, one 32-channel slab at a time through two staging buffers [128 pixels][32 channels], laid
            // out as TMA lays out the A tile (pixel m = row, 128-byte swizzle: 16-byte chunk c of row m sits at chunk
            // c ^ (m & 7)). A thread owns pixels m = 64 wg + 16 wq + g8 (+ 8) and, per 8-channel block jj of the slab,
            // channels 8 jj + 2 t4 (+ 1): the 8 bytes at chunk (2 jj + (t4 >> 1)) ^ g8, offset 8 (t4 & 1). Of one
            // warp's st.shared.v2 the eight rows g8 turn a row's two chunks into all eight chunks of the 128-byte
            // bank line, each hit by exactly two rows -- the two wavefronts that 256 bytes need anyway; unswizzled,
            // the eight rows would pile onto the same two chunks. Thread 0 then stores the slab with one TMA box
            // {32, TW, TH, 1}; TMA clips what lies outside the tensor (partial tiles), and the consumers go on
            // without waiting for the store to reach memory.
            //
            // Buffer q & 1 is rewritten for slab q only after the store of slab q - 2 has finished reading it: thread 0
            // learns that from cp.async.bulk.wait_group.read and publishes it -- with a residual by arriving on
            // res_free, on which the producer waits before it loads the residual slab there (res_full then releases
            // the consumers); without one by the named barrier ahead of the writes. A residual slab is always loaded
            // before the same slab is stored and no other slab touches those addresses, so each address sees its
            // read before its write, as with the direct epilogue, when `res` and `out` are the same slice. Pixels
            // outside the tensor read zeros and are clipped on the store.
            int m_tile, n0;
            item_tile(item, m_tile, n0);
            const int img = m_tile / tiles_per_img;
            const int trem = m_tile - img * tiles_per_img;
            const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
            const uint32_t row_off = (uint32_t)((wg * 64 + wq * 16 + g8) * 128 + (t4 & 1) * 8);
            const uint32_t swz = (uint32_t)(((t4 >> 1) ^ g8) << 4);
            const uint32_t slab_u = ptx::smem_u32(slab);
#pragma unroll
            for (int j = 0; j < SLABS; ++j, ++sq) {
                const uint32_t b = sq & 1u;
                const uint32_t base = slab_u + b * (uint32_t)CONV_SLAB_BYTES + row_off;
                float2 bv[4];
#pragma unroll
                for (int jj = 0; jj < 4; ++jj)
                    bv[jj] = __ldg(reinterpret_cast<const float2 *>(bias + n0 + CONV_SLAB * j + 8 * jj + 2 * t4));
                if (has_res) ptx::mbar_wait(&res_full[b], (sq >> 1) & 1u);
                else ptx::named_bar_sync(CONV_EPI_BAR, 256);
#pragma unroll
                for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const uint32_t addr = base + (uint32_t)(h * 8 * 128) + (swz ^ (uint32_t)(32 * jj));
                        const int a = 4 * (4 * j + jj) + 2 * h;
                        float2 v = make_float2(acc[a] + bv[jj].x, acc[a + 1] + bv[jj].y);
                        if (has_res) {
                            const float2 r = ptx::lds64(addr);
                            v.x += r.x;
                            v.y += r.y;
                        }
                        v.x = epi_act(v.x, g.act, g.round_out);
                        v.y = epi_act(v.y, g.act, g.round_out);
                        ptx::sts64(addr, v);
                    }
                ptx::fence_proxy_async();
                ptx::named_bar_sync(CONV_EPI_BAR, 256);
                if (threadIdx.x == 0) {
                    ptx::tma_store_4d(&tmOut, slab + b * CONV_SLAB_BYTES, n0 + CONV_SLAB * j, txi * g.TW, tyi * g.TH, img);
                    ptx::tma_store_commit();
                    // all but this store have finished reading (the item's last slab: this one too, so that both
                    // buffers are free for the next item's first slabs while its K loop runs)
                    if (j == SLABS - 1) ptx::tma_store_wait_read();
                    else ptx::tma_store_wait_read1();
                    if (has_res) {
                        if (j > 0) ptx::mbar_arrive(&res_free[b ^ 1u]);
                        if (j == SLABS - 1) ptx::mbar_arrive(&res_free[b]);
                    }
                }
                __syncwarp();       // warp 0 is whole again for the aligned barriers and MMAs that follow
            }
        }
        if (threadIdx.x == 0) ptx::tma_store_wait_all();   // the stores have reached memory before the kernel ends
    }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    });
    return fn;
}

int tma_encode(CUtensorMap *m, const void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides_bytes,
               const cuuint32_t *box, int swizzle_bytes)
{
    EncodeTiledFn fn = encode_fn();
    if (!fn) {
        set_error("cuTensorMapEncodeTiled entry point unavailable");
        return PVNET_E_CUDA;
    }
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                        : CU_TENSOR_MAP_SWIZZLE_32B;
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), dims,
                    strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_ERROR_INVALID_CONTEXT || r == CUDA_ERROR_NOT_INITIALIZED) {
        // a thread that has only selected its device through the runtime (nn.DataParallel's per-GPU workers) may
        // have no driver context bound yet: cudaFree(0) binds the device's primary context to this thread
        cudaFree(nullptr);
        r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), dims, strides_bytes, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d, dims %llu %llu, box %u %u, swizzle %d)",
                  (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1],
                  swizzle_bytes);
        return PVNET_E_CUDA;
    }
    return PVNET_OK;
}

// A fully described convolution launch (tensor maps are encoded once and can be reused as
// long as the pointers and shapes stay the same).
struct ConvPlan {
    AMaps amaps;
    CUtensorMap tmB;
    CUtensorMap tmOut, tmRes;   // destination and residual channel slices, boxes {32, TW, TH, 1}
    ConvGeom g;
    dim3 grid;
    size_t smem;
    const float *bias;
    int has_res;
};

int conv_plan(const ConvDesc &d, ConvPlan *p)
{
    PV_CHECK_ARG(d.in && d.w && d.bias && d.out, "conv: null pointer");
    PV_CHECK_ARG(!d.in2, "conv: a second input source is only supported by the column kernel");
    PV_CHECK_ARG(d.ksize == 1 || d.ksize == 3, "conv: kernel size %d unsupported", d.ksize);
    PV_CHECK_ARG(d.stride == 1 || d.stride == 2, "conv: stride %d unsupported", d.stride);
    PV_CHECK_ARG(d.stride == 1 || (d.dilation == 1 && d.H % 2 == 0 && d.W % 2 == 0),
                 "conv: stride 2 needs dilation 1 and even H,W");
    PV_CHECK_ARG(d.Cout % 32 == 0, "conv: Cout %d must be a multiple of 32", d.Cout);
    PV_CHECK_ARG(d.in_cs % 4 == 0 && d.in_co % 4 == 0 && d.out_cs % 4 == 0 && d.out_co % 4 == 0,
                 "conv: channel strides/offsets must be multiples of 4 floats");
    PV_CHECK_ARG(!d.res || (d.res_cs % 4 == 0 && d.res_co % 4 == 0), "conv: residual stride/offset alignment");
    PV_CHECK_ARG(((uintptr_t)d.in % 16 == 0) && ((uintptr_t)d.w % 16 == 0) && ((uintptr_t)d.out % 16 == 0) &&
                     ((uintptr_t)d.bias % 16 == 0),
                 "conv: pointers must be 16-byte aligned");
    PV_CHECK_ARG(d.Cin % 4 == 0, "conv: Cin %d must be a multiple of 4", d.Cin);
    const int kc = CONV_KC;             // ragged last channel chunk: TMA zero-fills, weights are zero-padded
    ConvGeom &g = p->g;
    g.Ho = d.H / d.stride;
    g.Wo = d.W / d.stride;
    g.TH = 8;
    g.TW = 16;
    g.tiles_x = (g.Wo + g.TW - 1) / g.TW;
    g.tiles_y = (g.Ho + g.TH - 1) / g.TH;
    g.total_m_tiles = g.tiles_x * g.tiles_y * d.b;
    g.taps = d.ksize * d.ksize;
    g.cin_chunks = (d.Cin + kc - 1) / kc;
    g.cin_pad = g.cin_chunks * kc;
    g.Cout = d.Cout;
    // N tile: the divisor of Cout among 256/128/64/32 that the model says finishes first. The kernel is bound
    // by operand delivery into shared memory -- every K-block brings a 16 KB A box and a BN x 128 B weight
    // tile, whatever BN is -- and the persistent CTAs (one per SM) take the items round-robin, so a layer
    // costs about rounds x per-item bytes, rounds = ceil(items / SMs). Ties go to the wider tile. Every BN
    // sums each output element over the same K sequence, so the choice does not change the results.
    {
        const long long sms = sm_count() > 0 ? sm_count() : 1;
        long long best = -1;
        for (int bn = 256; bn >= 32; bn >>= 1) {
            if (d.Cout % bn) continue;
            const long long items = (long long)g.total_m_tiles * (d.Cout / bn);
            const long long cost = (items + sms - 1) / sms * (CONV_A_BYTES + bn * kc * 4);
            if (best < 0 || cost < best) {
                best = cost;
                g.BN = bn;
            }
        }
    }
    g.out_cs = d.out_cs;
    g.out_co = d.out_co;
    g.res_cs = d.res_cs;
    g.res_co = d.res_co;
    g.act = d.act;
    g.round_out = d.round_out;
    const int pad = d.dilation * (d.ksize - 1) / 2;
    for (int t = 0; t < g.taps; ++t) {
        const int kh = t / d.ksize, kw = t - kh * d.ksize;
        if (d.stride == 1) {
            g.tap_map[t] = 0;
            g.tap_ox[t] = (short)(kw * d.dilation - pad);
            g.tap_oy[t] = (short)(kh * d.dilation - pad);
        } else {
            // input coordinate 2*o + k - pad: parity plane (k-pad)&1, plane coordinate o + floor((k-pad)/2)
            const int dy = kh - pad, dx = kw - pad;
            const int py = dy & 1, px = dx & 1;
            g.tap_map[t] = (signed char)(py * 2 + px);
            g.tap_oy[t] = (short)((dy - py) / 2);
            g.tap_ox[t] = (short)((dx - px) / 2);
        }
    }
    const int swz = kc * 4;
    // A: NHWC input (or its four parity planes for stride 2)
    const int nplanes = d.stride == 2 ? 4 : 1;
    for (int pl = 0; pl < nplanes; ++pl) {
        const int py = pl >> 1, px = pl & 1;
        const float *base = d.in + d.in_co + ((size_t)py * d.W + px) * d.in_cs;
        cuuint64_t dims[4] = {(cuuint64_t)d.Cin, (cuuint64_t)(d.W / d.stride), (cuuint64_t)(d.H / d.stride),
                              (cuuint64_t)d.b};
        cuuint64_t strides[3] = {(cuuint64_t)d.stride * d.in_cs * 4, (cuuint64_t)d.stride * d.W * d.in_cs * 4,
                                 (cuuint64_t)d.H * d.W * d.in_cs * 4};
        cuuint32_t box[4] = {(cuuint32_t)kc, (cuuint32_t)g.TW, (cuuint32_t)g.TH, 1};
        int rc = tma_encode(&p->amaps.m[pl], base, 4, dims, strides, box, swz);
        if (rc) return rc;
    }
    for (int pl = nplanes; pl < 4; ++pl) p->amaps.m[pl] = p->amaps.m[0];
    // B: packed weights [Cout][taps*cin_pad]
    {
        cuuint64_t dims[2] = {(cuuint64_t)g.taps * g.cin_pad, (cuuint64_t)d.Cout};
        cuuint64_t strides[1] = {(cuuint64_t)g.taps * g.cin_pad * 4};
        cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)g.BN};
        int rc = tma_encode(&p->tmB, d.w, 2, dims, strides, box, swz);
        if (rc) return rc;
    }
    // destination and residual: the channel slice [co, co + Cout) of an NHWC buffer, stored / loaded one
    // {32 channels, TW, TH, 1 image} box per slab. The argument checks above (16-byte aligned pointers, strides and
    // offsets multiples of 4 floats) are what these maps need.
    {
        cuuint64_t dims[4] = {(cuuint64_t)d.Cout, (cuuint64_t)g.Wo, (cuuint64_t)g.Ho, (cuuint64_t)d.b};
        cuuint32_t box[4] = {(cuuint32_t)CONV_SLAB, (cuuint32_t)g.TW, (cuuint32_t)g.TH, 1};
        cuuint64_t ostr[3] = {(cuuint64_t)d.out_cs * 4, (cuuint64_t)g.Wo * d.out_cs * 4,
                              (cuuint64_t)g.Ho * g.Wo * d.out_cs * 4};
        int rc = tma_encode(&p->tmOut, d.out + d.out_co, 4, dims, ostr, box, CONV_SLAB * 4);
        if (rc) return rc;
        p->tmRes = p->tmOut;
        if (d.res) {
            PV_CHECK_ARG((uintptr_t)d.res % 16 == 0, "conv: pointers must be 16-byte aligned");
            cuuint64_t rstr[3] = {(cuuint64_t)d.res_cs * 4, (cuuint64_t)g.Wo * d.res_cs * 4,
                                  (cuuint64_t)g.Ho * g.Wo * d.res_cs * 4};
            rc = tma_encode(&p->tmRes, d.res + d.res_co, 4, dims, rstr, box, CONV_SLAB * 4);
            if (rc) return rc;
        }
    }
    // ring: as many stages as fit (at most 8) in the 227 KB a block may use, beside the epilogue's two 16 KB slab
    // buffers: 4 stages at BN 256 and 8 at BN 64 and 32, as without the buffers; BN 128 has 6 where 7 would fit
    const size_t stage_b = (size_t)CONV_A_BYTES + (size_t)g.BN * kc * 4;
    int st = (int)((227 * 1024 - 1024 - 256 - 2 * CONV_SLAB_BYTES) / stage_b);
    if (st > 8) st = 8;
    g.stages = st;
    p->smem = 1024 + (size_t)st * stage_b + 2 * CONV_SLAB_BYTES + 256;
    // items: (M tile, N tile); one persistent CTA per SM, or one per item when there are fewer
    g.n_items = g.total_m_tiles * (d.Cout / g.BN);
    long long grid = (long long)sm_count();
    if (grid > g.n_items) grid = g.n_items;
    p->grid = dim3((unsigned)grid);
    p->bias = d.bias;
    p->has_res = d.res != nullptr;
    return PVNET_OK;
}

template <int BN>
int conv_launch_t(const ConvPlan &p, cudaStream_t s)
{
    const cudaError_t attr_err = ensure_max_smem((const void *)k_conv_tap<BN>, 227 * 1024);
    PV_CUDA(attr_err);
    k_conv_tap<BN><<<p.grid, CONV_THREADS, p.smem, s>>>(p.amaps, p.tmB, p.tmOut, p.tmRes, p.g, p.bias, p.has_res);
    PV_LAUNCHED("k_conv_tap");
    return PVNET_OK;
}

int conv_launch(const ConvPlan &p, cudaStream_t s)
{
    if (p.g.BN == 256) return conv_launch_t<256>(p, s);
    if (p.g.BN == 128) return conv_launch_t<128>(p, s);
    if (p.g.BN == 64) return conv_launch_t<64>(p, s);
    return conv_launch_t<32>(p, s);
}

size_t conv_plan_size() { return sizeof(ConvPlan); }
int conv_plan_at(const ConvDesc &d, void *storage) { return conv_plan(d, new (storage) ConvPlan()); }
int conv_launch_at(const void *storage, cudaStream_t s) { return conv_launch(*static_cast<const ConvPlan *>(storage), s); }

}  // namespace pvnet

extern "C" {

int pvnet_conv2d_nhwc(const float *in, int in_cs, int in_co, int Cin, const float *w_packed, const float *bias,
                      const float *res, int res_cs, int res_co, float *out, int out_cs, int out_co, int Cout, int b,
                      int H, int W, int ksize, int stride, int dilation, int act, int round_out,
                      pvnet_stream_t stream)
{
    pvnet::ConvDesc d{in, in_cs, in_co, Cin, w_packed, bias, res, res_cs, res_co, out, out_cs, out_co, Cout,
                      b, H, W, ksize, stride, dilation, act, round_out};
    const bool col = pvnet::g_conv_mode == 2 || (pvnet::g_conv_mode == 0 && pvnet::conv_col_eligible(d));
    if (col) {
        alignas(64) unsigned char storage[2048];
        static_assert(sizeof(storage) >= 1024, "plan storage");
        if (pvnet::conv_col_plan_size() > sizeof(storage)) {
            pvnet::set_error("column plan larger than its stack storage");
            return PVNET_E_STATE;
        }
        int rc = pvnet::conv_col_plan_at(d, nullptr, storage);
        if (rc) return rc;
        return pvnet::conv_col_launch_at(storage, (cudaStream_t)stream);
    }
    pvnet::ConvPlan plan;
    int rc = pvnet::conv_plan(d, &plan);
    if (rc) return rc;
    return pvnet::conv_launch(plan, (cudaStream_t)stream);
}

}  // extern "C"
