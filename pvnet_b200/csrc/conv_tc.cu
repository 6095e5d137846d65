// conv_tc.cu -- implicit-GEMM 2-D convolution on the Hopper tensor cores (wgmma, sm_90a).
//
// One CTA computes 128-pixel x BN-channel output tiles of an NHWC convolution
// (lib/networks/resnet.py:28-35 `conv3x3`, the 1x1 downsample convs, and the decoder convs
// of lib/networks/model_repository.py:22-58), with BatchNorm folded into weights/bias and
// the activation / residual add fused into the epilogue:
//
//   M = 128 output pixels (a TH x TW = 8 x 16 patch of one image)
//   N = BN output channels (32, 64 or 128)
//   K = taps x Cin, walked tap by tap in chunks of 32 input channels
//
//   warp 8       TMA producer: per K-block one 4-D box {32 ch, TW, TH, 1 image} of the NHWC input,
//                shifted by the tap's (dy,dx)*dilation -- out-of-bounds coordinates are zero-filled
//                by TMA, which IS the conv padding -- plus one 2-D box {32, BN} of the packed weights
//                [Cout][tap][Cin]; 128-byte-swizzled K-major tiles in a ring of mbarrier-guarded stages.
//   warps 0-7    two consumer warpgroups, 64 pixel rows each: wgmma.m64nBNk8 (tf32 in, fp32
//                accumulate in registers) straight from the stage, then the epilogue: +bias (+residual)
//                -> ReLU / LeakyReLU(0.1) -> optional round-to-tf32 -> NHWC output at a channel offset
//                of a (possibly wider) destination buffer, so torch.cat never happens.
//
// CTAs are persistent over (M tile, N tile) items (static round-robin; the ring runs on across items,
// so the producer fetches the next item's operands during the current epilogue), or one item per CTA.
// MC (pvnet_conv_set_multicast(1)): clusters of two CTAs on adjacent M tiles of the same N tile; each CTA
// loads its A box and HALF of the weight tile, multicast into both, so the weights cross L2 -> SM once per
// pair; a stage is refilled only after the consumers of BOTH CTAs released it.
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

template <int BN, bool MC>
__global__ void __launch_bounds__(CONV_THREADS, 1)
    k_conv_tap(const __grid_constant__ AMaps amaps, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ConvGeom g,
               const float *__restrict__ bias, const float *__restrict__ res, float *__restrict__ out)
{
    constexpr int B_BYTES = BN * CONV_KC * 4;
    constexpr int STAGE_BYTES = CONV_A_BYTES + B_BYTES;
    const int STAGES = g.stages;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + (size_t)STAGES * STAGE_BYTES);
    uint64_t *empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_img = g.tiles_x * g.tiles_y;
    const int n_tiles_n = g.Cout / BN;
    const int nkb = g.taps * g.cin_chunks;
    // MC: item = (M tile pair, N tile); CTA rank r of the pair takes M tile 2*pair + r (an odd tile count
    // leaves the last pair one tile short: its second CTA recomputes the last tile, identical values)
    const uint32_t crank = MC ? ptx::cluster_ctarank() : 0u;
    const int unit = MC ? (int)blockIdx.x >> 1 : (int)blockIdx.x, nunits = MC ? (int)gridDim.x >> 1 : (int)gridDim.x;
    auto item_tile = [&](int item, int &m_tile, int &n0) {
        const int mi = item / n_tiles_n;
        n0 = (item - mi * n_tiles_n) * BN;
        m_tile = MC ? min(2 * mi + (int)crank, g.total_m_tiles - 1) : mi;
    };

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            ptx::mbar_init(&full[s], 1);
            ptx::mbar_init(&empty[s], MC ? 16 : 8);    // one arrive per consumer warp (of both CTAs with MC)
        }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    if (MC) ptx::cluster_sync();                      // the peer's barriers exist before any remote arrive or multicast

    if (warp == 8) {
        if (lane == 0) {
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
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)STAGE_BYTES);
                        uint8_t *sa = smem + (size_t)s * STAGE_BYTES;
                        ptx::tma_load_4d(sa, &amaps.m[g.tap_map[tap]], &full[s], cc * CONV_KC, x0 + g.tap_ox[tap],
                                         y0 + g.tap_oy[tap], img);
                        if (MC)     // rows [crank*BN/2, +BN/2) of the weight tile, into both CTAs
                            ptx::tma_load_2d_mc(sa + CONV_A_BYTES + crank * (B_BYTES / 2), &tmB, &full[s],
                                                tap * g.cin_pad + cc * CONV_KC, n0 + (int)crank * (BN / 2), (uint16_t)0x3);
                        else
                            ptx::tma_load_2d(sa + CONV_A_BYTES, &tmB, &full[s], tap * g.cin_pad + cc * CONV_KC, n0);
                        if (++s == STAGES) {
                            s = 0;
                            ph ^= 1u;
                        }
                    }
            }
        }
    } else {
        // consumer warpgroup wg: pixel rows [64 wg, 64 wg + 64) of the tile
        const int wg = warp >> 2, wq = warp & 3;
        const int g8 = lane >> 2, t4 = lane & 3;
        const uint32_t smem_u = ptx::smem_u32(smem);
        auto release = [&](int st) {        // this warp is done reading stage st (in both CTAs' rings with MC)
            ptx::mbar_arrive(&empty[st]);
            if (MC) ptx::mbar_arrive_cluster(&empty[st], crank ^ 1u);
        };
        int s = 0;
        uint32_t ph = 0;
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
                if (prev >= 0 && lane == 0) release(prev);
                prev = s;
                if (++s == STAGES) {
                    s = 0;
                    ph ^= 1u;
                }
            }
            ptx::wgmma_wait<0>();
            ptx::fence_regs(acc);
            if (lane == 0) release(prev);

            int m_tile, n0;
            item_tile(item, m_tile, n0);
            const int img = m_tile / tiles_per_img;
            const int trem = m_tile - img * tiles_per_img;
            const int tyi = trem / g.tiles_x, txi = trem - tyi * g.tiles_x;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = wg * 64 + wq * 16 + g8 + 8 * h;
                const int y = tyi * g.TH + m / g.TW, x = txi * g.TW + m % g.TW;
                if (y >= g.Ho || x >= g.Wo) continue;
                const size_t pix = ((size_t)img * g.Ho + y) * g.Wo + x;
                float *optr = out + pix * g.out_cs + g.out_co + n0;
                const float *rptr = res ? res + pix * g.res_cs + g.res_co + n0 : nullptr;
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    const int c = 8 * j + 2 * t4;
                    const float2 bv = __ldg(reinterpret_cast<const float2 *>(bias + n0 + c));
                    float2 v = make_float2(acc[4 * j + 2 * h] + bv.x, acc[4 * j + 2 * h + 1] + bv.y);
                    if (rptr) {
                        const float2 rv = __ldg(reinterpret_cast<const float2 *>(rptr + c));
                        v.x += rv.x;
                        v.y += rv.y;
                    }
                    v.x = epi_act(v.x, g.act, g.round_out);
                    v.y = epi_act(v.y, g.act, g.round_out);
                    *reinterpret_cast<float2 *>(optr + c) = v;
                }
            }
        }
    }
    if (MC) ptx::cluster_sync();                      // no CTA exits while its peer may still write into it
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
    ConvGeom g;
    dim3 grid;
    size_t smem;
    int mc;
    const float *bias, *res;
    float *out;
};

// 1: CTAs persistent over the items (grid = one CTA per SM); 0: one item per CTA (pvnet_conv_set_persistent)
int g_conv_persist = 1;
// 1: CTA pairs share each weight tile through TMA multicast (pvnet_conv_set_multicast; default 0)
int g_conv_mc = 0;

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
    // N tile: 128 channels (64 fp32 accumulators per consumer thread) where Cout allows
    g.BN = d.Cout % 128 == 0 ? 128 : (d.Cout % 64 == 0 ? 64 : 32);
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
        p->mc = g_conv_mc;
        cuuint32_t box[2] = {(cuuint32_t)kc, (cuuint32_t)(p->mc ? g.BN / 2 : g.BN)};    // MC: each CTA loads half
        int rc = tma_encode(&p->tmB, d.w, 2, dims, strides, box, swz);
        if (rc) return rc;
    }
    // ring: as many stages as fit (at most 8) in the 227 KB a block may use
    const size_t stage_b = (size_t)CONV_A_BYTES + (size_t)g.BN * kc * 4;
    int st = (int)((227 * 1024 - 1024 - 256) / stage_b);
    if (st > 8) st = 8;
    g.stages = st;
    p->smem = 1024 + (size_t)st * stage_b + 256;
    // items: (M tile, N tile), or with MC (M tile pair, N tile) run by a two-CTA cluster
    const int m_units = p->mc ? (g.total_m_tiles + 1) / 2 : g.total_m_tiles;
    g.n_items = m_units * (d.Cout / g.BN);
    long long units = g_conv_persist ? (long long)sm_count() / (p->mc ? 2 : 1) : (long long)g.n_items;
    if (units > g.n_items) units = g.n_items;
    p->grid = dim3((unsigned)(units * (p->mc ? 2 : 1)));
    p->bias = d.bias;
    p->res = d.res;
    p->out = d.out;
    return PVNET_OK;
}

template <int BN, bool MC>
int conv_launch_t(const ConvPlan &p, cudaStream_t s)
{
    const cudaError_t attr_err = ensure_max_smem((const void *)k_conv_tap<BN, MC>, 227 * 1024);
    PV_CUDA(attr_err);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = p.grid;
    cfg.blockDim = dim3(CONV_THREADS);
    cfg.dynamicSmemBytes = p.smem;
    cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = MC ? 2 : 1;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = MC ? 1 : 0;
    PV_CUDA(cudaLaunchKernelEx(&cfg, k_conv_tap<BN, MC>, p.amaps, p.tmB, p.g, p.bias, p.res, p.out));
    PV_LAUNCHED("k_conv_tap");
    return PVNET_OK;
}

int conv_launch(const ConvPlan &p, cudaStream_t s)
{
    if (p.mc) {
        if (p.g.BN == 128) return conv_launch_t<128, true>(p, s);
        if (p.g.BN == 64) return conv_launch_t<64, true>(p, s);
        return conv_launch_t<32, true>(p, s);
    }
    if (p.g.BN == 128) return conv_launch_t<128, false>(p, s);
    if (p.g.BN == 64) return conv_launch_t<64, false>(p, s);
    return conv_launch_t<32, false>(p, s);
}

size_t conv_plan_size() { return sizeof(ConvPlan); }
int conv_plan_at(const ConvDesc &d, void *storage) { return conv_plan(d, new (storage) ConvPlan()); }
int conv_launch_at(const void *storage, cudaStream_t s) { return conv_launch(*static_cast<const ConvPlan *>(storage), s); }

}  // namespace pvnet

extern "C" {

int pvnet_conv_set_multicast(int on)
{
    PV_CHECK_ARG(on == 0 || on == 1, "multicast mode must be 0 or 1");
    pvnet::g_conv_mc = on;
    return PVNET_OK;
}

int pvnet_conv_set_persistent(int on)
{
    pvnet::g_conv_persist = on ? 1 : 0;
    return PVNET_OK;
}

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
