// backbone_aux.cu -- the non-GEMM kernels of Resnet18_8s (lib/networks/resnet.py:200-220,
// lib/networks/model_repository.py:64-80): the image's space-to-depth + NHWC slice packing for the
// tensor-core stem and convraw.0, max-pool 3x3/2, bilinear x2 upsampling (align_corners=True), and the
// final 1x1 conv + per-pixel argmax head that writes the reference's NCHW outputs.
// All of them are HBM-bound streaming kernels.
#include "conv_tc.cuh"
#include "ptx.cuh"
#include <algorithm>
#include <cmath>

namespace pvnet {

// ------------------------------------------------------------------ space-to-depth + image packing
// One pass over the NCHW image that writes (a) S [b,H/2,W/2,16]: the 2x2 space-to-depth image,
// channel (py*2+px)*3+c, 4 zero channels, for the tensor-core stem (a 7x7 stride-2 conv is a
// 4x4 stride-1 conv on S), and (b) the image slice of the convraw.0 input buffer (3 channels +
// 5 zeros at out_co).  Values rounded to tf32.
// U8 = true: `in` is a raw uint8 HWC image [b,H,W,3] (what an image decoder yields) and the kernel
// applies torchvision's ToTensor + Normalize in their own fp32 arithmetic (tools/demo.py:89-95,
// lib/datasets/linemod_dataset.py:191-195): (float(v) / 255 - mean[c]) / std[c], three correctly
// rounded ops -- bit-identical to feeding the float path with the torch-normalised tensor, at a
// quarter of the input bytes.
// RAW = true (the training stem, pvnet_stem_s2d_nhwc): the image slice gets the fp32 image values unrounded (the
// normalised values for a uint8 input), the image convraw.0 reads in training; S stays TF32-rounded.
// HALF = true (Resnet50_8s_2o): instead of the full-resolution image slice, `out` [b,H/2,W/2,out_cs] gets at out_co
// x_ds = F.interpolate(image, scale_factor=0.5, mode='bilinear') (3 channels + 5 zeros), the average of the 2x2 block
// this thread already holds, in the rounding sequence of torch's CUDA kernel (DESIGN.md §21); TF32-rounded unless RAW.
struct Norm3 {
    float mean[3], std[3];
};
template <bool U8, bool RAW = false, bool HALF = false>
__global__ void __launch_bounds__(128)
    k_s2d_pack(const void *__restrict__ in_v, Norm3 nrm, float *__restrict__ s2d, float *__restrict__ out, int H, int W,
               int out_cs, int out_co)
{
    const float *in = static_cast<const float *>(in_v);
    // grid.y = image * H/2 + half-resolution row; a block covers 128 half-resolution columns.
    // Loads are coalesced float2 reads of the six (channel, row) lines; both outputs are staged in
    // shared memory so that the stores are coalesced too (a thread-per-pixel store touches 32
    // different 64-byte / 160-byte-strided records per instruction).
    __shared__ float4 sS[128 * 4];        // [px][4 chunks], chunk j of px at j ^ ((px >> 1) & 3)
    __shared__ float4 sI[2][256];         // [row parity][full-resolution column]: (r, g, b, 0)
    const int W2 = W >> 1, H2 = H >> 1;
    const int xb = blockIdx.x * 128, t = threadIdx.x;
    const int x2 = xb + t;
    const int n = blockIdx.y / H2, y2 = blockIdx.y - n * H2;
    const size_t plane = (size_t)H * W;
    if (x2 < W2) {
        float v[16];
        float raw[12];                    // RAW: the unrounded values, in v's order
        if (U8) {
            // two rows x (2 pixels x 3 bytes): three 16-bit loads per row, coalesced across the warp
            const unsigned short *src8 = reinterpret_cast<const unsigned short *>(
                static_cast<const unsigned char *>(in_v) + (((size_t)n * H + 2 * y2) * W + 2 * x2) * 3);
#pragma unroll
            for (int py = 0; py < 2; ++py) {
                unsigned bytes[6];
#pragma unroll
                for (int j = 0; j < 3; ++j) {
                    const unsigned q = __ldg(src8 + (size_t)py * W * 3 / 2 + j);
                    bytes[2 * j] = q & 0xffu;
                    bytes[2 * j + 1] = q >> 8;
                }
#pragma unroll
                for (int px = 0; px < 2; ++px)
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float t = __fdiv_rn(__fsub_rn(__fdiv_rn((float)bytes[px * 3 + c], 255.f), nrm.mean[c]), nrm.std[c]);
                        v[(py * 2 + px) * 3 + c] = ptx::round_tf32(t);
                        if constexpr (RAW || HALF) raw[(py * 2 + px) * 3 + c] = t;
                    }
            }
        } else {
            const float *src = in + (size_t)n * 3 * plane + (size_t)(2 * y2) * W + 2 * x2;
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int py = 0; py < 2; ++py) {
                    const float2 q = __ldg(reinterpret_cast<const float2 *>(src + c * plane + py * W));
                    v[(py * 2 + 0) * 3 + c] = ptx::round_tf32(q.x);
                    v[(py * 2 + 1) * 3 + c] = ptx::round_tf32(q.y);
                    if constexpr (RAW || HALF) {
                        raw[(py * 2 + 0) * 3 + c] = q.x;
                        raw[(py * 2 + 1) * 3 + c] = q.y;
                    }
                }
        }
        v[12] = v[13] = v[14] = v[15] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j)
            sS[t * 4 + (j ^ ((t >> 1) & 3))] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
        if constexpr (HALF) {
            // torch's upsample_bilinear2d_out_frame at source 2i + 0.5 (every weight 0.5):
            // h0 * (w0 * a + w1 * b) + h1 * (w0 * c + w1 * d), products exact
            float xd[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float t0 = __fadd_rn(__fmul_rn(0.5f, raw[c]), __fmul_rn(0.5f, raw[3 + c]));
                const float t1 = __fadd_rn(__fmul_rn(0.5f, raw[6 + c]), __fmul_rn(0.5f, raw[9 + c]));
                const float m = __fadd_rn(__fmul_rn(0.5f, t0), __fmul_rn(0.5f, t1));
                xd[c] = RAW ? m : ptx::round_tf32(m);
            }
            float4 *o = reinterpret_cast<float4 *>(out + ((size_t)blockIdx.y * W2 + x2) * out_cs + out_co);
            o[0] = make_float4(xd[0], xd[1], xd[2], 0.f);
            o[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int py = 0; py < 2 && !HALF; ++py)
#pragma unroll
            for (int px = 0; px < 2; ++px) {
                const int b = (py * 2 + px) * 3;
                if constexpr (RAW)
                    sI[py][2 * t + px] = make_float4(raw[b], raw[b + 1], raw[b + 2], 0.f);
                else
                    sI[py][2 * t + px] = make_float4(v[b], v[b + 1], v[b + 2], 0.f);
            }
    }
    __syncthreads();
    const int npx = min(128, W2 - xb);                    // half-resolution pixels this block holds
    float4 *so = reinterpret_cast<float4 *>(s2d + ((size_t)blockIdx.y * W2 + xb) * 16);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int L = t + 128 * r, px = L >> 2, j = L & 3;
        if (px < npx) so[L] = sS[px * 4 + (j ^ ((px >> 1) & 3))];
    }
    // image slice: lane pairs write the 32 bytes (3 channels + 5 zeros) of one full-resolution pixel
#pragma unroll
    for (int py = 0; py < 2 && !HALF; ++py) {
        float *orow = out + (((size_t)n * H + 2 * y2 + py) * W + 2 * xb) * out_cs + out_co;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int L = t + 128 * r, px = L >> 1, half = L & 1;
            if (px < 2 * npx)
                *reinterpret_cast<float4 *>(orow + (size_t)px * out_cs + half * 4) =
                    half ? make_float4(0.f, 0.f, 0.f, 0.f) : sI[py][px];
        }
    }
}

int launch_s2d_pack(const void *in, int in_is_u8, const float *mean3, const float *std3, float *s2d, float *out, int b,
                    int H, int W, int out_cs, int out_co, int half, cudaStream_t s)
{
    dim3 grid((unsigned)((W / 2 + 127) / 128), (unsigned)(b * (H / 2)));
    Norm3 nrm{};
    if (in_is_u8) {
        for (int c = 0; c < 3; ++c) {
            nrm.mean[c] = mean3[c];
            nrm.std[c] = std3[c];
        }
        if (half)
            k_s2d_pack<true, false, true><<<grid, 128, 0, s>>>(in, nrm, s2d, out, H, W, out_cs, out_co);
        else
            k_s2d_pack<true><<<grid, 128, 0, s>>>(in, nrm, s2d, out, H, W, out_cs, out_co);
    } else if (half) {
        k_s2d_pack<false, false, true><<<grid, 128, 0, s>>>(in, nrm, s2d, out, H, W, out_cs, out_co);
    } else {
        k_s2d_pack<false><<<grid, 128, 0, s>>>(in, nrm, s2d, out, H, W, out_cs, out_co);
    }
    PV_LAUNCHED("k_s2d_pack");
    return PVNET_OK;
}

// ------------------------------------------------------------------ max-pool 3x3/2 pad 1
// (resnet.py:142,204).  in NHWC [b,H,W,in_cs] at in_co (C channels) -> out [b,H/2,W/2,C]
__global__ void __launch_bounds__(256)
    k_maxpool(const float *__restrict__ in, float *__restrict__ out, int H, int W, int C, int in_cs, int in_co)
{
    // grid.y = image * H/2 + output row
    const int c4 = C >> 2, Ho = H >> 1, Wo = W >> 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Wo * c4) return;
    const int ox = i / c4, cg = i - ox * c4;
    const int n = blockIdx.y / Ho, oy = blockIdx.y - n * Ho;
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
        const int iy = oy * 2 + dy;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int ix = ox * 2 + dx;
            if (ix < 0 || ix >= W) continue;
            const float4 v = __ldg(reinterpret_cast<const float4 *>(in + (((size_t)n * H + iy) * W + ix) * in_cs + in_co) + cg);
            m.x = fmaxf(m.x, v.x);
            m.y = fmaxf(m.y, v.y);
            m.z = fmaxf(m.z, v.z);
            m.w = fmaxf(m.w, v.w);
        }
    }
    reinterpret_cast<float4 *>(out)[((size_t)blockIdx.y * Wo + ox) * c4 + cg] = m;
}

int launch_maxpool(const float *in, float *out, int b, int H, int W, int C, int in_cs, int in_co, cudaStream_t s)
{
    dim3 grid((unsigned)(((W / 2) * (C / 4) + 255) / 256), (unsigned)(b * (H / 2)));
    k_maxpool<<<grid, 256, 0, s>>>(in, out, H, W, C, in_cs, in_co);
    PV_LAUNCHED("k_maxpool");
    return PVNET_OK;
}

// ------------------------------------------------------------------ max-pool 3x3/2 pad 1, training
// Forward with argmax: torch's rule -- the window scanned row-major from -inf, an element wins when `v > max ||
// isnan(v)`, and with no winner (all -inf) the first in-image element is the argmax.  The argmax is stored as a
// uint8 window code (dy*3 + dx, dy/dx = 0..2 from the window origin (2oy-1, 2ox-1)).  One thread = one output pixel's
// 4-channel group.  in NHWC [b,H,W,C] dense -> out NHWC [b,H/2,W/2,C], code [b,H/2,W/2,C]; 64-bit offsets.
__global__ void __launch_bounds__(256)
    k_maxpool_train(const float *__restrict__ in, float *__restrict__ out, uchar4 *__restrict__ code, int H, int W,
                    int C, long long total)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c4 = C >> 2, Ho = H >> 1, Wo = W >> 1;
    const long long pix = i / c4;
    const int cg = (int)(i - pix * c4);
    const int ox = (int)(pix % Wo);
    const long long t = pix / Wo;
    const int oy = (int)(t % Ho);
    const long long n = t / Ho;
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    int k[4] = {-1, -1, -1, -1};
    int first = -1;
#pragma unroll
    for (int dy = 0; dy < 3; ++dy) {
        const int iy = 2 * oy - 1 + dy;
        if (iy < 0 || iy >= H) continue;
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) {
            const int ix = 2 * ox - 1 + dx;
            if (ix < 0 || ix >= W) continue;
            const float4 q = __ldg(reinterpret_cast<const float4 *>(in + ((n * H + iy) * W + ix) * C) + cg);
            const float v[4] = {q.x, q.y, q.z, q.w};
            const int cd = dy * 3 + dx;
            if (first < 0) first = cd;
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (v[e] > m[e] || isnan(v[e])) {
                    m[e] = v[e];
                    k[e] = cd;
                }
        }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e)
        if (k[e] < 0) k[e] = first;
    reinterpret_cast<float4 *>(out)[i] = make_float4(m[0], m[1], m[2], m[3]);
    code[i] = make_uchar4((unsigned char)k[0], (unsigned char)k[1], (unsigned char)k[2], (unsigned char)k[3]);
}

// Backward as a gather: input pixel (iy, ix) adds the dY of the windows whose code points at it, in ATen's order --
// outputs (oy, ox) ascending over ATen's window bounds, from 0.0f, one rounded fp32 add each.  No atomics.
// dout NHWC [b,H/2,W/2,C] dense, code as the forward wrote it -> din NHWC [b,H,W,C] dense, every element written.
__global__ void __launch_bounds__(256)
    k_maxpool_train_backward(const float *__restrict__ dout, const uchar4 *__restrict__ code, float *__restrict__ din,
                             int H, int W, int C, long long total)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c4 = C >> 2, Ho = H >> 1, Wo = W >> 1;
    const long long pix = i / c4;
    const int cg = (int)(i - pix * c4);
    const int ix = (int)(pix % W);
    const long long t = pix / W;
    const int iy = (int)(t % H);
    const long long n = t / H;
    // ATen's p_start / p_end for kernel 3, stride 2, pad 1, dilation 1
    const int oy0 = iy + 1 < 3 ? 0 : (iy + 1 - 3) / 2 + 1, oy1 = min((iy + 1) / 2 + 1, Ho);
    const int ox0 = ix + 1 < 3 ? 0 : (ix + 1 - 3) / 2 + 1, ox1 = min((ix + 1) / 2 + 1, Wo);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int oy = oy0; oy < oy1; ++oy)
        for (int ox = ox0; ox < ox1; ++ox) {
            const int want = (iy - (2 * oy - 1)) * 3 + (ix - (2 * ox - 1));
            const long long o = ((n * Ho + oy) * Wo + ox) * c4 + cg;
            const uchar4 kq = __ldg(code + o);
            const unsigned char kk[4] = {kq.x, kq.y, kq.z, kq.w};
            if (kk[0] != want && kk[1] != want && kk[2] != want && kk[3] != want) continue;
            const float4 gq = __ldg(reinterpret_cast<const float4 *>(dout) + o);
            const float g[4] = {gq.x, gq.y, gq.z, gq.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (kk[e] == want) acc[e] = __fadd_rn(acc[e], g[e]);
        }
    reinterpret_cast<float4 *>(din)[i] = make_float4(acc[0], acc[1], acc[2], acc[3]);
}

// ------------------------------------------------------------------ bilinear x2, align_corners=True
// nn.UpsamplingBilinear2d(scale_factor=2) (model_repository.py:35,43,51).  Same arithmetic
// as ATen's upsample_bilinear2d: scale=(in-1)/(out-1) in fp32, src=scale*dst, i0=(int)src,
// l1=src-i0, l0=1-l1, out = h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11).
// in NHWC [b,h,w,C] dense -> out NHWC [b,2h,2w,out_cs] at out_co; values rounded to tf32.
// w0*a + w1*b with lerp3's rounding sequence (fmul, then fma), four lanes
__device__ __forceinline__ float4 lerp2_4(float w0, const float4 &a, float w1, const float4 &b)
{
    return make_float4(__fmaf_rn(w1, b.x, __fmul_rn(w0, a.x)), __fmaf_rn(w1, b.y, __fmul_rn(w0, a.y)),
                       __fmaf_rn(w1, b.z, __fmul_rn(w0, a.z)), __fmaf_rn(w1, b.w, __fmul_rn(w0, a.w)));
}
// cvt.rna.tf32.f32 (nearest, ties away) as integer add + mask: identical for every finite input and infinity,
// two instructions per value instead of the four the conversion compiles to
__device__ __forceinline__ float4 round_tf32_4(const float4 &v)
{
    return make_float4(__uint_as_float((__float_as_uint(v.x) + 0x1000u) & 0xffffe000u),
                       __uint_as_float((__float_as_uint(v.y) + 0x1000u) & 0xffffe000u),
                       __uint_as_float((__float_as_uint(v.z) + 0x1000u) & 0xffffe000u),
                       __uint_as_float((__float_as_uint(v.w) + 0x1000u) & 0xffffe000u));
}
// ATen's index expressions for output index o of one axis (area_pixel_compute_source_index with align_corners, then
// upsample_bilinear2d's clamp): output o reads input i0 with weight l0 and i1 = i0 + (i0 < in-1) with weight l1.
// Written with _rn intrinsics so that no contraction can fuse `scale*o - i0` (torch's kernel rounds src first).
struct UpSrc {
    int i0, i1;
    float l0, l1;
};
__device__ __forceinline__ UpSrc up_src(float scale, int o, int in)
{
    const float src = __fmul_rn(scale, (float)o);
    const int i0 = (int)src;
    const float l1 = __fsub_rn(src, (float)i0);
    return {i0, i0 + (i0 < in - 1 ? 1 : 0), __fsub_rn(1.f, l1), l1};
}

// The training forward: torch's CUDA F.interpolate on a channels_last tensor (upsample_bilinear2d_nhwc_out_frame)
// bit for bit.  Its SASS (sm_90, torch 2.11) contracts h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11) as
//   a = fma(w1, v01, w0*v00)     b = fma(w0, v10, w1*v11)     out = fma(h0, a, h1*b)
// -- not lerp2's sequence for b and out -- so each output is computed from its own four loads, unrounded.
__device__ __forceinline__ void upsample2x_exact_block(const float *__restrict__ in, float *__restrict__ out, int n,
                                                       int j, int k, int h, int w, int C, int out_cs, int out_co,
                                                       float sy, float sx)
{
    const int c4 = C >> 2;
    const unsigned Wo = 2u * w;
#pragma unroll
    for (int oy = 0; oy < 2; ++oy) {
        const UpSrc ry = up_src(sy, 2 * j + oy, h);
        const unsigned r0 = ((unsigned)n * h + ry.i0) * (unsigned)w, r1 = ((unsigned)n * h + ry.i1) * (unsigned)w;
#pragma unroll
        for (int ox = 0; ox < 2; ++ox) {
            const UpSrc rx = up_src(sx, 2 * k + ox, w);
            const unsigned o00 = (r0 + rx.i0) * (unsigned)C, o01 = (r0 + rx.i1) * (unsigned)C;
            const unsigned o10 = (r1 + rx.i0) * (unsigned)C, o11 = (r1 + rx.i1) * (unsigned)C;
            const unsigned oo = (((unsigned)n * 2u * h + 2u * j + oy) * Wo + 2u * k + ox) * (unsigned)out_cs +
                                (unsigned)out_co;
            for (int cg = threadIdx.x; cg < c4; cg += 8) {
                const float *ip = in + cg * 4;
                const float4 v00 = __ldg(reinterpret_cast<const float4 *>(ip + o00));
                const float4 v01 = __ldg(reinterpret_cast<const float4 *>(ip + o01));
                const float4 v10 = __ldg(reinterpret_cast<const float4 *>(ip + o10));
                const float4 v11 = __ldg(reinterpret_cast<const float4 *>(ip + o11));
                float4 r;
#define PV_UP_EXACT(f)                                                                                     \
    r.f = __fmaf_rn(ry.l0, __fmaf_rn(rx.l1, v01.f, __fmul_rn(rx.l0, v00.f)),                               \
                    __fmul_rn(ry.l1, __fmaf_rn(rx.l0, v10.f, __fmul_rn(rx.l1, v11.f))))
                PV_UP_EXACT(x);
                PV_UP_EXACT(y);
                PV_UP_EXACT(z);
                PV_UP_EXACT(w);
#undef PV_UP_EXACT
                *reinterpret_cast<float4 *>(out + oo + cg * 4) = r;
            }
        }
    }
}

// TF32 = true: the eval path's kernel (values rounded to tf32 for the next tensor-core conv); false: the training
// forward, exact fp32 in torch's rounding sequence (upsample2x_exact_block).
template <bool TF32>
__global__ void __launch_bounds__(256)
    k_upsample2x(const float *__restrict__ in, float *__restrict__ out, int h, int w, int C, int out_cs, int out_co,
                 float sy, float sx)
{
    if constexpr (!TF32) {
        const int k = blockIdx.x * blockDim.y + threadIdx.y;
        if (k >= w) return;
        const int n = blockIdx.y / h, j = blockIdx.y - n * h;
        upsample2x_exact_block(in, out, n, j, k, h, w, C, out_cs, out_co, sy, sx);
        return;
    }
    // One thread = the 2x2 output block (2j..2j+1, 2k..2k+1) of 4-channel groups cg, cg+8, ...  With
    // align_corners=True and scale 2 the source rows of output rows 2j, 2j+1 all lie in
    // {j-1, j, j+1} (same for columns), so the block needs a 3x3 neighbourhood: 9 loads for 4
    // outputs instead of 16.  Each output keeps PyTorch's separable form
    // h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11); the third row/column enters with weight 0 (and a
    // clamped row/column index reproduces v10 = v00 at the border, as ATen's index clamp does).
    // The kernel was instruction-issue bound (ncu: 79 % issue-active, 31 instructions per output
    // float), so weights and offsets are computed once per thread and kept in 32-bit arithmetic.
    // blockDim = (8 channel groups, 32 pixel pairs); grid.y = image * h + j.
    const int c4 = C >> 2;
    const int k = blockIdx.x * blockDim.y + threadIdx.y;
    if (k >= w) return;
    const int n = blockIdx.y / h, j = blockIdx.y - n * h;

    float wy[2][3], wx[2][3];
    bool pat[2][2];                                     // [o][0] = uy, [o][1] = ux
#pragma unroll
    for (int o = 0; o < 2; ++o) {
        const float fy = sy * (float)(2 * j + o), fx = sx * (float)(2 * k + o);
        const int y0 = (int)fy, x0 = (int)fx;
        const float h1 = fy - (float)y0, h0 = 1.f - h1, w1 = fx - (float)x0, w0 = 1.f - w1;
        const bool uy = y0 >= j, ux = x0 >= k;          // source pair is rows (j, j+1) rather than (j-1, j)
        pat[o][0] = uy;
        pat[o][1] = ux;
        wy[o][0] = uy ? 0.f : h0;
        wy[o][1] = uy ? h0 : h1;
        wy[o][2] = uy ? h1 : 0.f;
        wx[o][0] = ux ? 0.f : w0;
        wx[o][1] = ux ? w0 : w1;
        wx[o][2] = ux ? w1 : 0.f;
    }
    // element offsets of the 3x3 neighbourhood (clamped) and of the 2x2 outputs; 32-bit by contract
    unsigned ioff[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const unsigned y = (unsigned)min(max(j - 1 + r, 0), h - 1);
        const unsigned rowb = ((unsigned)n * h + y) * (unsigned)w;
#pragma unroll
        for (int c = 0; c < 3; ++c) ioff[r][c] = (rowb + (unsigned)min(max(k - 1 + c, 0), w - 1)) * (unsigned)C;
    }
    const unsigned Wo = 2u * w;
    const unsigned o00 = (((unsigned)n * 2u * h + 2u * j) * Wo + 2u * k) * (unsigned)out_cs + (unsigned)out_co;
    const unsigned orow = Wo * (unsigned)out_cs;

    // All blocks but those of the first row / column (and a last one whose scale*index rounds down) have the same
    // pattern: output 2j reads source rows (j-1, j), output 2j+1 rows (j, j+1), same for columns -- two-term sums (8 instead of 12
    // floating-point instructions per float4; the kernel is issue-bound).  lerp3 with its zero weight rounds
    // identically (fmul of the first product, fma of the second; adding 0*x changes nothing), so both paths
    // agree to the last bit.
    const bool interior = !pat[0][0] && pat[1][0] && !pat[0][1] && pat[1][1];
    if (interior) {
        const float a0 = wx[0][0], a1 = wx[0][1], b0 = wx[1][1], b1 = wx[1][2];      // column weights of outputs 2k, 2k+1
        const float p0 = wy[0][0], p1 = wy[0][1], q0 = wy[1][1], q1 = wy[1][2];      // row weights of outputs 2j, 2j+1
        for (int cg = threadIdx.x; cg < c4; cg += 8) {
            const float *ip = in + cg * 4;
            float4 t[3][2];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const float4 a = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][0]));
                const float4 bq = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][1]));
                const float4 c = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][2]));
                t[r][0] = lerp2_4(a0, a, a1, bq);
                t[r][1] = lerp2_4(b0, bq, b1, c);
            }
            float *op = out + cg * 4;
#pragma unroll
            for (int ox = 0; ox < 2; ++ox) {
                *reinterpret_cast<float4 *>(op + o00 + (unsigned)ox * (unsigned)out_cs) = round_tf32_4(lerp2_4(p0, t[0][ox], p1, t[1][ox]));
                *reinterpret_cast<float4 *>(op + o00 + orow + (unsigned)ox * (unsigned)out_cs) = round_tf32_4(lerp2_4(q0, t[1][ox], q1, t[2][ox]));
            }
        }
        return;
    }
    for (int cg = threadIdx.x; cg < c4; cg += 8) {
        const float *ip = in + cg * 4;
        float4 t[3][2];                                   // per source row: the two horizontally interpolated values
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float4 a = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][0]));
            const float4 bq = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][1]));
            const float4 c = __ldg(reinterpret_cast<const float4 *>(ip + ioff[r][2]));
#pragma unroll
            for (int o = 0; o < 2; ++o) {
                t[r][o].x = lerp3(wx[o][0], a.x, wx[o][1], bq.x, wx[o][2], c.x);
                t[r][o].y = lerp3(wx[o][0], a.y, wx[o][1], bq.y, wx[o][2], c.y);
                t[r][o].z = lerp3(wx[o][0], a.z, wx[o][1], bq.z, wx[o][2], c.z);
                t[r][o].w = lerp3(wx[o][0], a.w, wx[o][1], bq.w, wx[o][2], c.w);
            }
        }
        float *op = out + cg * 4;
#pragma unroll
        for (int oy = 0; oy < 2; ++oy)
#pragma unroll
            for (int ox = 0; ox < 2; ++ox) {
                float4 v;
                v.x = lerp3(wy[oy][0], t[0][ox].x, wy[oy][1], t[1][ox].x, wy[oy][2], t[2][ox].x);
                v.y = lerp3(wy[oy][0], t[0][ox].y, wy[oy][1], t[1][ox].y, wy[oy][2], t[2][ox].y);
                v.z = lerp3(wy[oy][0], t[0][ox].z, wy[oy][1], t[1][ox].z, wy[oy][2], t[2][ox].z);
                v.w = lerp3(wy[oy][0], t[0][ox].w, wy[oy][1], t[1][ox].w, wy[oy][2], t[2][ox].w);
                *reinterpret_cast<float4 *>(op + o00 + (unsigned)oy * orow + (unsigned)ox * (unsigned)out_cs) = round_tf32_4(v);
            }
    }
}

int launch_upsample2x(const float *in, float *out, int b, int h, int w, int C, int out_cs, int out_co, cudaStream_t s)
{
    PV_CHECK_ARG((long long)b * 4 * h * w * out_cs < (1LL << 32) && (long long)b * h * w * C < (1LL << 32),
                 "upsample: tensor too large for 32-bit element offsets");
    const float sy = (float)(h - 1) / (float)(2 * h - 1), sx = (float)(w - 1) / (float)(2 * w - 1);
    dim3 grid((unsigned)((w + 31) / 32), (unsigned)(b * h));
    k_upsample2x<true><<<grid, dim3(8, 32), 0, s>>>(in, out, h, w, C, out_cs, out_co, sy, sx);
    PV_LAUNCHED("k_upsample2x");
    return PVNET_OK;
}

// ------------------------------------------------------------------ bilinear x2 backward
// dX = U^T dY for the training forward above, as a gather: input pixel (i, j) sums exactly the terms ATen's CUDA
// backward (upsample_bilinear2d_backward_nhwc_out_frame) adds to it with atomics -- term = (hl * wl) * g, two
// rounded products -- in a fixed order: output pixels ascending (row-major), and within one output pixel ATen's term
// order (l0 l0, l0 l1, l1 l0, l1 l1).  No atomics: run-to-run identical, and a sum torch's own backward can return.
// Window rule (oracle/upsample_oracle.py, tests/test_upsample_grad_cpu.py): input index i along an axis is fed by
// the outputs o = 2i-2 ... 2i+3 whose up_src lands on i (slot 0 if i0 == i, slot 1 if i1 == i; both at the last
// index, where i0p = 0).  Away from the borders that is always o = 2i-1, 2i through slot 1 and 2i+1, 2i+2 through
// slot 0 (the interior pattern): a thread whose row and column are both interior takes 16 unconditional terms with
// the products hl*wl computed once; every other thread walks the 6 x 6 candidates.
// One thread = one input pixel, 4-channel groups cg, cg+8, ...  blockDim = (8 channel groups, 32 pixels of a row),
// grid.y = image * h + i.  dY rows 2i-1 ... 2i+2 are shared with the neighbouring rows' blocks through L1/L2, so dY
// comes from HBM about once.
__device__ __forceinline__ bool up_interior(float scale, int i, int in)
{
    if (i < 1 || i > in - 2) return false;
    bool ok = true;
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const UpSrc u = up_src(scale, 2 * i - 2 + r, in);
        const bool s0 = u.i0 == i, s1 = u.i1 == i;
        ok = ok && (r == 1 || r == 2 ? (s1 && !s0) : r == 3 || r == 4 ? (s0 && !s1) : (!s0 && !s1));
    }
    return ok;
}

__global__ void __launch_bounds__(256)
    k_upsample2x_backward(const float *__restrict__ dout, int dout_cs, int dout_co, float *__restrict__ din, int h,
                          int w, int C, float sy, float sx)
{
    const int c4 = C >> 2;
    const int j = blockIdx.x * blockDim.y + threadIdx.y;
    if (j >= w) return;
    const int n = blockIdx.y / h, i = blockIdx.y - n * h;
    const unsigned Wo = 2u * w;
    const unsigned img = (unsigned)n * 2u * h;
    const unsigned dx_off = ((unsigned)blockIdx.y * (unsigned)w + (unsigned)j) * (unsigned)C;
    const float *gp = dout + dout_co;

    if (up_interior(sy, i, h) && up_interior(sx, j, w)) {
        float wy[4], wx[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const UpSrc uy = up_src(sy, 2 * i - 1 + r, h), ux = up_src(sx, 2 * j - 1 + r, w);
            wy[r] = r < 2 ? uy.l1 : uy.l0;
            wx[r] = r < 2 ? ux.l1 : ux.l0;
        }
        float p[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) p[r][c] = __fmul_rn(wy[r], wx[c]);
        const unsigned g00 = ((img + 2u * i - 1u) * Wo + 2u * j - 1u) * (unsigned)dout_cs;
        const unsigned grow = Wo * (unsigned)dout_cs;
        for (int cg = threadIdx.x; cg < c4; cg += 8) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float4 g = __ldg(reinterpret_cast<const float4 *>(
                        gp + g00 + (unsigned)r * grow + (unsigned)c * (unsigned)dout_cs + cg * 4));
                    acc.x = __fadd_rn(acc.x, __fmul_rn(p[r][c], g.x));
                    acc.y = __fadd_rn(acc.y, __fmul_rn(p[r][c], g.y));
                    acc.z = __fadd_rn(acc.z, __fmul_rn(p[r][c], g.z));
                    acc.w = __fadd_rn(acc.w, __fmul_rn(p[r][c], g.w));
                }
            *reinterpret_cast<float4 *>(din + dx_off + cg * 4) = acc;
        }
        return;
    }
    // borders: every candidate (oy, ox), the terms that land on (i, j) in ATen's order
    for (int cg = threadIdx.x; cg < c4; cg += 8) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
        for (int r = 0; r < 6; ++r) {
            const int oy = 2 * i - 2 + r;
            if (oy < 0 || oy >= 2 * h) continue;
            const UpSrc uy = up_src(sy, oy, h);
            const bool y0 = uy.i0 == i, y1 = uy.i1 == i;
            if (!y0 && !y1) continue;
#pragma unroll 1
            for (int c = 0; c < 6; ++c) {
                const int ox = 2 * j - 2 + c;
                if (ox < 0 || ox >= (int)Wo) continue;
                const UpSrc ux = up_src(sx, ox, w);
                const bool x0 = ux.i0 == j, x1 = ux.i1 == j;
                if (!x0 && !x1) continue;
                const float4 g = __ldg(reinterpret_cast<const float4 *>(
                    gp + ((img + (unsigned)oy) * Wo + (unsigned)ox) * (unsigned)dout_cs + cg * 4));
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const bool hit = (t < 2 ? y0 : y1) && ((t & 1) ? x1 : x0);
                    if (!hit) continue;
                    const float q = __fmul_rn(t < 2 ? uy.l0 : uy.l1, (t & 1) ? ux.l1 : ux.l0);
                    acc.x = __fadd_rn(acc.x, __fmul_rn(q, g.x));
                    acc.y = __fadd_rn(acc.y, __fmul_rn(q, g.y));
                    acc.z = __fadd_rn(acc.z, __fmul_rn(q, g.z));
                    acc.w = __fadd_rn(acc.w, __fmul_rn(q, g.w));
                }
            }
        }
        *reinterpret_cast<float4 *>(din + dx_off + cg * 4) = acc;
    }
}

static int check_upsample_args(const char *what, const float *dense, int C, const float *sliced, int cs, int co,
                               int b, int h, int w)
{
    PV_CHECK_ARG(dense && sliced, "%s: null pointer", what);
    PV_CHECK_ARG(b > 0 && h > 0 && w > 0, "%s: b, h, w must be positive", what);
    PV_CHECK_ARG(C > 0 && C % 4 == 0 && cs % 4 == 0 && co % 4 == 0 && co >= 0,
                 "%s: channels, stride and offset must be multiples of 4 floats", what);
    PV_CHECK_ARG(co + C <= cs, "%s: channel slice exceeds its buffer", what);
    PV_CHECK_ARG((uintptr_t)dense % 16 == 0 && (uintptr_t)sliced % 16 == 0, "%s: pointers must be 16-byte aligned",
                 what);
    PV_CHECK_ARG((long long)b * 4 * h * w * cs < (1LL << 32) && (long long)b * h * w * C < (1LL << 32),
                 "%s: tensor too large for 32-bit element offsets", what);
    return PVNET_OK;
}

}  // namespace pvnet

extern "C" {

int pvnet_upsample2x_nhwc(const float *in, int C, float *out, int out_cs, int out_co, int b, int h, int w,
                          pvnet_stream_t stream)
{
    if (int rc = pvnet::check_upsample_args("upsample2x", in, C, out, out_cs, out_co, b, h, w)) return rc;
    const float sy = (float)(h - 1) / (float)(2 * h - 1), sx = (float)(w - 1) / (float)(2 * w - 1);
    dim3 grid((unsigned)((w + 31) / 32), (unsigned)(b * h));
    pvnet::k_upsample2x<false><<<grid, dim3(8, 32), 0, (cudaStream_t)stream>>>(in, out, h, w, C, out_cs, out_co, sy, sx);
    PV_LAUNCHED("k_upsample2x_exact");
    return PVNET_OK;
}

int pvnet_upsample2x_backward_nhwc(const float *dout, int dout_cs, int dout_co, int C, float *din, int b, int h, int w,
                                   pvnet_stream_t stream)
{
    if (int rc = pvnet::check_upsample_args("upsample2x backward", din, C, dout, dout_cs, dout_co, b, h, w)) return rc;
    const float sy = (float)(h - 1) / (float)(2 * h - 1), sx = (float)(w - 1) / (float)(2 * w - 1);
    dim3 grid((unsigned)((w + 31) / 32), (unsigned)(b * h));
    pvnet::k_upsample2x_backward<<<grid, dim3(8, 32), 0, (cudaStream_t)stream>>>(dout, dout_cs, dout_co, din, h, w, C,
                                                                                 sy, sx);
    PV_LAUNCHED("k_upsample2x_backward");
    return PVNET_OK;
}

static int check_maxpool_args(const char *what, const void *a, const void *b, const void *c, int bn, int H, int W,
                              int C)
{
    PV_CHECK_ARG(a && b && c, "%s: null pointer", what);
    PV_CHECK_ARG(bn > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "%s: b, H, W must be positive, H and W even",
                 what);
    PV_CHECK_ARG(C > 0 && C % 4 == 0, "%s: C must be a positive multiple of 4", what);
    PV_CHECK_ARG((uintptr_t)a % 16 == 0 && (uintptr_t)b % 16 == 0 && (uintptr_t)c % 16 == 0,
                 "%s: pointers must be 16-byte aligned", what);
    return PVNET_OK;
}

int pvnet_maxpool3x3s2_nhwc(const float *in, float *out, uint8_t *code, int b, int H, int W, int C,
                            pvnet_stream_t stream)
{
    if (int rc = check_maxpool_args("maxpool", in, out, code, b, H, W, C)) return rc;
    const long long total = (long long)b * (H / 2) * (W / 2) * (C / 4);
    pvnet::k_maxpool_train<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        in, out, reinterpret_cast<uchar4 *>(code), H, W, C, total);
    PV_LAUNCHED("k_maxpool_train");
    return PVNET_OK;
}

int pvnet_maxpool3x3s2_backward_nhwc(const float *dout, const uint8_t *code, float *din, int b, int H, int W, int C,
                                     pvnet_stream_t stream)
{
    if (int rc = check_maxpool_args("maxpool backward", dout, code, din, b, H, W, C)) return rc;
    const long long total = (long long)b * H * W * (C / 4);
    pvnet::k_maxpool_train_backward<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        dout, reinterpret_cast<const uchar4 *>(code), din, H, W, C, total);
    PV_LAUNCHED("k_maxpool_train_backward");
    return PVNET_OK;
}

}  // extern "C"

// pvnet_stem_s2d_nhwc (half = 0: the image slice of img at full resolution) and pvnet_stem_s2d_half_nhwc (half = 1:
// x_ds of img at H/2 x W/2)
static int stem_s2d(const void *image, int image_is_u8, const float *mean3, const float *std3, const float *w_s2d,
                    const float *bias, float *s2d, float *out, float *img, int img_cs, int img_co, int b, int H, int W,
                    int half, pvnet_stream_t stream)
{
    PV_CHECK_ARG(image && w_s2d && bias && s2d && out && img, "stem: null pointer");
    PV_CHECK_ARG(image_is_u8 ? mean3 && std3 : !mean3 && !std3,
                 "stem: mean and std must be given for a uint8 image and NULL for a float image");
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0, "stem: b, H, W must be positive");
    PV_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "stem: H and W must be even, got %d x %d", H, W);
    PV_CHECK_ARG((uintptr_t)image % (image_is_u8 ? 2 : 8) == 0 && (uintptr_t)s2d % 16 == 0 &&
                     (uintptr_t)out % 16 == 0 && (uintptr_t)img % 16 == 0 && (uintptr_t)w_s2d % 16 == 0,
                 "stem: image must be 2-byte (uint8) or 8-byte (float), s2d / out / img / weights 16-byte aligned");
    PV_CHECK_ARG(img_co >= 0 && img_co % 4 == 0 && img_cs % 4 == 0 && img_co + 8 <= img_cs,
                 "stem: image slice [%d, %d+8) must lie in a channel stride %d, offset and stride multiples of 4",
                 img_co, img_co, img_cs);
    pvnet::Norm3 nrm{};                    // read by the uint8 form only
    for (int c = 0; image_is_u8 && c < 3; ++c) {
        PV_CHECK_ARG(std::isfinite(mean3[c]) && std::isfinite(std3[c]) && std3[c] != 0.f,
                     "stem: mean and std must be finite and std nonzero (channel %d: %g, %g)", c, mean3[c], std3[c]);
        nrm.mean[c] = mean3[c];
        nrm.std[c] = std3[c];
    }
    // k_s2d_pack's grid.y is image * H/2 + row, at most 65535: launch it over chunks of whole images.  Either image
    // holds 3*H*W elements per image.
    PV_CHECK_ARG(H / 2 <= 65535, "stem: H/2 = %d rows exceed the 65535-row launch limit", H / 2);
    const int per = 65535 / (H / 2);
    for (int n0 = 0; n0 < b; n0 += per) {
        const int nb = std::min(per, b - n0);
        const dim3 grid((unsigned)((W / 2 + 127) / 128), (unsigned)(nb * (H / 2)));
        const size_t in0 = (size_t)n0 * 3 * H * W;
        float *s2d0 = s2d + (size_t)n0 * (H / 2) * (W / 2) * 16;
        float *img0 = img + (size_t)n0 * (half ? (size_t)(H / 2) * (W / 2) : (size_t)H * W) * img_cs;
        cudaStream_t st = (cudaStream_t)stream;
        const void *im0 = image_is_u8 ? (const void *)(static_cast<const uint8_t *>(image) + in0)
                                      : (const void *)(static_cast<const float *>(image) + in0);
        if (image_is_u8 && half)
            pvnet::k_s2d_pack<true, true, true><<<grid, 128, 0, st>>>(im0, nrm, s2d0, img0, H, W, img_cs, img_co);
        else if (image_is_u8)
            pvnet::k_s2d_pack<true, true><<<grid, 128, 0, st>>>(im0, nrm, s2d0, img0, H, W, img_cs, img_co);
        else if (half)
            pvnet::k_s2d_pack<false, true, true><<<grid, 128, 0, st>>>(im0, nrm, s2d0, img0, H, W, img_cs, img_co);
        else
            pvnet::k_s2d_pack<false, true><<<grid, 128, 0, st>>>(im0, nrm, s2d0, img0, H, W, img_cs, img_co);
        PV_LAUNCHED("k_s2d_pack");
    }
    // the 7x7/2 convolution as the 4x4 stride-1 convolution on S (taps at offsets -2..1): the eval path's instantiation
    return pvnet_conv2d_nhwc(s2d, 16, 0, 16, w_s2d, bias, nullptr, 0, 0, out, 64, 0, 64, b, H / 2, W / 2, 4, 1, 1, 0,
                             0, stream);
}

extern "C" {

int pvnet_stem_s2d_nhwc(const void *image, int image_is_u8, const float *mean3, const float *std3, const float *w_s2d,
                        const float *bias, float *s2d, float *out, float *img, int img_cs, int img_co, int b, int H,
                        int W, pvnet_stream_t stream)
{
    return stem_s2d(image, image_is_u8, mean3, std3, w_s2d, bias, s2d, out, img, img_cs, img_co, b, H, W, 0, stream);
}

int pvnet_stem_s2d_half_nhwc(const void *image, int image_is_u8, const float *mean3, const float *std3,
                             const float *w_s2d, const float *bias, float *s2d, float *out, float *img, int img_cs,
                             int img_co, int b, int H, int W, pvnet_stream_t stream)
{
    return stem_s2d(image, image_is_u8, mean3, std3, w_s2d, bias, s2d, out, img, img_cs, img_co, b, H, W, 1, stream);
}

}  // extern "C"

namespace pvnet {

// ------------------------------------------------------------------ head
// convraw.3: 1x1 conv raw_dim (CIN = 32 or 64) -> seg_dim+ver_dim with bias (model_repository.py:57), in
// exact fp32, fused with torch.argmax(seg_pred,1) (tools/demo.py:52; first maximum wins).
// in NHWC [b,H,W,CIN] -> out NCHW [b,Cout,H,W]; mask int64 [b,H,W] (or u8) optional.
constexpr int HEAD_MAX_COUT = 64;
template <int CIN>
__global__ void __launch_bounds__(256)
    k_head(const float *__restrict__ in, const float *__restrict__ w /*[Cout][CIN]*/, const float *__restrict__ bias,
           float *__restrict__ out, void *__restrict__ mask, int mask_esz, int seg_dim, int Cout, int npix,
           long long total, int nhwc)
{
    __shared__ float sw[HEAD_MAX_COUT * CIN];
    __shared__ float sb[HEAD_MAX_COUT];
    for (int i = threadIdx.x; i < Cout * CIN; i += 256) sw[i] = w[i];
    for (int i = threadIdx.x; i < Cout; i += 256) sb[i] = bias[i];
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const long long n = i / npix;
    const long long p = i - n * npix;
    float v[CIN];
    const float4 *src = reinterpret_cast<const float4 *>(in + i * CIN);
#pragma unroll
    for (int j = 0; j < CIN / 4; ++j) {
        const float4 t = __ldg(src + j);
        v[4 * j] = t.x;
        v[4 * j + 1] = t.y;
        v[4 * j + 2] = t.z;
        v[4 * j + 3] = t.w;
    }
    float best = -INFINITY;
    int best_c = 0;
    float *o = nhwc ? out + i * Cout : out + n * Cout * (long long)npix + p;
    const long long ostride = nhwc ? 1 : npix;
    for (int co = 0; co < Cout; ++co) {
        float acc = sb[co];
        const float *wr = sw + co * CIN;
#pragma unroll
        for (int j = 0; j < CIN; ++j) acc = fmaf(v[j], wr[j], acc);
        o[(long long)co * ostride] = acc;
        if (co < seg_dim && acc > best) {
            best = acc;
            best_c = co;
        }
    }
    if (mask) {
        if (mask_esz == 8)
            reinterpret_cast<long long *>(mask)[i] = best_c;
        else
            reinterpret_cast<unsigned char *>(mask)[i] = (unsigned char)best_c;
    }
}

int launch_head(const float *in, int cin, const float *w, const float *bias, float *out, void *mask, int mask_esz,
                int seg_dim, int Cout, int b, int H, int W, int nhwc, cudaStream_t s)
{
    PV_CHECK_ARG(Cout >= 1 && Cout <= HEAD_MAX_COUT, "head: %d output channels unsupported (max %d)", Cout,
                 HEAD_MAX_COUT);
    PV_CHECK_ARG(cin == 32 || cin == 64, "head: %d input channels unsupported (32 or 64)", cin);
    const long long total = (long long)b * H * W;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (cin == 32)
        k_head<32><<<grid, 256, 0, s>>>(in, w, bias, out, mask, mask_esz, seg_dim, Cout, H * W, total, nhwc);
    else
        k_head<64><<<grid, 256, 0, s>>>(in, w, bias, out, mask, mask_esz, seg_dim, Cout, H * W, total, nhwc);
    PV_LAUNCHED("k_head");
    return PVNET_OK;
}

}  // namespace pvnet
