// head3x3.cu -- the score heads of Resnet18_8s_detector and Resnet18_8s_detector_v2 (model_repository.py:302-331):
// a 3x3 convolution, padding 1, dilation 1, with bias and ONE output channel (fc = Conv2d(512, 1, 3, 1, 1) on
// layer4's output; out_conv = Conv2d(128, 1, 3, 1, 1) on layer2's output).  One output channel gives wgmma N = 1, so
// these are direct fp32 / fp64 kernels in the spirit of k_head.  The same forward serves the eval plan (ST_SCORE in
// backbone.cu, on the TF32 trunk's output) and forward_train (on the unrounded activations).
//
// Layouts: x NHWC [b,H,W,C] dense (C a multiple of 32, at most 512), w [9][C] (tap t = ky*3 + kx, the torch weight
// [1,C,3,3] permuted), out / dout [b,1,H,W] = [b][H][W].
//
// Forward.  out[n,y,x] is ONE fp32 fmaf chain from bias[0]: for each 32-channel chunk c0 ascending, for each tap t
// ascending, for each channel c of the chunk ascending, acc = fmaf(w[t][c], x[n, y+ky-1, x+kx-1, c], acc); a tap
// whose neighbour lies outside the image is skipped.
// Data gradient.  dx[n,y,x,c] = fmaf chain from 0 over t ascending of w[t][c] * dout[n, y+1-ky, x+1-kx], taps
// outside the image skipped.
// Weight and bias gradients.  dw[t][c] = sum_p dout[p] * x[p + (ky-1, kx-1)][c] and db = sum_p dout[p] in fp64 (the
// fp32 x fp32 products are exact): per H3_CHUNK-pixel partial, pixels ascending (flat index (n*H + y)*W + x); the
// partials are merged by train_layers.cu's k_head_train_reduce (lanes, then a halving tree) and rounded once to fp32.
// No atomics and nothing depends on the grid or the SM count.
#include "conv_tc.cuh"

namespace pvnet {

// train_layers.cu: one block of HEAD_LANES (256) threads per item; items < ndw go to dw[item], the rest to db
__global__ void k_head_train_reduce(const double *__restrict__ part, int nparts, int ndw, float *__restrict__ dw,
                                    float *__restrict__ db);

constexpr int H3_MAXC = 512;
constexpr int H3_THREADS = 128;
constexpr int H3_CHUNK = 512;      // pixels per fp64 partial of dw / db (fixed partition)
constexpr int H3_REDUCE_LANES = 256;

__global__ void __launch_bounds__(H3_THREADS)
    k_head3x3(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
              float *__restrict__ out, int H, int W, int C, long long P)
{
    __shared__ __align__(16) float sw[9 * H3_MAXC];
    for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) sw[i] = w[i];
    __syncthreads();
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int xx = (int)(i % W), yy = (int)((i / W) % H);
    const long long n = i / ((long long)H * W);
    float acc = __ldg(bias);
    for (int c0 = 0; c0 < C; c0 += 32) {
#pragma unroll 1
        for (int t = 0; t < 9; ++t) {
            const int sy = yy + t / 3 - 1, sx = xx + t % 3 - 1;
            if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
            const float4 *src = reinterpret_cast<const float4 *>(x + ((n * H + sy) * W + sx) * C + c0);
            const float4 *wr = reinterpret_cast<const float4 *>(sw + t * C + c0);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 v = __ldg(src + j), ww = wr[j];
                acc = __fmaf_rn(ww.x, v.x, acc);
                acc = __fmaf_rn(ww.y, v.y, acc);
                acc = __fmaf_rn(ww.z, v.z, acc);
                acc = __fmaf_rn(ww.w, v.w, acc);
            }
        }
    }
    out[i] = acc;
}

// one thread = one (pixel, channel quad)
__global__ void __launch_bounds__(H3_THREADS)
    k_head3x3_dgrad(const float *__restrict__ dout, const float *__restrict__ w, float *__restrict__ dx, int H, int W,
                    int C, long long items)
{
    const long long it = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (it >= items) return;
    const int cq = C >> 2;
    const long long i = it / cq;
    const int c = 4 * (int)(it - i * cq);
    const int xx = (int)(i % W), yy = (int)((i / W) % H);
    const long long n = i / ((long long)H * W);
    float a[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 9; ++t) {
        const int sy = yy + 1 - t / 3, sx = xx + 1 - t % 3;
        if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
        const float g = __ldg(dout + (n * H + sy) * W + sx);
        const float4 ww = __ldg(reinterpret_cast<const float4 *>(w + t * C + c));
        a[0] = __fmaf_rn(ww.x, g, a[0]);
        a[1] = __fmaf_rn(ww.y, g, a[1]);
        a[2] = __fmaf_rn(ww.z, g, a[2]);
        a[3] = __fmaf_rn(ww.w, g, a[3]);
    }
    reinterpret_cast<float4 *>(dx + i * C + c)[0] = make_float4(a[0], a[1], a[2], a[3]);
}

// grid (nparts, C / H3_THREADS): one thread = one channel of one H3_CHUNK-pixel partial, its 9 tap sums (and, for
// channel 0, the bias sum) -> part[(t*C + c) * nparts + chunk], part[(9*C) * nparts + chunk]
__global__ void __launch_bounds__(H3_THREADS)
    k_head3x3_wgrad(const float *__restrict__ dout, const float *__restrict__ x, double *__restrict__ part, int H,
                    int W, int C, long long P, int nparts)
{
    const int c = blockIdx.y * H3_THREADS + threadIdx.x;
    if (c >= C) return;
    const long long p0 = (long long)blockIdx.x * H3_CHUNK;
    const long long p1 = min(p0 + H3_CHUNK, P);
    double acc[9], sb = 0.0;
#pragma unroll
    for (int t = 0; t < 9; ++t) acc[t] = 0.0;
    for (long long p = p0; p < p1; ++p) {
        const int xx = (int)(p % W), yy = (int)((p / W) % H);
        const long long n = p / ((long long)H * W);
        const double g = (double)__ldg(dout + p);
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const int sy = yy + t / 3 - 1, sx = xx + t % 3 - 1;
            if (sy < 0 || sy >= H || sx < 0 || sx >= W) continue;
            acc[t] = __fma_rn(g, (double)__ldg(x + ((n * H + sy) * W + sx) * C + c), acc[t]);
        }
        sb = __dadd_rn(sb, g);
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) part[((long long)t * C + c) * nparts + blockIdx.x] = acc[t];
    if (c == 0) part[(long long)9 * C * nparts + blockIdx.x] = sb;
}

static int check_head3x3_args(const char *what, int b, int H, int W, int C)
{
    PV_CHECK_ARG(b > 0 && H > 0 && W > 0, "%s: b, H, W must be positive", what);
    PV_CHECK_ARG(C > 0 && C % 32 == 0 && C <= H3_MAXC, "%s: C %d must be a positive multiple of 32, at most %d",
                 what, C, H3_MAXC);
    PV_CHECK_ARG((long long)b * H * W < (1ll << 40), "%s: too many pixels", what);
    return PVNET_OK;
}

static long long head3x3_nparts(int b, int H, int W) { return ((long long)b * H * W + H3_CHUNK - 1) / H3_CHUNK; }

int launch_head3x3(const float *in, int C, const float *w, const float *bias, float *out, int b, int H, int W,
                   cudaStream_t s)
{
    if (int rc = check_head3x3_args("head3x3", b, H, W, C)) return rc;
    const long long P = (long long)b * H * W;
    k_head3x3<<<(unsigned)((P + H3_THREADS - 1) / H3_THREADS), H3_THREADS, 0, s>>>(in, w, bias, out, H, W, C, P);
    PV_LAUNCHED("k_head3x3");
    return PVNET_OK;
}

}  // namespace pvnet

extern "C" {

int pvnet_head3x3_nchw(const float *x, const float *w, const float *bias, float *out, int b, int H, int W, int C,
                       pvnet_stream_t stream)
{
    PV_CHECK_ARG(x && w && bias && out, "head3x3: null pointer");
    PV_CHECK_ARG((uintptr_t)x % 16 == 0, "head3x3: x must be 16-byte aligned");
    return pvnet::launch_head3x3(x, C, w, bias, out, b, H, W, (cudaStream_t)stream);
}

int pvnet_head3x3_backward_workspace_bytes(int b, int H, int W, int C, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "head3x3 backward: null bytes");
    if (int rc = pvnet::check_head3x3_args("head3x3 backward", b, H, W, C)) return rc;
    *bytes = ((size_t)9 * C + 1) * (size_t)pvnet::head3x3_nparts(b, H, W) * sizeof(double);
    return PVNET_OK;
}

int pvnet_head3x3_backward(const float *dout, const float *x, const float *w, float *dx, float *dw, float *db, int b,
                           int H, int W, int C, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    if (int rc = pvnet::check_head3x3_args("head3x3 backward", b, H, W, C)) return rc;
    PV_CHECK_ARG(dout, "head3x3 backward: null dout");
    PV_CHECK_ARG(!dx || (w && (uintptr_t)w % 16 == 0 && (uintptr_t)dx % 16 == 0),
                 "head3x3 backward: dx needs w, and both must be 16-byte aligned");
    const bool sums = dw || db;
    PV_CHECK_ARG(!sums || x, "head3x3 backward: dw / db need x");
    const long long nparts = pvnet::head3x3_nparts(b, H, W);
    PV_CHECK_ARG(nparts < (1ll << 31), "head3x3 backward: too many pixels");
    const size_t need = ((size_t)9 * C + 1) * (size_t)nparts * sizeof(double);
    PV_CHECK_ARG(!sums || (workspace && workspace_bytes >= need), "head3x3 backward: workspace of %zu bytes, %zu needed",
                 workspace_bytes, need);
    PV_CHECK_ARG(!sums || (uintptr_t)workspace % 16 == 0, "head3x3 backward: workspace must be 16-byte aligned");
    cudaStream_t s = (cudaStream_t)stream;
    const long long P = (long long)b * H * W;
    if (dx) {
        const long long items = P * (C / 4);
        pvnet::k_head3x3_dgrad<<<(unsigned)((items + pvnet::H3_THREADS - 1) / pvnet::H3_THREADS), pvnet::H3_THREADS, 0,
                                 s>>>(dout, w, dx, H, W, C, items);
        PV_LAUNCHED("k_head3x3_dgrad");
    }
    if (sums) {
        double *part = static_cast<double *>(workspace);
        pvnet::k_head3x3_wgrad<<<dim3((unsigned)nparts, (unsigned)(C / pvnet::H3_THREADS + (C % pvnet::H3_THREADS != 0))),
                                 pvnet::H3_THREADS, 0, s>>>(dout, x, part, H, W, C, P, (int)nparts);
        PV_LAUNCHED("k_head3x3_wgrad");
        pvnet::k_head_train_reduce<<<(unsigned)(9 * C + 1), pvnet::H3_REDUCE_LANES, 0, s>>>(part, (int)nparts, 9 * C,
                                                                                           dw, db);
        PV_LAUNCHED("k_head_train_reduce");
    }
    return PVNET_OK;
}

}  // extern "C"
