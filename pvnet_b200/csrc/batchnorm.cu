// batchnorm.cu -- train-mode BatchNorm2d on NHWC fp32, fused with its activation and the BasicBlock residual add
// (lib/networks/resnet.py BasicBlock, model_repository.py's conv -> BatchNorm2d -> ReLU/LeakyReLU(0.1) sequences).
//
// Forms (include/pvnet_b200.h, DESIGN.md §16):
//   0  y = act(bn(x))                 act: none, ReLU, LeakyReLU(0.1)
//   1  y = relu(bn(x) + z)            identity block tail, z the skip
//   2  y = relu(bn(x) + bn_z(z))      downsample block tail, z the downsample convolution's output
// bn(v) = fma(v, scale, shift) in fp32, scale = fp32(gamma*invstd), shift = fp32(beta - mean*scale).
//
// Statistics and the backward's sums are fp64 over a fixed partition of the pixels: partial j sums pixels
// [j*BN_CHUNK, (j+1)*BN_CHUNK) in ascending order, and one block per channel merges the partials with 256 lanes (lane t
// takes partials t, t+256, ... ascending) and a fixed halving tree.  Nothing depends on the SM count or the grid, so
// results are identical run to run; oracle/bn_train_oracle.py restates the order.  Every fp64 operation is an explicit
// _rn intrinsic, so no contraction changes a bit.  No atomics, no allocation, no synchronisation.
#include "common.cuh"

namespace pvnet {
namespace {

constexpr int BN_CHUNK = 256;     // pixels per partial sum
constexpr int BN_LANES = 256;     // threads merging one channel's partials (the tree below assumes a power of two)
constexpr int BN_THREADS = 256;   // reduce-pass block size target (channel quads x partial slots)
// Channel limits per form.  act(bn(x)) keeps its contract of up to 1024 channels.  The block tails take 2048:
// Resnet50_8s's layer4 ends every Bottleneck in bn3 + skip (form 1) or bn3 + the downsample's BatchNorm (form 2) at
// 2048 channels, while no BatchNorm outside a block tail of the three networks is wider than 512.
constexpr int BN_MAX_C = 1024;
constexpr int BN_MAX_C_TAIL = 2048;

int max_channels(int form) { return form == 0 ? BN_MAX_C : BN_MAX_C_TAIL; }

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2 };

// one BatchNorm as the kernels see it
struct BnDev {
    const float *weight, *bias;
    float *running_mean, *running_var;
    double *saved;                 // [3][C]: mean, biased variance, invstd
    float *coef;                   // [2][C]: scale, shift
    double factor, eps;
    int batch_stats;
};

template <int ACT>
__device__ __forceinline__ float act_fwd(float v)
{
    if (ACT == ACT_RELU) return v <= 0.f ? 0.f : v;             // NaN passes, as torch's relu
    if (ACT == ACT_LEAKY) return v > 0.f ? v : __fmul_rn(v, 0.1f);
    return v;
}

// dy * act'(pre), act' from the sign of the pre-activation value: torch's threshold_backward(result <= 0 -> 0) and
// leaky_relu_backward(result > 0 ? dy : dy * 0.1f) on the result, which has the sign of `pre`
template <int ACT>
__device__ __forceinline__ float act_bwd(float dy, float pre)
{
    if (ACT == ACT_RELU) return pre <= 0.f ? 0.f : dy;
    if (ACT == ACT_LEAKY) return pre > 0.f ? dy : __fmul_rn(dy, 0.1f);
    return dy;
}

// the forward's pre-activation value of one element, in the module graph's rounding sequence
template <int FORM>
__device__ __forceinline__ float pre_act(float x, float z, float s, float t, float sz, float tz)
{
    float v = __fmaf_rn(x, s, t);
    if (FORM == 1) v = __fadd_rn(v, z);
    if (FORM == 2) v = __fadd_rn(v, __fmaf_rn(z, sz, tz));
    return v;
}

// blockIdx.x read afresh: the fp64 division/sqrt slow paths are subroutine calls, and a block index kept live across
// them would be spilled
__device__ __forceinline__ int block_x()
{
    int v;
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(v));
    return v;
}

__device__ __forceinline__ float f4(const float4 &v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// The reduce passes: a block holds R partials of Qb channel quads (thread t: quad blockIdx.y * Qb + t % Qb, partial
// blockIdx.x * R + t / Qb).  Up to 1024 channels one block row covers all Q quads (Qb = Q, gridDim.y = 1); wider layers
// spread their quads over gridDim.y rows of BN_THREADS.  Which thread sums a partial changes nothing in its order.
__device__ __forceinline__ int quad_of(int Qb) { return blockIdx.y * Qb + threadIdx.x % Qb; }

// ------------------------------------------------------------------ statistics: fp64 shifted sums per partial
// part[k][c][j], k = 0: sum (x - K_c), k = 1: sum (x - K_c)^2, K_c = x[pixel 0][c]
__global__ void __launch_bounds__(BN_THREADS) k_bn_stats_partial(const float *__restrict__ x, long long npix, int Q, int Qb,
                                                                 int R, long long P, double *__restrict__ part)
{
    const int q = quad_of(Qb), r = threadIdx.x / Qb;
    if (q >= Q) return;
    const long long j = (long long)blockIdx.x * R + r;
    if (j >= P) return;
    const float4 *x4 = reinterpret_cast<const float4 *>(x);
    const float4 k4 = __ldg(x4 + q);
    const double K[4] = {k4.x, k4.y, k4.z, k4.w};
    double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
    const long long p0 = j * BN_CHUNK, p1 = min(p0 + BN_CHUNK, npix);
    const float4 *src = x4 + p0 * Q + q;
#pragma unroll 8
    for (long long p = p0; p < p1; ++p, src += Q) {
        const float4 v = __ldg(src);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double d = __dadd_rn((double)f4(v, i), -K[i]);
            s1[i] = __dadd_rn(s1[i], d);
            s2[i] = __dadd_rn(s2[i], __dmul_rn(d, d));
        }
    }
    const long long C = 4LL * Q;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long c = 4LL * q + i;
        part[c * P + j] = s1[i];
        part[(C + c) * P + j] = s2[i];
    }
}

// lanes t = 0..255 sum partials t, t+256, ... ascending; then lane[i] += lane[i+s] for s = 128, 64, ..., 1
__device__ double merge_partials(const double *__restrict__ p, long long P, double *sh)
{
    double acc = 0.0;
    for (long long k = threadIdx.x; k < P; k += BN_LANES) acc = __dadd_rn(acc, p[k]);
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int s = BN_LANES / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
        __syncthreads();
    }
    const double v = sh[0];
    __syncthreads();
    return v;
}

// one block per channel: the batch statistics (or the running ones), scale/shift and the running-stat update
__global__ void __launch_bounds__(BN_LANES) k_bn_finalize(const float *__restrict__ x, const double *__restrict__ part,
                                                          long long P, long long npix, int C, BnDev bn)
{
    __shared__ double sh[BN_LANES];
    int c = blockIdx.x;
    double S1 = 0.0, S2 = 0.0;
    if (bn.batch_stats) {
        S1 = merge_partials(part + (long long)c * P, P, sh);
        S2 = merge_partials(part + (long long)(C + c) * P, P, sh);
    }
    if (threadIdx.x != 0) return;
    const double N = (double)npix, rN = __drcp_rn(N);
    double mean, var;
    if (bn.batch_stats) {
        const double m = __dmul_rn(S1, rN);
        mean = __dadd_rn((double)x[c], m);
        var = fmax(__dadd_rn(__dmul_rn(S2, rN), -__dmul_rn(m, m)), 0.0);
    } else {
        mean = (double)bn.running_mean[c];
        var = (double)bn.running_var[c];
    }
    const double gamma = bn.weight ? (double)bn.weight[c] : 1.0, beta = bn.bias ? (double)bn.bias[c] : 0.0;
    const float rm = bn.running_mean ? bn.running_mean[c] : 0.f, rv = bn.running_var ? bn.running_var[c] : 0.f;
    const double invstd = __drcp_rn(__dsqrt_rn(__dadd_rn(var, bn.eps)));
    const float scale = (float)__dmul_rn(gamma, invstd);
    const float shift = (float)__dadd_rn(beta, -__dmul_rn(mean, (double)scale));
    const float unbiased = (float)__dmul_rn(__dmul_rn(var, N), __drcp_rn(N - 1.0));
    c = block_x();
    bn.saved[c] = mean;
    bn.saved[C + c] = var;
    bn.saved[2 * C + c] = invstd;
    bn.coef[c] = scale;
    bn.coef[C + c] = shift;
    if (bn.batch_stats && bn.running_mean) {
        // nn.BatchNorm2d's rule in fp32: r <- (1 - f) * r + f * stat, running_var from the unbiased variance
        const float omf = (float)(1.0 - bn.factor), f = (float)bn.factor;
        bn.running_mean[c] = __fadd_rn(__fmul_rn(rm, omf), __fmul_rn((float)mean, f));
        bn.running_var[c] = __fadd_rn(__fmul_rn(rv, omf), __fmul_rn(unbiased, f));
    }
}

// ------------------------------------------------------------------ apply: one streaming pass, float4
template <int FORM, int ACT>
__global__ void __launch_bounds__(256) k_bn_apply(const float4 *__restrict__ x, const float4 *__restrict__ z,
                                                  long long nvec, int Q, const float *__restrict__ coef,
                                                  const float *__restrict__ coef_z, float4 *__restrict__ y)
{
    const float4 *S = reinterpret_cast<const float4 *>(coef), *T = S + Q;
    const float4 *Sz = reinterpret_cast<const float4 *>(coef_z), *Tz = Sz + Q;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(v % Q);
        const float4 a = x[v], s = __ldg(S + q), t = __ldg(T + q);
        float4 b = make_float4(0.f, 0.f, 0.f, 0.f), sz = b, tz = b;
        if (FORM != 0) b = z[v];
        if (FORM == 2) sz = __ldg(Sz + q), tz = __ldg(Tz + q);
        float4 o;
        o.x = act_fwd<ACT>(pre_act<FORM>(a.x, b.x, s.x, t.x, sz.x, tz.x));
        o.y = act_fwd<ACT>(pre_act<FORM>(a.y, b.y, s.y, t.y, sz.y, tz.y));
        o.z = act_fwd<ACT>(pre_act<FORM>(a.z, b.z, s.z, t.z, sz.z, tz.z));
        o.w = act_fwd<ACT>(pre_act<FORM>(a.w, b.w, s.w, t.w, sz.w, tz.w));
        y[v] = o;
    }
}

// ------------------------------------------------------------------ backward
// g = dy * act'(pre).  part[k][c][j]: k = 0 sum g, 1 sum g*(x - mean), 2 (form 2) sum g*(z - mean_z), fp64, in the
// statistics' partition
template <int FORM, int ACT>
__global__ void __launch_bounds__(BN_THREADS) k_bn_backward_reduce(const float *__restrict__ dy, const float *__restrict__ x,
                                                             const float *__restrict__ z, long long npix, int Q, int Qb,
                                                             int R, long long P, BnDev bn, BnDev bz,
                                                             double *__restrict__ part)
{
    const int q = quad_of(Qb), r = threadIdx.x / Qb;
    if (q >= Q) return;
    const long long j = (long long)blockIdx.x * R + r;
    if (j >= P) return;
    const int C = 4 * Q;
    const float4 s = __ldg(reinterpret_cast<const float4 *>(bn.coef) + q);
    const float4 t = __ldg(reinterpret_cast<const float4 *>(bn.coef + C) + q);
    float4 sz = make_float4(0.f, 0.f, 0.f, 0.f), tz = sz;
    double mz[4] = {0.0, 0.0, 0.0, 0.0};
    if (FORM == 2) {
        sz = __ldg(reinterpret_cast<const float4 *>(bz.coef) + q);
        tz = __ldg(reinterpret_cast<const float4 *>(bz.coef + C) + q);
#pragma unroll
        for (int i = 0; i < 4; ++i) mz[i] = bz.saved[4 * q + i];
    }
    double mx[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) mx[i] = bn.saved[4 * q + i];
    double sg[4] = {0.0, 0.0, 0.0, 0.0}, sgx[4] = {0.0, 0.0, 0.0, 0.0}, sgz[4] = {0.0, 0.0, 0.0, 0.0};
    const long long p0 = j * BN_CHUNK, p1 = min(p0 + BN_CHUNK, npix);
    const long long off0 = p0 * Q + q;
    const float4 *dy4 = reinterpret_cast<const float4 *>(dy) + off0, *x4 = reinterpret_cast<const float4 *>(x) + off0;
    const float4 *z4 = FORM != 0 ? reinterpret_cast<const float4 *>(z) + off0 : nullptr;
#pragma unroll 4
    for (long long p = p0; p < p1; ++p, dy4 += Q, x4 += Q) {
        const float4 gv = __ldg(dy4), xv = __ldg(x4);
        float4 zv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (FORM != 0) {
            zv = __ldg(z4);
            z4 += Q;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float xi = f4(xv, i), zi = f4(zv, i);
            const double g = (double)act_bwd<ACT>(f4(gv, i), pre_act<FORM>(xi, zi, f4(s, i), f4(t, i), f4(sz, i),
                                                                             f4(tz, i)));
            sg[i] = __dadd_rn(sg[i], g);
            sgx[i] = __dadd_rn(sgx[i], __dmul_rn(g, __dadd_rn((double)xi, -mx[i])));
            if (FORM == 2) sgz[i] = __dadd_rn(sgz[i], __dmul_rn(g, __dadd_rn((double)zi, -mz[i])));
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long c = 4LL * q + i;
        part[c * P + j] = sg[i];
        part[(C + c) * P + j] = sgx[i];
        if (FORM == 2) part[(2LL * C + c) * P + j] = sgz[i];
    }
}

// dx = A*g + B*x + Cc per channel (fp32 coefficients, each rounded once from fp64), dgamma = invstd * sum g*(x-mean),
// dbeta = sum g.  Batch statistics: A = gamma*invstd, B = -A*invstd^2*Sgx/N, Cc = -A*Sg/N - B*mean; running
// statistics (frozen module): A = gamma*invstd, B = Cc = 0.
__device__ void bn_backward_coef(const BnDev &bn, int C, int c, double rN, double Sg, double Sgx, float *abc,
                                 float *dweight, float *dbias)
{
    const double invstd = bn.saved[2 * C + c], mean = bn.saved[c];
    const double gamma = bn.weight ? (double)bn.weight[c] : 1.0;
    const double A = __dmul_rn(gamma, invstd);
    double B = 0.0, Cc = 0.0;
    if (bn.batch_stats) {
        B = -__dmul_rn(__dmul_rn(A, __dmul_rn(invstd, invstd)), __dmul_rn(Sgx, rN));
        Cc = __dadd_rn(-__dmul_rn(A, __dmul_rn(Sg, rN)), -__dmul_rn(B, mean));
    }
    abc[c] = (float)A;
    abc[C + c] = (float)B;
    abc[2 * C + c] = (float)Cc;
    if (dweight) dweight[c] = (float)__dmul_rn(Sgx, invstd);
    if (dbias) dbias[c] = (float)Sg;
}

__global__ void __launch_bounds__(BN_LANES) k_bn_backward_finalize(const double *__restrict__ part, long long P,
                                                                   long long npix, int C, int nz, BnDev bn, BnDev bz,
                                                                   float *abc, float *abc_z, float *dweight,
                                                                   float *dbias, float *dweight_z, float *dbias_z)
{
    __shared__ double sh[BN_LANES];
    const int c = blockIdx.x;
    const double rN = __drcp_rn((double)npix);
    const double Sg = merge_partials(part + (long long)c * P, P, sh);
    const double Sgx = merge_partials(part + (long long)(C + c) * P, P, sh);
    const double Sgz = nz ? merge_partials(part + (long long)(2 * C + c) * P, P, sh) : 0.0;
    if (threadIdx.x != 0) return;
    bn_backward_coef(bn, C, c, rN, Sg, Sgx, abc, dweight, dbias);
    if (nz) bn_backward_coef(bz, C, c, rN, Sg, Sgz, abc_z, dweight_z, dbias_z);
}

// dx = A*g + B*x + Cc; form 1 writes dz = g (the skip's gradient), form 2 dz = A_z*g + B_z*z + Cc_z
template <int FORM, int ACT>
__global__ void __launch_bounds__(256) k_bn_backward_apply(const float4 *__restrict__ dy, const float4 *__restrict__ x,
                                                           const float4 *__restrict__ z, long long nvec, int Q,
                                                           const float *__restrict__ coef,
                                                           const float *__restrict__ coef_z,
                                                           const float *__restrict__ abc,
                                                           const float *__restrict__ abc_z, float4 *__restrict__ dx,
                                                           float4 *__restrict__ dz)
{
    const float4 *S = reinterpret_cast<const float4 *>(coef), *T = S + Q;
    const float4 *Sz = reinterpret_cast<const float4 *>(coef_z), *Tz = Sz + Q;
    const float4 *A = reinterpret_cast<const float4 *>(abc), *B = A + Q, *Cc = B + Q;
    const float4 *Az = reinterpret_cast<const float4 *>(abc_z), *Bz = Az + Q, *Cz = Bz + Q;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(v % Q);
        const float4 gv = dy[v], xv = x[v], s = __ldg(S + q), t = __ldg(T + q);
        const float4 a = __ldg(A + q), b = __ldg(B + q), cc = __ldg(Cc + q);
        float4 zv = make_float4(0.f, 0.f, 0.f, 0.f), sz = zv, tz = zv;
        if (FORM != 0) zv = z[v];
        if (FORM == 2) sz = __ldg(Sz + q), tz = __ldg(Tz + q);
        float g[4], o[4], oz[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            g[i] = act_bwd<ACT>(f4(gv, i), pre_act<FORM>(f4(xv, i), f4(zv, i), f4(s, i), f4(t, i), f4(sz, i), f4(tz, i)));
            o[i] = __fmaf_rn(f4(a, i), g[i], __fmaf_rn(f4(b, i), f4(xv, i), f4(cc, i)));
        }
        dx[v] = make_float4(o[0], o[1], o[2], o[3]);
        if (FORM == 1) dz[v] = make_float4(g[0], g[1], g[2], g[3]);
        if (FORM == 2) {
            const float4 az = __ldg(Az + q), bz = __ldg(Bz + q), cz = __ldg(Cz + q);
#pragma unroll
            for (int i = 0; i < 4; ++i) oz[i] = __fmaf_rn(f4(az, i), g[i], __fmaf_rn(f4(bz, i), f4(zv, i), f4(cz, i)));
            dz[v] = make_float4(oz[0], oz[1], oz[2], oz[3]);
        }
    }
}

// ------------------------------------------------------------------ host side
struct Partition {
    int Q, Qb, R;
    long long P;
    dim3 grid;
};

Partition partition(int C, long long npix)
{
    Partition p;
    p.Q = C / 4;
    p.Qb = p.Q < BN_THREADS ? p.Q : BN_THREADS;
    p.R = BN_THREADS / p.Qb;
    p.P = (npix + BN_CHUNK - 1) / BN_CHUNK;
    p.grid = dim3((unsigned)((p.P + p.R - 1) / p.R), (unsigned)((p.Q + p.Qb - 1) / p.Qb));
    return p;
}

int nsums(int form) { return form == 2 ? 4 : 2; }

size_t workspace_bytes(int form, int C, long long npix)
{
    const Partition p = partition(C, npix);
    return align_up((size_t)nsums(form) * C * p.P * sizeof(double), 256) + 2 * align_up(3 * (size_t)C * sizeof(float), 256);
}

bool aligned16(const void *p) { return (uintptr_t)p % 16 == 0; }

int check_common(const char *what, int form, int act, const float *x, const float *z, long long npix, int C,
                 const pvnet_batchnorm_t *bn, const pvnet_batchnorm_t *bz, void *ws, size_t ws_bytes)
{
    PV_CHECK_ARG(form >= 0 && form <= 2, "%s: form must be 0, 1 or 2, got %d", what, form);
    PV_CHECK_ARG(act >= 0 && act <= 2, "%s: act must be 0 (none), 1 (ReLU) or 2 (LeakyReLU), got %d", what, act);
    PV_CHECK_ARG(form == 0 || act == ACT_RELU, "%s: the block tails (forms 1, 2) end in ReLU", what);
    PV_CHECK_ARG(C > 0 && C % 4 == 0 && C <= max_channels(form),
                 "%s: C must be a positive multiple of 4 up to %d (form %d), got %d", what, max_channels(form), form, C);
    PV_CHECK_ARG(npix > 0, "%s: the pixel count must be positive", what);
    // element offsets are 64-bit throughout; the grid of the reduce passes is what bounds the size
    PV_CHECK_ARG((npix + BN_CHUNK - 1) / BN_CHUNK < (1LL << 31) && npix <= (1LL << 62) / C,
                 "%s: tensor too large (%lld pixels x %d channels)", what, npix, C);
    PV_CHECK_ARG(x && bn, "%s: null x or BatchNorm", what);
    PV_CHECK_ARG(form == 0 || z, "%s: forms 1 and 2 need z", what);
    PV_CHECK_ARG(form != 2 || bz, "%s: form 2 needs the second BatchNorm", what);
    PV_CHECK_ARG(aligned16(x) && (!z || aligned16(z)), "%s: tensors must be 16-byte aligned", what);
    for (const pvnet_batchnorm_t *b : {bn, form == 2 ? bz : nullptr}) {
        if (!b) continue;
        PV_CHECK_ARG(b->saved && b->coef && aligned16(b->coef), "%s: null (or misaligned) saved/coef buffers", what);
        PV_CHECK_ARG(b->batch_stats || (b->running_mean && b->running_var),
                     "%s: normalising with running statistics needs running_mean and running_var", what);
        PV_CHECK_ARG(!b->batch_stats || npix > 1 || !b->running_mean,
                     "%s: batch statistics with a running-stat update need more than one value per channel", what);
        PV_CHECK_ARG(b->eps > 0.0, "%s: eps must be positive", what);
    }
    PV_CHECK_ARG(ws && ws_bytes >= workspace_bytes(form, C, npix), "%s: workspace of %zu bytes, %zu needed", what,
                 ws_bytes, workspace_bytes(form, C, npix));
    return PVNET_OK;
}

BnDev to_dev(const pvnet_batchnorm_t *b)
{
    BnDev d{};
    if (!b) return d;
    d.weight = b->weight;
    d.bias = b->bias;
    d.running_mean = b->running_mean;
    d.running_var = b->running_var;
    d.saved = b->saved;
    d.coef = b->coef;
    d.factor = b->factor;
    d.eps = b->eps;
    d.batch_stats = b->batch_stats;
    return d;
}

unsigned stream_blocks(long long nvec)
{
    const long long want = (nvec + 255) / 256, cap = (long long)sm_count() * 16;
    return (unsigned)(want < cap ? want : cap);
}

template <int FORM, int ACT>
void launch_apply(const float *x, const float *z, long long nvec, int Q, const float *coef, const float *coef_z,
                  float *y, cudaStream_t st)
{
    k_bn_apply<FORM, ACT><<<stream_blocks(nvec), 256, 0, st>>>(
        reinterpret_cast<const float4 *>(x), reinterpret_cast<const float4 *>(z), nvec, Q, coef, coef_z,
        reinterpret_cast<float4 *>(y));
}

template <int FORM, int ACT>
void launch_backward(const float *dy, const float *x, const float *z, long long npix, const Partition &pt,
                     const BnDev &bn, const BnDev &bz, double *part, const float *abc, const float *abc_z, float *dx,
                     float *dz, cudaStream_t st, bool reduce)
{
    if (reduce) {
        k_bn_backward_reduce<FORM, ACT><<<pt.grid, pt.Qb * pt.R, 0, st>>>(dy, x, z, npix, pt.Q, pt.Qb, pt.R, pt.P, bn,
                                                                           bz, part);
        return;
    }
    const long long nvec = npix * pt.Q;
    k_bn_backward_apply<FORM, ACT><<<stream_blocks(nvec), 256, 0, st>>>(
        reinterpret_cast<const float4 *>(dy), reinterpret_cast<const float4 *>(x),
        reinterpret_cast<const float4 *>(z), nvec, pt.Q, bn.coef, bz.coef, abc, abc_z,
        reinterpret_cast<float4 *>(dx), reinterpret_cast<float4 *>(dz));
}

// (form, act) -> one instantiation; forms 1 and 2 are ReLU only
#define PV_BN_DISPATCH(form, act, F, ...)                                  \
    do {                                                                   \
        if (form == 0 && act == ACT_NONE) F<0, ACT_NONE>(__VA_ARGS__);     \
        else if (form == 0 && act == ACT_RELU) F<0, ACT_RELU>(__VA_ARGS__); \
        else if (form == 0) F<0, ACT_LEAKY>(__VA_ARGS__);                  \
        else if (form == 1) F<1, ACT_RELU>(__VA_ARGS__);                   \
        else F<2, ACT_RELU>(__VA_ARGS__);                                  \
    } while (0)

}  // namespace
}  // namespace pvnet

extern "C" {

int pvnet_batchnorm_workspace_bytes(int form, int C, long long npix, size_t *bytes)
{
    PV_CHECK_ARG(bytes, "batchnorm workspace: null output");
    PV_CHECK_ARG(form >= 0 && form <= 2 && C > 0 && C % 4 == 0 && C <= pvnet::max_channels(form) && npix > 0,
                 "batchnorm workspace: form must be 0, 1 or 2, C a positive multiple of 4 up to %d (form 0) or %d "
                 "(forms 1, 2) and the pixel count positive (form %d, C %d, %lld pixels)", pvnet::BN_MAX_C,
                 pvnet::BN_MAX_C_TAIL, form, C, npix);
    *bytes = pvnet::workspace_bytes(form, C, npix);
    return PVNET_OK;
}

int pvnet_batchnorm_act_forward(int form, int act, const float *x, const float *z, long long npix, int C,
                                const pvnet_batchnorm_t *bn, const pvnet_batchnorm_t *bn_z, float *y, void *workspace,
                                size_t workspace_bytes, pvnet_stream_t stream)
{
    using namespace pvnet;
    if (int rc = check_common("batchnorm forward", form, act, x, z, npix, C, bn, bn_z, workspace, workspace_bytes))
        return rc;
    PV_CHECK_ARG(y && aligned16(y), "batchnorm forward: null or misaligned output");
    const cudaStream_t st = (cudaStream_t)stream;
    const Partition pt = partition(C, npix);
    double *part = static_cast<double *>(workspace);
    const BnDev d = to_dev(bn), dz = form == 2 ? to_dev(bn_z) : BnDev{};
    const float *xs[2] = {x, z};
    const BnDev *ds[2] = {&d, &dz};
    for (int k = 0; k < (form == 2 ? 2 : 1); ++k) {
        double *pk = part + (size_t)k * 2 * C * pt.P;
        if (ds[k]->batch_stats) {
            k_bn_stats_partial<<<pt.grid, pt.Qb * pt.R, 0, st>>>(xs[k], npix, pt.Q, pt.Qb, pt.R, pt.P, pk);
            PV_LAUNCHED("k_bn_stats_partial");
        }
        k_bn_finalize<<<C, BN_LANES, 0, st>>>(xs[k], pk, pt.P, npix, C, *ds[k]);
        PV_LAUNCHED("k_bn_finalize");
    }
    PV_BN_DISPATCH(form, act, launch_apply, x, z, npix * pt.Q, pt.Q, d.coef, dz.coef, y, st);
    PV_LAUNCHED("k_bn_apply");
    return PVNET_OK;
}

int pvnet_batchnorm_act_backward(int form, int act, const float *dy, const float *x, const float *z, long long npix,
                                 int C, const pvnet_batchnorm_t *bn, const pvnet_batchnorm_t *bn_z, float *dx,
                                 float *dz, float *dweight, float *dbias, float *dweight_z, float *dbias_z,
                                 void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    using namespace pvnet;
    if (int rc = check_common("batchnorm backward", form, act, x, z, npix, C, bn, bn_z, workspace, workspace_bytes))
        return rc;
    PV_CHECK_ARG(dy && dx && aligned16(dy) && aligned16(dx), "batchnorm backward: null or misaligned dy/dx");
    PV_CHECK_ARG(form == 0 || (dz && aligned16(dz)), "batchnorm backward: forms 1 and 2 need an aligned dz");
    const cudaStream_t st = (cudaStream_t)stream;
    const Partition pt = partition(C, npix);
    double *part = static_cast<double *>(workspace);
    float *abc = reinterpret_cast<float *>(static_cast<char *>(workspace) +
                                           align_up((size_t)nsums(form) * C * pt.P * sizeof(double), 256));
    float *abc_z = abc + align_up(3 * (size_t)C * sizeof(float), 256) / sizeof(float);
    const BnDev d = to_dev(bn), dzb = form == 2 ? to_dev(bn_z) : BnDev{};
    PV_BN_DISPATCH(form, act, launch_backward, dy, x, z, npix, pt, d, dzb, part, abc, abc_z, dx, dz, st, true);
    PV_LAUNCHED("k_bn_backward_reduce");
    k_bn_backward_finalize<<<C, BN_LANES, 0, st>>>(part, pt.P, npix, C, form == 2, d, dzb, abc, abc_z, dweight, dbias,
                                                   form == 2 ? dweight_z : nullptr, form == 2 ? dbias_z : nullptr);
    PV_LAUNCHED("k_bn_backward_finalize");
    PV_BN_DISPATCH(form, act, launch_backward, dy, x, z, npix, pt, d, dzb, part, abc, abc_z, dx, dz, st, false);
    PV_LAUNCHED("k_bn_backward_apply");
    return PVNET_OK;
}

}  // extern "C"
