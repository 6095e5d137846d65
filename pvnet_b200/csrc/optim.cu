// optim.cu -- the optimizer step of a training iteration: Adam over a table of tensors in one multi-tensor launch.
//
// The floating-point sequence is torch.optim.Adam(foreach=False)'s (_single_tensor_adam, amsgrad / maximize /
// capturable / differentiable off) as ATen's CUDA element-wise kernels compute it, written out in DESIGN.md §19 and
// restated in oracle/adam_oracle.py.  Every operation below is an explicit round-to-nearest intrinsic, so the
// compiler's FMA contraction has no say in it.
#include <climits>
#include <cmath>

#include "common.cuh"

namespace pvnet {

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_VEC_PER_THREAD = 2;                                  // float4 per array per thread
constexpr int ADAM_BLOCK_ELEMS = ADAM_THREADS * ADAM_VEC_PER_THREAD * 4;  // 2048 elements per (tensor, block) pair
// Entries of the tensor table one launch carries in the kernel's parameter space: 128 * 48 B + scalars = 6.2 KB, which
// needs the large-parameter launches of CUDA 12.1+ on sm_70+ (limit 32,764 B) and leaves the launch cheap.
constexpr int ADAM_CHUNK_TENSORS = 128;

struct AdamEntry {
    float *p;
    const float *g;
    float *m;
    float *v;
    long long numel;
    int first_block;  // this tensor's first block in the launch's grid
    int vec;          // all four pointers 16-byte aligned: float4 accesses
};

// the step's scalars as fp32, each converted once from the double the host computed (DESIGN.md §19)
struct AdamScalars {
    float wd;         // float(weight_decay); applied only when has_wd
    float w1;         // float(1 - beta1): lerp's weight
    float one_m_w1;   // 1.0f - w1, fp32 subtraction: lerp's |w| >= 0.5 branch
    float b2;         // float(beta2)
    float w2;         // float(1 - beta2)
    float inv_bc2;    // float(1.0 / bias_correction2_sqrt): the reciprocal taken in double, rounded once
    float eps;        // float(eps)
    float neg_step;   // float(-step_size)
    int has_wd;
    int lerp_small;   // |w1| < 0.5f
};

struct AdamChunk {
    AdamEntry e[ADAM_CHUNK_TENSORS];
    AdamScalars s;
    int n;
};

__device__ __forceinline__ void adam_element(float &p, float g, float &m, float &v, const AdamScalars &s)
{
    if (s.has_wd) g = __fmaf_rn(p, s.wd, g);                            // grad.add(param, alpha=wd): g + p*wd, one FMA
    const float d = __fsub_rn(g, m);                                    // lerp: end - self
    m = s.lerp_small ? __fmaf_rn(s.w1, d, m)                            //   self + w*(end - self)
                     : __fmaf_rn(-d, s.one_m_w1, g);                    //   end - (end - self)*(1 - w)
    v = __fmul_rn(v, s.b2);                                             // mul_(beta2)
    v = __fmaf_rn(s.w2, __fmul_rn(g, g), v);                            // addcmul_: v + w2*(g*g), product rounded first
    const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(v), s.inv_bc2), s.eps);  // sqrt() / scalar = * reciprocal; add_(eps)
    p = __fmaf_rn(s.neg_step, __fdiv_rn(m, denom), p);                  // addcdiv_: p + (-step_size)*(m/denom)
}

__global__ void __launch_bounds__(ADAM_THREADS) k_adam_multi_tensor(const __grid_constant__ AdamChunk c)
{
    // the tensor this block belongs to: the last entry whose first_block <= blockIdx.x
    int lo = 0, hi = c.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (c.e[mid].first_block <= (int)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const AdamEntry &e = c.e[lo];
    const long long base = (long long)((int)blockIdx.x - e.first_block) * ADAM_BLOCK_ELEMS;
    const long long left = e.numel - base;
    const int n = left < ADAM_BLOCK_ELEMS ? (int)left : ADAM_BLOCK_ELEMS;
    float *p = e.p + base, *m = e.m + base, *v = e.v + base;
    const float *g = e.g + base;
    int done = 0;
    if (e.vec) {
        const int nvec = n >> 2;
        float4 P[ADAM_VEC_PER_THREAD], G[ADAM_VEC_PER_THREAD], M[ADAM_VEC_PER_THREAD], V[ADAM_VEC_PER_THREAD];
#pragma unroll
        for (int k = 0; k < ADAM_VEC_PER_THREAD; ++k) {
            const int i = threadIdx.x + k * ADAM_THREADS;
            if (i < nvec) {
                P[k] = reinterpret_cast<const float4 *>(p)[i];
                G[k] = __ldcs(reinterpret_cast<const float4 *>(g) + i);   // the gradient is not read again
                M[k] = reinterpret_cast<const float4 *>(m)[i];
                V[k] = reinterpret_cast<const float4 *>(v)[i];
            }
        }
#pragma unroll
        for (int k = 0; k < ADAM_VEC_PER_THREAD; ++k) {
            const int i = threadIdx.x + k * ADAM_THREADS;
            if (i < nvec) {
                adam_element(P[k].x, G[k].x, M[k].x, V[k].x, c.s);
                adam_element(P[k].y, G[k].y, M[k].y, V[k].y, c.s);
                adam_element(P[k].z, G[k].z, M[k].z, V[k].z, c.s);
                adam_element(P[k].w, G[k].w, M[k].w, V[k].w, c.s);
                reinterpret_cast<float4 *>(p)[i] = P[k];
                reinterpret_cast<float4 *>(m)[i] = M[k];
                reinterpret_cast<float4 *>(v)[i] = V[k];
            }
        }
        done = nvec << 2;
    }
    // unaligned tensors, and the last numel % 4 elements of an aligned one
    for (int i = done + threadIdx.x; i < n; i += ADAM_THREADS) {
        float pi = p[i], mi = m[i], vi = v[i];
        adam_element(pi, g[i], mi, vi, c.s);
        p[i] = pi;
        m[i] = mi;
        v[i] = vi;
    }
}

static bool finite_nonneg(double x) { return std::isfinite(x) && x >= 0.0; }

}  // namespace pvnet

extern "C" {

int pvnet_adam_step(const pvnet_adam_tensor_t *tensors, int n_tensors, double lr, double beta1, double beta2,
                    double eps, double weight_decay, int64_t step, pvnet_stream_t stream)
{
    using namespace pvnet;
    PV_CHECK_ARG(n_tensors >= 0, "adam: n_tensors must not be negative, got %d", n_tensors);
    PV_CHECK_ARG(tensors || n_tensors == 0, "adam: null tensor table");
    PV_CHECK_ARG(step >= 1, "adam: step counts from 1 (the value after this step), got %lld", (long long)step);
    PV_CHECK_ARG(finite_nonneg(lr), "adam: lr must be finite and not negative, got %g", lr);
    PV_CHECK_ARG(finite_nonneg(eps), "adam: eps must be finite and not negative, got %g", eps);
    PV_CHECK_ARG(finite_nonneg(weight_decay), "adam: weight_decay must be finite and not negative, got %g",
                 weight_decay);
    PV_CHECK_ARG(beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0,
                 "adam: betas must lie in [0, 1), got %g and %g", beta1, beta2);
    for (int i = 0; i < n_tensors; ++i) {
        const pvnet_adam_tensor_t &t = tensors[i];
        PV_CHECK_ARG(t.numel >= 0, "adam: tensor %d has a negative numel %lld", i, (long long)t.numel);
        if (t.numel == 0) continue;
        PV_CHECK_ARG(t.param && t.grad && t.exp_avg && t.exp_avg_sq, "adam: tensor %d has a null pointer", i);
        PV_CHECK_ARG(((uintptr_t)t.param | (uintptr_t)t.grad | (uintptr_t)t.exp_avg | (uintptr_t)t.exp_avg_sq) % 4 == 0,
                     "adam: tensor %d has a pointer that is not 4-byte aligned", i);
        PV_CHECK_ARG((t.numel + ADAM_BLOCK_ELEMS - 1) / ADAM_BLOCK_ELEMS <= INT_MAX,
                     "adam: tensor %d is too large (numel %lld)", i, (long long)t.numel);
    }

    // the scalars in double as torch's Python computes them, each rounded to fp32 where ATen's kernels take it
    const double bias_correction1 = 1.0 - std::pow(beta1, (double)step);
    const double bias_correction2 = 1.0 - std::pow(beta2, (double)step);
    const double step_size = lr / bias_correction1;
    const double bias_correction2_sqrt = std::pow(bias_correction2, 0.5);
    AdamChunk c;
    c.s.wd = (float)weight_decay;
    c.s.has_wd = weight_decay != 0.0;
    c.s.w1 = (float)(1.0 - beta1);
    c.s.one_m_w1 = 1.0f - c.s.w1;
    c.s.lerp_small = std::fabs(c.s.w1) < 0.5f;
    c.s.b2 = (float)beta2;
    c.s.w2 = (float)(1.0 - beta2);
    c.s.inv_bc2 = (float)(1.0 / bias_correction2_sqrt);
    c.s.eps = (float)eps;
    c.s.neg_step = (float)(-step_size);

    int i = 0;
    while (i < n_tensors) {
        long long blocks = 0;
        c.n = 0;
        for (; i < n_tensors && c.n < ADAM_CHUNK_TENSORS; ++i) {
            const pvnet_adam_tensor_t &t = tensors[i];
            if (t.numel == 0) continue;
            const long long nb = (t.numel + ADAM_BLOCK_ELEMS - 1) / ADAM_BLOCK_ELEMS;
            if (blocks + nb > INT_MAX) break;  // the grid is full: this tensor opens the next launch
            AdamEntry &e = c.e[c.n++];
            e.p = static_cast<float *>(t.param);
            e.g = static_cast<const float *>(t.grad);
            e.m = static_cast<float *>(t.exp_avg);
            e.v = static_cast<float *>(t.exp_avg_sq);
            e.numel = t.numel;
            e.first_block = (int)blocks;
            e.vec = ((uintptr_t)t.param | (uintptr_t)t.grad | (uintptr_t)t.exp_avg | (uintptr_t)t.exp_avg_sq) % 16 == 0;
            blocks += nb;
        }
        if (c.n == 0) continue;
        k_adam_multi_tensor<<<(unsigned)blocks, ADAM_THREADS, 0, (cudaStream_t)stream>>>(c);
        PV_LAUNCHED("k_adam_multi_tensor");
    }
    return PVNET_OK;
}

int pvnet_adam_chunk_tensors(void) { return pvnet::ADAM_CHUNK_TENSORS; }

}  // extern "C"
