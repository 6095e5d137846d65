// losses.cu -- the per-image validation losses of the reference's NetWrapper.forward
// (tools/train_linemod.py:79-91, tools/demo.py:31-43) in one HBM-streaming pass over the network outputs and targets.
//
// Reference:
//   torch.nn.CrossEntropyLoss(reduce=False) + torch.mean(.view(b,-1), 1)   train_linemod.py:83,87-88   -> loss_seg
//   lib/utils/net_utils.py:54-80     smooth_l1_loss                                                   -> loss_vertex
//   lib/utils/net_utils.py:329-348   compute_precision_recall                                         -> precision, recall
//
// FP sequence (DESIGN.md §10):
//   cross-entropy, per pixel in fp32 as torch's log-softmax: m = max_c x_c, s = sum_c expf(x_c - m) in channel order,
//     term = -((x_t - m) - logf(s)); t = -100 contributes 0 (and still counts in the mean); any other t outside [0,C)
//     makes the image's value NaN (torch raises a device-side assert there).
//   smooth-L1, per element, every op rounded on its own (no contraction), which is torch's chain of fp32 kernels:
//     diff = w * (p - t), s = |diff| < c1, in = ((diff * diff) * c2) * s + (|diff| - c3) * (1 - s)
//   precision / recall: p = argmax_c x_c (first maximum; a NaN wins, the first NaN on ties, as torch.argmax on CUDA),
//     tp = sum p t, fp = sum p (1 - t), fn = sum (1 - p) t exactly in int64, then (tp+1)/(tp+fp+1), (tp+1)/(tp+fn+1)
//     in fp32.
//
// Reduction: pixels are assigned to threads and CTAs from the shape alone (4-pixel quads along a row, LS_QPB quads per
// CTA), each thread accumulates in fp64 / int64, a CTA reduces its threads in a fixed shuffle + warp order into the
// caller's workspace, and k_losses_final adds the CTA partials in chunk order: results are run-to-run identical and
// the two launches can be captured in a CUDA graph (no atomics, no allocation, no synchronisation).
//
// Keypoint targets (DESIGN.md §12): the loader's ground-truth vertex field, compute_vertex_hcoords
// (lib/datasets/linemod_dataset.py:68-81; tools/demo.py:58-71 is the same with hw = 1), per pixel (x, y) with
// mask == 1 and keypoint (hx, hy, hw) widened to fp64, every op rounded on its own as numpy does:
//   vx = hx - x*hw, vy = hy - y*hw; unless use_motion: n = sqrt(vx*vx + vy*vy), n < 1e-3 -> n + 1e-3, v = v / n;
//   channel 2k = (float)vx, 2k+1 = (float)vy; every other pixel +0.
// k_vertex_targets writes it as [b,2K,h,w]; k_losses_partial<MT, true> computes it in registers in place of the
// target load, so its sums equal those over the materialised field bit for bit.
#include "common.cuh"

#include <cmath>

namespace {

constexpr int LS_THREADS = 256;
constexpr int LS_QPT = 2;                          // quads per thread
constexpr int LS_QPB = LS_THREADS * LS_QPT;        // quads (of 4 pixels) per CTA
constexpr int LS_IGNORE = -100;                    // nn.CrossEntropyLoss's default ignore_index

struct LossArgs {
    const float *seg;                              // [b,C,h,w] logits
    long long seg_b, seg_c, seg_h;
    const void *mask;                              // [b,h,w] targets
    long long m_b, m_h;
    const float *pred;                             // [b,vd,h,w]
    long long p_b, p_c, p_h;
    const float *tgt;                              // [b,vd,h,w]
    long long t_b, t_c, t_h;
    const float *wgt;                              // [b,1,h,w]
    long long w_b, w_h;
    float *elem;                                   // [b,vd,h,w] contiguous elementwise smooth-L1, or NULL
    int h, w, C, vd, qw, nquads;
    float c1, c2, c3;
    int do_ce, do_pr, do_ver, vec;
};

// one CTA's sums; k_losses_final reads them in chunk order
struct LossPartial {
    double ce, in, w;
    long long tp, fp, fn, bad;
};

__device__ __forceinline__ void load4(const float *p, bool full, int n, float (&v)[4])
{
    if (full) {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = j < n ? __ldg(p + j) : 0.f;
    }
}

template <typename MT>
__device__ __forceinline__ void load_mask4(const MT *p, bool full, int n, long long (&t)[4])
{
    if (full) {
        if constexpr (sizeof(MT) == 8) {
            const longlong2 a = __ldg(reinterpret_cast<const longlong2 *>(p));
            const longlong2 b = __ldg(reinterpret_cast<const longlong2 *>(p) + 1);
            t[0] = a.x, t[1] = a.y, t[2] = b.x, t[3] = b.y;
        } else if constexpr (sizeof(MT) == 4) {
            const int4 a = __ldg(reinterpret_cast<const int4 *>(p));
            t[0] = a.x, t[1] = a.y, t[2] = a.z, t[3] = a.w;
        } else {
            const uchar4 a = __ldg(reinterpret_cast<const uchar4 *>(p));
            t[0] = a.x, t[1] = a.y, t[2] = a.z, t[3] = a.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) t[j] = j < n ? (long long)p[j] : 0;
    }
}

// keypoints [b,K,3] contiguous, float32 or float64, for the keypoint-target forms
struct KpArgs {
    const void *hc;
    int K, f64, motion;
};

__device__ __forceinline__ void load_kp(const KpArgs &kp, int img, int k, double &hx, double &hy, double &hw)
{
    const long long i = ((long long)img * kp.K + k) * 3;
    if (kp.f64) {
        const double *p = static_cast<const double *>(kp.hc) + i;
        hx = __ldg(p), hy = __ldg(p + 1), hw = __ldg(p + 2);
    } else {
        const float *p = static_cast<const float *>(kp.hc) + i;
        hx = (double)__ldg(p), hy = (double)__ldg(p + 1), hw = (double)__ldg(p + 2);
    }
}

// compute_vertex_hcoords for one foreground pixel and one keypoint, numpy's fp64 sequence op by op
__device__ __forceinline__ void kp_target(double hx, double hy, double hw, int x, int y, bool motion, float &tx,
                                          float &ty)
{
    double vx = __dsub_rn(hx, __dmul_rn((double)x, hw));
    double vy = __dsub_rn(hy, __dmul_rn((double)y, hw));
    if (!motion) {
        double n = __dsqrt_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)));
        if (n < 1e-3) n = __dadd_rn(n, 1e-3);
        vx = __ddiv_rn(vx, n);
        vy = __ddiv_rn(vy, n);
    }
    tx = __double2float_rn(vx);
    ty = __double2float_rn(vy);
}

// the targets of keypoint k for a quad's pixels: fg[j] pixels computed, the rest +0
__device__ __forceinline__ void kp_quad(const KpArgs &kp, int img, int k, int x0, int y, const bool (&fg)[4],
                                        float (&tx)[4], float (&ty)[4])
{
#pragma unroll
    for (int j = 0; j < 4; ++j) tx[j] = ty[j] = 0.f;
    if (!(fg[0] || fg[1] || fg[2] || fg[3])) return;
    double hx, hy, hw;
    load_kp(kp, img, k, hx, hy, hw);
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (fg[j]) kp_target(hx, hy, hw, x0 + j, y, kp.motion, tx[j], ty[j]);
}

template <typename MT>
__device__ __forceinline__ void fg_quad(const MT *p, bool full, int n, bool (&fg)[4])
{
    long long t[4];
    load_mask4(p, full, n, t);
#pragma unroll
    for (int j = 0; j < 4; ++j) fg[j] = j < n && t[j] == 1;       // np.argwhere(mask == 1)
}

// the vertex weights of a quad: read from a.wgt, or (MW: the caller passed no weights) the pixel's mask value
// converted to float -- the reference's vertex_weights = mask.unsqueeze(0).float() (linemod_dataset.py:227)
template <typename MT, bool MW>
__device__ __forceinline__ void weights4(const LossArgs &a, int img, int y, int x0, bool full, int n, float (&wv)[4])
{
    if constexpr (MW) {
        long long t[4];
        load_mask4(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, full, n, t);
#pragma unroll
        for (int j = 0; j < 4; ++j) wv[j] = (float)t[j];
    } else {
        load4(a.wgt + img * a.w_b + y * a.w_h + x0, full, n, wv);
    }
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// smooth-L1 of one vertex channel c of a quad: into e0's channel c (elementwise) or added to sin; the keypoint form's
// copy of the loop body in k_losses_partial, which stays written out so that its instantiations keep their code
__device__ __forceinline__ void ver_channel(const LossArgs &a, int c, float *e0, bool full, int n, const float (&wv)[4],
                                            const float (&pv)[4], const float (&tv)[4], double &sin)
{
    float in[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float d = __fmul_rn(wv[j], __fsub_rn(pv[j], tv[j]));
        const float ad = fabsf(d);
        const float s = ad < a.c1 ? 1.f : 0.f;
        in[j] = __fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), a.c2), s),
                          __fmul_rn(__fsub_rn(ad, a.c3), __fsub_rn(1.f, s)));
    }
    if (e0) {
        float *e = e0 + (size_t)c * a.h * a.w;
        if (full)
            *reinterpret_cast<float4 *>(e) = make_float4(in[0], in[1], in[2], in[3]);
        else
            for (int j = 0; j < n; ++j) e[j] = in[j];
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (j < n) sin += (double)in[j];
    }
}

// The keypoint form needs 104 registers without spilling (DESIGN.md §12): at 3 CTAs per SM (80 registers) ptxas
// spills 72 bytes, so it runs at 2.
constexpr int LS_KP_MIN_BLOCKS = 2;

// grid (chunks, b), MT = the mask element type (int64, int32, uint8 / bool); KP: the vertex targets are computed
// from the keypoints `kp` (foreground = mask == 1) instead of read from a.tgt; MW: the vertex weights are the mask
// values (weights4) instead of read from a.wgt
template <typename MT, bool KP, bool MW = false>
__global__ void __launch_bounds__(LS_THREADS, KP ? LS_KP_MIN_BLOCKS : 3)
    k_losses_partial(LossArgs a, LossPartial *__restrict__ partial, KpArgs kp)
{
    const int img = blockIdx.y;
    double ce = 0.0, sin = 0.0, sw = 0.0;
    long long tp = 0, fp = 0, fn = 0, bad = 0;
    const int q_end = min(a.nquads, (int)(blockIdx.x + 1) * LS_QPB);
    for (int q = blockIdx.x * LS_QPB + threadIdx.x; q < q_end; q += LS_THREADS) {
        const int y = q / a.qw;
        const int x0 = (q - y * a.qw) * 4;
        const int n = min(4, a.w - x0);
        const bool full = a.vec && n == 4;

        if (a.do_ce || a.do_pr) {
            const float *s0 = a.seg + img * a.seg_b + y * a.seg_h + x0;
            long long t[4];
            load_mask4(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, full, n, t);
            float v[4], m[4], best[4];
            int arg[4];
            load4(s0, full, n, v);
#pragma unroll
            for (int j = 0; j < 4; ++j) m[j] = best[j] = v[j], arg[j] = 0;
            for (int c = 1; c < a.C; ++c) {
                load4(s0 + c * a.seg_c, full, n, v);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    m[j] = fmaxf(m[j], v[j]);
                    if (!isnan(best[j]) && (isnan(v[j]) || v[j] > best[j])) best[j] = v[j], arg[j] = c;
                }
            }
            if (a.do_pr) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (j >= n) continue;
                    const long long p = arg[j];
                    tp += p * t[j];
                    fp += p * (1 - t[j]);
                    fn += (1 - p) * t[j];
                }
            }
            if (a.do_ce) {
                float s[4] = {0.f, 0.f, 0.f, 0.f};
                for (int c = 0; c < a.C; ++c) {
                    load4(s0 + c * a.seg_c, full, n, v);
#pragma unroll
                    for (int j = 0; j < 4; ++j) s[j] = __fadd_rn(s[j], expf(__fsub_rn(v[j], m[j])));
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    if (j >= n || t[j] == LS_IGNORE) continue;
                    if (t[j] < 0 || t[j] >= a.C) {
                        bad = 1;
                        continue;
                    }
                    const float xt = __ldg(s0 + t[j] * a.seg_c + j);
                    ce += (double)(-__fsub_rn(__fsub_rn(xt, m[j]), logf(s[j])));
                }
            }
        }

        if (a.do_ver) {
            float wv[4];
            weights4<MT, MW>(a, img, y, x0, full, n, wv);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < n) sw += (double)wv[j];
            const float *p0 = a.pred + img * a.p_b + y * a.p_h + x0;
            float *e0 = a.elem ? a.elem + ((size_t)img * a.vd * a.h + y) * a.w + x0 : nullptr;
            if constexpr (KP) {
                // channels 2k, 2k+1 in the same order as the loop below, so the sums are those of the field
                bool fg[4];
                fg_quad(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, full, n, fg);
                for (int k = 0; k < kp.K; ++k) {
                    float px[4], py[4], tx[4], ty[4];
                    load4(p0 + 2 * k * a.p_c, full, n, px);          // in flight while the targets are computed
                    load4(p0 + (2 * k + 1) * a.p_c, full, n, py);
                    kp_quad(kp, img, k, x0, y, fg, tx, ty);
                    ver_channel(a, 2 * k, e0, full, n, wv, px, tx, sin);
                    ver_channel(a, 2 * k + 1, e0, full, n, wv, py, ty, sin);
                }
            } else {
                const float *t0 = a.tgt + img * a.t_b + y * a.t_h + x0;
#pragma unroll 2
                for (int c = 0; c < a.vd; ++c) {
                    float pv[4], tv[4], in[4];
                    load4(p0 + c * a.p_c, full, n, pv);
                    load4(t0 + c * a.t_c, full, n, tv);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float d = __fmul_rn(wv[j], __fsub_rn(pv[j], tv[j]));
                        const float ad = fabsf(d);
                        const float s = ad < a.c1 ? 1.f : 0.f;
                        in[j] = __fadd_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), a.c2), s),
                                          __fmul_rn(__fsub_rn(ad, a.c3), __fsub_rn(1.f, s)));
                    }
                    if (e0) {
                        float *e = e0 + (size_t)c * a.h * a.w;
                        if (full)
                            *reinterpret_cast<float4 *>(e) = make_float4(in[0], in[1], in[2], in[3]);
                        else
                            for (int j = 0; j < n; ++j) e[j] = in[j];
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            if (j < n) sin += (double)in[j];
                    }
                }
            }
        }
    }

    // fixed-order reduction: shuffle tree inside each warp, then the warps in index order
    __shared__ LossPartial s_w[LS_THREADS / 32];
    ce = warp_sum(ce), sin = warp_sum(sin), sw = warp_sum(sw);
    tp = warp_sum(tp), fp = warp_sum(fp), fn = warp_sum(fn), bad = warp_sum(bad);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) s_w[wid] = {ce, sin, sw, tp, fp, fn, bad};
    __syncthreads();
    if (threadIdx.x == 0) {
        LossPartial r = s_w[0];
        for (int i = 1; i < LS_THREADS / 32; ++i) {
            r.ce += s_w[i].ce, r.in += s_w[i].in, r.w += s_w[i].w;
            r.tp += s_w[i].tp, r.fp += s_w[i].fp, r.fn += s_w[i].fn, r.bad += s_w[i].bad;
        }
        partial[(size_t)img * gridDim.x + blockIdx.x] = r;
    }
}

// one thread per image: the CTA partials in chunk order -> the four per-image values
__global__ void k_losses_final(const LossPartial *__restrict__ partial, int chunks, int b, double npix, int vd,
                               float *loss_seg, float *loss_vertex, float *precision, float *recall)
{
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= b) return;
    LossPartial r = partial[(size_t)img * chunks];
    for (int c = 1; c < chunks; ++c) {
        const LossPartial &p = partial[(size_t)img * chunks + c];
        r.ce += p.ce, r.in += p.in, r.w += p.w;
        r.tp += p.tp, r.fp += p.fp, r.fn += p.fn, r.bad += p.bad;
    }
    if (loss_seg) loss_seg[img] = r.bad ? __int_as_float(0x7fffffff) : __double2float_rn(r.ce / npix);
    // net_utils.py:74 with torch's fp32 ops: sum(in) / (ver_dim * sum(w) + 1e-3)
    if (loss_vertex)
        loss_vertex[img] = __fdiv_rn(__double2float_rn(r.in),
                                     __fadd_rn(__fmul_rn((float)vd, __double2float_rn(r.w)), 1e-3f));
    // net_utils.py:343-344; exact integer counts, rounded once to fp32 (equal to torch's fp32 sums below 2^24)
    const float tpf = (float)r.tp;
    const float num = __fadd_rn(tpf, 1.f);
    if (precision) precision[img] = __fdiv_rn(num, __fadd_rn(__fadd_rn(tpf, (float)r.fp), 1.f));
    if (recall) recall[img] = __fdiv_rn(num, __fadd_rn(__fadd_rn(tpf, (float)r.fn), 1.f));
}

// grid (chunks, b): the keypoint targets [b,2K,h,w] (contiguous), same quad assignment as k_losses_partial; a
// thread stores a quad's 4 pixels of every channel, as one float4 where alignment allows
struct VtArgs {
    const void *mask;
    long long m_b, m_h;
    float *out;
    int h, w, qw, nquads, mvec, ovec;
};

template <typename MT>
__global__ void __launch_bounds__(LS_THREADS) k_vertex_targets(VtArgs a, KpArgs kp)
{
    const int img = blockIdx.y;
    const size_t plane = (size_t)a.h * a.w;
    const int q_end = min(a.nquads, (int)(blockIdx.x + 1) * LS_QPB);
    for (int q = blockIdx.x * LS_QPB + threadIdx.x; q < q_end; q += LS_THREADS) {
        const int y = q / a.qw;
        const int x0 = (q - y * a.qw) * 4;
        const int n = min(4, a.w - x0);
        bool fg[4];
        fg_quad(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, a.mvec && n == 4, n, fg);
        const bool full = a.ovec && n == 4;
        float *o = a.out + (size_t)img * 2 * kp.K * plane + (size_t)y * a.w + x0;
        for (int k = 0; k < kp.K; ++k) {
            float tx[4], ty[4];
            kp_quad(kp, img, k, x0, y, fg, tx, ty);
            float *ox = o + (size_t)(2 * k) * plane, *oy = ox + plane;
            if (full) {
                *reinterpret_cast<float4 *>(ox) = make_float4(tx[0], tx[1], tx[2], tx[3]);
                *reinterpret_cast<float4 *>(oy) = make_float4(ty[0], ty[1], ty[2], ty[3]);
            } else {
                for (int j = 0; j < n; ++j) ox[j] = tx[j], oy[j] = ty[j];
            }
        }
    }
}

// ------------------------------------------------------------------ gradients (DESIGN.md §13)
// The gradients of loss_seg and of the normalised loss_vertex with respect to seg_pred and vertex_pred, each the
// sequence torch's CUDA autograd runs through the reference's expressions, every op rounded on its own:
//   cross-entropy: g = gs * (1.0f / (float)(h*w))   (MeanBackward: ATen divides a CUDA tensor by a CPU scalar as a
//     multiplication by its float reciprocal); per pixel lp_c = (x_c - m) - logf(s) as in the forward,
//     S = 0 + gO_0 + ... + gO_{C-1} with gO_t = -g at the target and 0 elsewhere (NLLLoss2d backward), and
//     grad_c = fmaf(-expf(lp_c), S, gO_c) (the log-softmax backward epilogue gO - exp(out)*S, which nvcc contracts);
//     t = -100 gives gO = 0; any other t outside [0,C) makes every seg-gradient element of the image NaN.
//   smooth-L1: gi = gv / den with den = ver_dim*(float)Σw + 1e-3f recomputed in the forward's fixed order
//     (k_weight_sum_partial + k_grad_final), then per element with d = w*(p - t), s = |d| < c1:
//     A = ((gi*s)*c2)*(2*d)  (MulBackward, MulBackward, PowBackward)   B = (gi*(1 - s))*sgn(d)  (AbsBackward)
//     grad = (A + B)*w: autograd runs PowBackward0 before AbsBackward0, so A is in the buffer and B is added.
//     sgn is torch's CUDA sign: (0 < d) - (d < 0), so 0 for +-0 and NaN.
struct GradArgs {
    float *gseg;                                   // [b,C,h,w] through strides, or NULL
    long long gs_b, gs_c, gs_h;
    float *gver;                                   // [b,vd,h,w] through strides, or NULL
    long long gv_b, gv_c, gv_h;
    const float *gls;                              // grad_loss_seg [b]; NULL: gseg is written as zeros
    const float *gi;                               // gv / den per image (k_grad_final); NULL: gver written as zeros
    int *bad;                                      // [b, chunks] per-CTA invalid-target flags
    float inv_n;                                   // 1.0f / (float)(h*w)
};

__device__ __forceinline__ void store4(float *p, bool full, int n, const float (&v)[4])
{
    if (full)
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else
        for (int j = 0; j < n; ++j) p[j] = v[j];
}

// the smooth-L1 gradient of one vertex channel of a quad
__device__ __forceinline__ void ver_grad(const LossArgs &a, float gi, const float (&wv)[4], const float (&pv)[4],
                                         const float (&tv)[4], float (&o)[4])
{
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float d = __fmul_rn(wv[j], __fsub_rn(pv[j], tv[j]));
        const float s = fabsf(d) < a.c1 ? 1.f : 0.f;
        const float sg = (float)((0.f < d) - (d < 0.f));
        const float A = __fmul_rn(__fmul_rn(__fmul_rn(gi, s), a.c2), __fmul_rn(2.f, d));
        const float B = __fmul_rn(__fmul_rn(gi, __fsub_rn(1.f, s)), sg);
        o[j] = __fmul_rn(__fadd_rn(A, B), wv[j]);
    }
}

// grid (chunks, b), the quad assignment of k_losses_partial; each thread writes its quads' gradients (MW as there)
template <typename MT, bool KP, bool MW = false>
__global__ void __launch_bounds__(LS_THREADS, KP ? LS_KP_MIN_BLOCKS : 3)
    k_losses_backward(LossArgs a, GradArgs g, KpArgs kp)
{
    const int img = blockIdx.y;
    const float gs = g.gls ? __fmul_rn(__ldg(g.gls + img), g.inv_n) : 0.f;
    const float gi = g.gi ? __ldg(g.gi + img) : 0.f;
    const float zero[4] = {0.f, 0.f, 0.f, 0.f};
    int bad = 0;
    const int q_end = min(a.nquads, (int)(blockIdx.x + 1) * LS_QPB);
    for (int q = blockIdx.x * LS_QPB + threadIdx.x; q < q_end; q += LS_THREADS) {
        const int y = q / a.qw;
        const int x0 = (q - y * a.qw) * 4;
        const int n = min(4, a.w - x0);
        const bool full = a.vec && n == 4;

        if (g.gseg) {
            float *o0 = g.gseg + img * g.gs_b + y * g.gs_h + x0;
            if (!g.gls) {
                for (int c = 0; c < a.C; ++c) store4(o0 + c * g.gs_c, full, n, zero);
            } else {
                const float *s0 = a.seg + img * a.seg_b + y * a.seg_h + x0;
                long long t[4];
                load_mask4(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, full, n, t);
                float v[4], m[4], s[4] = {0.f, 0.f, 0.f, 0.f}, ls[4], S[4];
                load4(s0, full, n, m);
                for (int c = 1; c < a.C; ++c) {
                    load4(s0 + c * a.seg_c, full, n, v);
#pragma unroll
                    for (int j = 0; j < 4; ++j) m[j] = fmaxf(m[j], v[j]);
                }
                for (int c = 0; c < a.C; ++c) {
                    load4(s0 + c * a.seg_c, full, n, v);
#pragma unroll
                    for (int j = 0; j < 4; ++j) s[j] = __fadd_rn(s[j], expf(__fsub_rn(v[j], m[j])));
                }
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    ls[j] = logf(s[j]);
                    const bool valid = t[j] >= 0 && t[j] < a.C;
                    if (j < n && !valid && t[j] != LS_IGNORE) bad = 1;
                    S[j] = valid ? __fadd_rn(0.f, -gs) : 0.f;          // the zeros of the other channels add nothing
                }
                for (int c = 0; c < a.C; ++c) {
                    load4(s0 + c * a.seg_c, full, n, v);
                    float o[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float e = expf(__fsub_rn(__fsub_rn(v[j], m[j]), ls[j]));
                        o[j] = __fmaf_rn(-e, S[j], t[j] == c ? -gs : 0.f);
                    }
                    store4(o0 + c * g.gs_c, full, n, o);
                }
            }
        }

        if (g.gver) {
            float *o0 = g.gver + img * g.gv_b + y * g.gv_h + x0;
            if (!g.gi) {
                for (int c = 0; c < a.vd; ++c) store4(o0 + c * g.gv_c, full, n, zero);
                continue;
            }
            float wv[4], o[4];
            weights4<MT, MW>(a, img, y, x0, full, n, wv);
            const float *p0 = a.pred + img * a.p_b + y * a.p_h + x0;
            if constexpr (KP) {
                bool fg[4];
                fg_quad(static_cast<const MT *>(a.mask) + img * a.m_b + y * a.m_h + x0, full, n, fg);
                for (int k = 0; k < kp.K; ++k) {
                    float px[4], py[4], tx[4], ty[4];
                    load4(p0 + 2 * k * a.p_c, full, n, px);
                    load4(p0 + (2 * k + 1) * a.p_c, full, n, py);
                    kp_quad(kp, img, k, x0, y, fg, tx, ty);
                    ver_grad(a, gi, wv, px, tx, o);
                    store4(o0 + 2 * k * g.gv_c, full, n, o);
                    ver_grad(a, gi, wv, py, ty, o);
                    store4(o0 + (2 * k + 1) * g.gv_c, full, n, o);
                }
            } else {
                const float *t0 = a.tgt + img * a.t_b + y * a.t_h + x0;
#pragma unroll 2
                for (int c = 0; c < a.vd; ++c) {
                    float pv[4], tv[4];
                    load4(p0 + c * a.p_c, full, n, pv);
                    load4(t0 + c * a.t_c, full, n, tv);
                    ver_grad(a, gi, wv, pv, tv, o);
                    store4(o0 + c * g.gv_c, full, n, o);
                }
            }
        }
    }
    if (g.gseg && g.gls) {
        bad = __syncthreads_or(bad);
        if (threadIdx.x == 0) g.bad[(size_t)img * gridDim.x + blockIdx.x] = bad;
    }
}

// grid (chunks, b): Σw of each CTA's quads, summed exactly as k_losses_partial sums `sw` (same thread order, shuffle
// tree and warp order), so that k_grad_final's denominator is the forward's bit for bit (MW: the weights are the mask
// values of element type MT, weights4)
template <typename MT, bool MW>
__global__ void __launch_bounds__(LS_THREADS) k_weight_sum_partial(LossArgs a, double *__restrict__ partial)
{
    const int img = blockIdx.y;
    double sw = 0.0;
    const int q_end = min(a.nquads, (int)(blockIdx.x + 1) * LS_QPB);
    for (int q = blockIdx.x * LS_QPB + threadIdx.x; q < q_end; q += LS_THREADS) {
        const int y = q / a.qw;
        const int x0 = (q - y * a.qw) * 4;
        const int n = min(4, a.w - x0);
        float wv[4];
        weights4<MT, MW>(a, img, y, x0, a.vec && n == 4, n, wv);
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (j < n) sw += (double)wv[j];
    }
    __shared__ double s_w[LS_THREADS / 32];
    sw = warp_sum(sw);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = sw;
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = s_w[0];
        for (int i = 1; i < LS_THREADS / 32; ++i) r += s_w[i];
        partial[(size_t)img * gridDim.x + blockIdx.x] = r;
    }
}

// one thread per image: gi = gv / (ver_dim * Σw + 1e-3), k_losses_final's denominator
__global__ void k_grad_final(const double *__restrict__ partial, int chunks, int b, int vd,
                             const float *__restrict__ grad_loss_vertex, float *gi)
{
    const int img = blockIdx.x * blockDim.x + threadIdx.x;
    if (img >= b) return;
    double r = partial[(size_t)img * chunks];
    for (int c = 1; c < chunks; ++c) r += partial[(size_t)img * chunks + c];
    const float den = __fadd_rn(__fmul_rn((float)vd, __double2float_rn(r)), 1e-3f);
    gi[img] = __fdiv_rn(grad_loss_vertex[img], den);
}

// grid (chunks, b): an image with an invalid target anywhere gets NaN in its whole seg gradient
__global__ void __launch_bounds__(LS_THREADS) k_seg_grad_invalid(LossArgs a, GradArgs g)
{
    const int img = blockIdx.y;
    int bad = 0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += LS_THREADS) bad |= g.bad[(size_t)img * gridDim.x + i];
    if (!__syncthreads_or(bad)) return;
    const float qnan = __int_as_float(0x7fffffff);
    const float nan4[4] = {qnan, qnan, qnan, qnan};
    const int q_end = min(a.nquads, (int)(blockIdx.x + 1) * LS_QPB);
    for (int q = blockIdx.x * LS_QPB + threadIdx.x; q < q_end; q += LS_THREADS) {
        const int y = q / a.qw;
        const int x0 = (q - y * a.qw) * 4;
        const int n = min(4, a.w - x0);
        for (int c = 0; c < a.C; ++c)
            store4(g.gseg + img * g.gs_b + y * g.gs_h + x0 + c * g.gs_c, a.vec && n == 4, n, nan4);
    }
}

int ls_chunks(int h, int w)
{
    const long long nq = (long long)h * ((w + 3) / 4);
    return (int)((nq + LS_QPB - 1) / LS_QPB);
}

bool aligned(const void *p, size_t a) { return p == nullptr || reinterpret_cast<uintptr_t>(p) % a == 0; }

bool strides_ok(const int64_t *s, int k)
{
    for (int i = 0; i < k; ++i)
        if (s[i] % 4) return false;
    return true;
}

template <bool KP, bool MW = false>
void launch_partial(int msz, dim3 grid, cudaStream_t st, const LossArgs &a, LossPartial *partial, const KpArgs &kp)
{
    if (msz == 8)
        k_losses_partial<long long, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, partial, kp);
    else if (msz == 4)
        k_losses_partial<int, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, partial, kp);
    else
        k_losses_partial<unsigned char, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, partial, kp);
}

template <bool KP, bool MW>
void launch_backward(int msz, dim3 grid, cudaStream_t st, const LossArgs &a, const GradArgs &g, const KpArgs &kp)
{
    if (msz == 8)
        k_losses_backward<long long, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, g, kp);
    else if (msz == 4)
        k_losses_backward<int, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, g, kp);
    else
        k_losses_backward<unsigned char, KP, MW><<<grid, LS_THREADS, 0, st>>>(a, g, kp);
}

// pvnet_seg_vertex_losses (kp == NULL: targets read from vertex) and pvnet_seg_vertex_losses_keypoints (kp: targets
// computed from the keypoints, foreground = mask == 1)
int seg_vertex_losses(const float *seg_pred, const int64_t seg_strides[4], const void *mask, int mask_elem_size,
                      const int64_t mask_strides[3], const float *vertex_pred, const int64_t pred_strides[4],
                      const float *vertex, const int64_t vertex_strides[4], const KpArgs *kp,
                      const float *vertex_weights, const int64_t weight_strides[4], int b, int h, int w, int C,
                      int ver_dim, double sigma, int normalize, float *loss_seg, float *loss_vertex, float *precision,
                      float *recall, void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1, "non-positive dimension (b=%d, h=%d, w=%d)", b, h, w);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    const bool do_ce = loss_seg != nullptr, do_pr = precision != nullptr || recall != nullptr;
    const bool do_ver = loss_vertex != nullptr;
    // no weights and no weight strides: the weights are the mask values (a NULL pointer with strides stays an error)
    const bool mw = do_ver && !vertex_weights && !weight_strides;
    const bool need_mask = do_ce || do_pr || (do_ver && (kp || mw));
    PV_CHECK_ARG(do_ce || do_pr || do_ver, "no output requested (loss_seg, loss_vertex, precision, recall all null)");
    if (do_ce || do_pr) {
        PV_CHECK_ARG(seg_pred && seg_strides, "null pointer (seg_pred or its strides)");
        PV_CHECK_ARG(C >= 1, "non-positive dimension (C=%d)", C);
        PV_CHECK_ARG(seg_strides[3] == 1, "unit stride along w is not 1 (seg %lld)", (long long)seg_strides[3]);
    }
    if (need_mask) {
        PV_CHECK_ARG(mask && mask_strides, "null pointer (mask or its strides)");
        PV_CHECK_ARG(mask_elem_size == 1 || mask_elem_size == 4 || mask_elem_size == 8,
                     "mask_elem_size %d is not 1, 4 or 8", mask_elem_size);
        PV_CHECK_ARG(mask_strides[2] == 1, "unit stride along w is not 1 (mask %lld)", (long long)mask_strides[2]);
    }
    if (do_ver) {
        PV_CHECK_ARG(vertex_pred && pred_strides && (mw || (vertex_weights && weight_strides)),
                     "null pointer (vertex_pred / vertex_weights or their strides)");
        PV_CHECK_ARG(ver_dim >= 1, "non-positive dimension (ver_dim=%d)", ver_dim);
        PV_CHECK_ARG(pred_strides[3] == 1 && (mw || weight_strides[3] == 1),
                     "unit stride along w is not 1 (vertex_pred %lld, vertex_weights %lld)",
                     (long long)pred_strides[3], mw ? 1LL : (long long)weight_strides[3]);
        if (kp) {
            PV_CHECK_ARG(kp->hc, "null pointer (hcoords)");
            PV_CHECK_ARG(ver_dim == 2 * kp->K, "ver_dim %d is not 2 x the number of keypoints", ver_dim);
        } else {
            PV_CHECK_ARG(vertex && vertex_strides, "null pointer (vertex or its strides)");
            PV_CHECK_ARG(vertex_strides[3] == 1, "unit stride along w is not 1 (vertex %lld)",
                         (long long)vertex_strides[3]);
        }
        PV_CHECK_ARG(sigma == sigma && sigma != 0.0, "sigma %g is zero or NaN", sigma);
    }
    PV_CHECK_ARG(workspace, "null pointer (workspace)");
    size_t need = 0;
    if (pvnet_seg_vertex_losses_workspace_bytes(b, h, w, &need) != PVNET_OK) return PVNET_E_INVALID;
    PV_CHECK_ARG(workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);

    LossArgs a = {};
    a.h = h, a.w = w, a.C = C, a.vd = ver_dim, a.qw = (w + 3) / 4, a.nquads = h * a.qw;
    a.do_ce = do_ce, a.do_pr = do_pr, a.do_ver = do_ver;
    bool vec = true;
    if (do_ce || do_pr) {
        a.seg = seg_pred, a.seg_b = seg_strides[0], a.seg_c = seg_strides[1], a.seg_h = seg_strides[2];
        vec = vec && aligned(seg_pred, 16) && strides_ok(seg_strides, 3);
    }
    if (need_mask) {
        a.mask = mask, a.m_b = mask_strides[0], a.m_h = mask_strides[1];
        vec = vec && aligned(mask, 4 * mask_elem_size) && strides_ok(mask_strides, 2);
    }
    if (do_ver) {
        // net_utils.py:65-71: sigma_2 = sigma ** 2 in double; the scalars reach the fp32 kernels rounded to float
        const double s2 = sigma * sigma;
        a.c1 = (float)(1.0 / s2), a.c2 = (float)(s2 / 2.0), a.c3 = (float)(0.5 / s2);
        a.pred = vertex_pred, a.p_b = pred_strides[0], a.p_c = pred_strides[1], a.p_h = pred_strides[2];
        if (!kp) {
            a.tgt = vertex, a.t_b = vertex_strides[0], a.t_c = vertex_strides[1], a.t_h = vertex_strides[2];
            vec = vec && aligned(vertex, 16) && strides_ok(vertex_strides, 3);
        }
        if (!mw) {
            a.wgt = vertex_weights, a.w_b = weight_strides[0], a.w_h = weight_strides[2];
            vec = vec && aligned(vertex_weights, 16) && weight_strides[0] % 4 == 0 && weight_strides[2] % 4 == 0;
        }
        a.elem = normalize ? nullptr : loss_vertex;
        vec = vec && aligned(vertex_pred, 16) && strides_ok(pred_strides, 3) &&
              (normalize || (aligned(loss_vertex, 16) && w % 4 == 0));
    }
    a.vec = vec;
    LossPartial *partial = static_cast<LossPartial *>(workspace);
    const int chunks = ls_chunks(h, w);
    const dim3 grid(chunks, b);
    cudaStream_t st = (cudaStream_t)stream;
    const int msz = need_mask ? mask_elem_size : 8;
    if (kp && do_ver) {
        if (mw)
            launch_partial<true, true>(msz, grid, st, a, partial, *kp);
        else
            launch_partial<true>(msz, grid, st, a, partial, *kp);
        PV_LAUNCHED(msz == 8 ? "k_losses_partial<int64, keypoints>"
                    : msz == 4 ? "k_losses_partial<int32, keypoints>" : "k_losses_partial<uint8, keypoints>");
    } else {
        if (mw)
            launch_partial<false, true>(msz, grid, st, a, partial, KpArgs{});
        else
            launch_partial<false>(msz, grid, st, a, partial, KpArgs{});
        PV_LAUNCHED(msz == 8 ? "k_losses_partial<int64>" : msz == 4 ? "k_losses_partial<int32>" : "k_losses_partial<uint8>");
    }
    k_losses_final<<<(b + 127) / 128, 128, 0, st>>>(partial, chunks, b, (double)h * w, ver_dim, loss_seg,
                                                    (do_ver && normalize) ? loss_vertex : nullptr, precision, recall);
    PV_LAUNCHED("k_losses_final");
    return PVNET_OK;
}

// pvnet_seg_vertex_losses_backward (kp == NULL) and pvnet_seg_vertex_losses_keypoints_backward (kp)
int seg_vertex_losses_backward(const float *seg_pred, const int64_t seg_strides[4], const void *mask,
                               int mask_elem_size, const int64_t mask_strides[3], const float *vertex_pred,
                               const int64_t pred_strides[4], const float *vertex, const int64_t vertex_strides[4],
                               const KpArgs *kp, const float *vertex_weights, const int64_t weight_strides[4], int b,
                               int h, int w, int C, int ver_dim, double sigma, int normalize,
                               const float *grad_loss_seg, const float *grad_loss_vertex, float *grad_seg,
                               const int64_t grad_seg_strides[4], float *grad_vertex,
                               const int64_t grad_vertex_strides[4], void *workspace, size_t workspace_bytes,
                               pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1, "non-positive dimension (b=%d, h=%d, w=%d)", b, h, w);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    PV_CHECK_ARG(grad_seg || grad_vertex, "no output requested (grad_seg, grad_vertex both null)");
    const bool do_ce = grad_seg && grad_loss_seg, do_ver = grad_vertex && grad_loss_vertex;
    const bool mw = do_ver && !vertex_weights && !weight_strides;     // weights = mask values, as in the forward
    const bool need_mask = do_ce || (do_ver && (kp || mw));
    if (grad_seg) {
        PV_CHECK_ARG(grad_seg_strides, "null pointer (grad_seg_strides)");
        PV_CHECK_ARG(C >= 1, "non-positive dimension (C=%d)", C);
        PV_CHECK_ARG(grad_seg_strides[3] == 1, "unit stride along w is not 1 (grad_seg %lld)",
                     (long long)grad_seg_strides[3]);
    }
    if (grad_vertex) {
        PV_CHECK_ARG(grad_vertex_strides, "null pointer (grad_vertex_strides)");
        PV_CHECK_ARG(ver_dim >= 1, "non-positive dimension (ver_dim=%d)", ver_dim);
        PV_CHECK_ARG(grad_vertex_strides[3] == 1, "unit stride along w is not 1 (grad_vertex %lld)",
                     (long long)grad_vertex_strides[3]);
    }
    if (do_ce) {
        PV_CHECK_ARG(seg_pred && seg_strides, "null pointer (seg_pred or its strides)");
        PV_CHECK_ARG(seg_strides[3] == 1, "unit stride along w is not 1 (seg %lld)", (long long)seg_strides[3]);
    }
    if (need_mask) {
        PV_CHECK_ARG(mask && mask_strides, "null pointer (mask or its strides)");
        PV_CHECK_ARG(mask_elem_size == 1 || mask_elem_size == 4 || mask_elem_size == 8,
                     "mask_elem_size %d is not 1, 4 or 8", mask_elem_size);
        PV_CHECK_ARG(mask_strides[2] == 1, "unit stride along w is not 1 (mask %lld)", (long long)mask_strides[2]);
    }
    if (do_ver) {
        PV_CHECK_ARG(vertex_pred && pred_strides && (mw || (vertex_weights && weight_strides)),
                     "null pointer (vertex_pred / vertex_weights or their strides)");
        PV_CHECK_ARG(pred_strides[3] == 1 && (mw || weight_strides[3] == 1),
                     "unit stride along w is not 1 (vertex_pred %lld, vertex_weights %lld)",
                     (long long)pred_strides[3], mw ? 1LL : (long long)weight_strides[3]);
        if (kp) {
            PV_CHECK_ARG(kp->hc, "null pointer (hcoords)");
            PV_CHECK_ARG(ver_dim == 2 * kp->K, "ver_dim %d is not 2 x the number of keypoints", ver_dim);
        } else {
            PV_CHECK_ARG(vertex && vertex_strides, "null pointer (vertex or its strides)");
            PV_CHECK_ARG(vertex_strides[3] == 1, "unit stride along w is not 1 (vertex %lld)",
                         (long long)vertex_strides[3]);
        }
        PV_CHECK_ARG(sigma == sigma && sigma != 0.0, "sigma %g is zero or NaN", sigma);
        PV_CHECK_ARG(normalize, "the gradient is that of the normalised loss (normalize must be nonzero)");
    }
    PV_CHECK_ARG(workspace, "null pointer (workspace)");
    size_t need = 0;
    if (pvnet_seg_vertex_losses_workspace_bytes(b, h, w, &need) != PVNET_OK) return PVNET_E_INVALID;
    PV_CHECK_ARG(workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);

    LossArgs a = {};
    GradArgs g = {};
    a.h = h, a.w = w, a.C = C, a.vd = ver_dim, a.qw = (w + 3) / 4, a.nquads = h * a.qw;
    bool vec = true;
    if (grad_seg) {
        g.gseg = grad_seg, g.gs_b = grad_seg_strides[0], g.gs_c = grad_seg_strides[1], g.gs_h = grad_seg_strides[2];
        vec = vec && aligned(grad_seg, 16) && strides_ok(grad_seg_strides, 3);
    }
    if (grad_vertex) {
        g.gver = grad_vertex, g.gv_b = grad_vertex_strides[0], g.gv_c = grad_vertex_strides[1];
        g.gv_h = grad_vertex_strides[2];
        vec = vec && aligned(grad_vertex, 16) && strides_ok(grad_vertex_strides, 3);
    }
    if (do_ce) {
        a.seg = seg_pred, a.seg_b = seg_strides[0], a.seg_c = seg_strides[1], a.seg_h = seg_strides[2];
        vec = vec && aligned(seg_pred, 16) && strides_ok(seg_strides, 3);
        g.gls = grad_loss_seg;
        g.inv_n = 1.0f / (float)((long long)h * w);    // ATen: opmath_t(1.0) / the scalar as opmath_t
    }
    if (need_mask) {
        a.mask = mask, a.m_b = mask_strides[0], a.m_h = mask_strides[1];
        vec = vec && aligned(mask, 4 * mask_elem_size) && strides_ok(mask_strides, 2);
    }
    if (do_ver) {
        const double s2 = sigma * sigma;
        a.c1 = (float)(1.0 / s2), a.c2 = (float)(s2 / 2.0);
        a.pred = vertex_pred, a.p_b = pred_strides[0], a.p_c = pred_strides[1], a.p_h = pred_strides[2];
        if (!kp) {
            a.tgt = vertex, a.t_b = vertex_strides[0], a.t_c = vertex_strides[1], a.t_h = vertex_strides[2];
            vec = vec && aligned(vertex, 16) && strides_ok(vertex_strides, 3);
        }
        if (!mw) {
            a.wgt = vertex_weights, a.w_b = weight_strides[0], a.w_h = weight_strides[2];
            vec = vec && aligned(vertex_weights, 16) && weight_strides[0] % 4 == 0 && weight_strides[2] % 4 == 0;
        }
        vec = vec && aligned(vertex_pred, 16) && strides_ok(pred_strides, 3);
    }
    a.vec = vec;
    // workspace: Σw partials (double [b, chunks]), gi (float [b]), invalid-target flags (int [b, chunks])
    const int chunks = ls_chunks(h, w);
    double *wsum = static_cast<double *>(workspace);
    float *gi = reinterpret_cast<float *>(wsum + (size_t)b * chunks);
    g.bad = reinterpret_cast<int *>(gi + b);
    const dim3 grid(chunks, b);
    cudaStream_t st = (cudaStream_t)stream;
    const int msz = need_mask ? mask_elem_size : 8;
    if (do_ver) {
        LossArgs wa = a;
        if (mw) {
            // the mask's own vectorisation rule; the sums do not depend on it
            wa.vec = aligned(mask, 4 * mask_elem_size) && strides_ok(mask_strides, 2);
            if (msz == 8)
                k_weight_sum_partial<long long, true><<<grid, LS_THREADS, 0, st>>>(wa, wsum);
            else if (msz == 4)
                k_weight_sum_partial<int, true><<<grid, LS_THREADS, 0, st>>>(wa, wsum);
            else
                k_weight_sum_partial<unsigned char, true><<<grid, LS_THREADS, 0, st>>>(wa, wsum);
        } else {
            wa.vec = aligned(vertex_weights, 16) && weight_strides[0] % 4 == 0 && weight_strides[2] % 4 == 0;
            k_weight_sum_partial<float, false><<<grid, LS_THREADS, 0, st>>>(wa, wsum);
        }
        PV_LAUNCHED("k_weight_sum_partial");
        k_grad_final<<<(b + 127) / 128, 128, 0, st>>>(wsum, chunks, b, ver_dim, grad_loss_vertex, gi);
        PV_LAUNCHED("k_grad_final");
        g.gi = gi;
    }
    if (kp && do_ver) {
        if (mw)
            launch_backward<true, true>(msz, grid, st, a, g, *kp);
        else
            launch_backward<true, false>(msz, grid, st, a, g, *kp);
        PV_LAUNCHED(msz == 8 ? "k_losses_backward<int64, keypoints>"
                    : msz == 4 ? "k_losses_backward<int32, keypoints>" : "k_losses_backward<uint8, keypoints>");
    } else {
        if (mw)
            launch_backward<false, true>(msz, grid, st, a, g, KpArgs{});
        else
            launch_backward<false, false>(msz, grid, st, a, g, KpArgs{});
        PV_LAUNCHED(msz == 8 ? "k_losses_backward<int64>" : msz == 4 ? "k_losses_backward<int32>"
                                                                      : "k_losses_backward<uint8>");
    }
    if (do_ce) {
        k_seg_grad_invalid<<<grid, LS_THREADS, 0, st>>>(a, g);
        PV_LAUNCHED("k_seg_grad_invalid");
    }
    return PVNET_OK;
}

}  // namespace

extern "C" {

int pvnet_seg_vertex_losses_workspace_bytes(int b, int h, int w, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1, "non-positive dimension (b=%d, h=%d, w=%d)", b, h, w);
    PV_CHECK_ARG(bytes, "null pointer");
    PV_CHECK_ARG((long long)h * ((w + 3) / 4) <= 0x7fffffffLL - LS_QPB, "image of %d x %d pixels too large", h, w);
    *bytes = (size_t)b * ls_chunks(h, w) * sizeof(LossPartial);
    return PVNET_OK;
}

int pvnet_seg_vertex_losses(const float *seg_pred, const int64_t seg_strides[4], const void *mask, int mask_elem_size,
                            const int64_t mask_strides[3], const float *vertex_pred, const int64_t pred_strides[4],
                            const float *vertex, const int64_t vertex_strides[4], const float *vertex_weights,
                            const int64_t weight_strides[4], int b, int h, int w, int C, int ver_dim, double sigma,
                            int normalize, float *loss_seg, float *loss_vertex, float *precision, float *recall,
                            void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    return seg_vertex_losses(seg_pred, seg_strides, mask, mask_elem_size, mask_strides, vertex_pred, pred_strides,
                             vertex, vertex_strides, nullptr, vertex_weights, weight_strides, b, h, w, C, ver_dim,
                             sigma, normalize, loss_seg, loss_vertex, precision, recall, workspace, workspace_bytes,
                             stream);
}

int pvnet_seg_vertex_losses_keypoints(const float *seg_pred, const int64_t seg_strides[4], const void *mask,
                                      int mask_elem_size, const int64_t mask_strides[3], const float *vertex_pred,
                                      const int64_t pred_strides[4], const void *hcoords, int hcoords_f64,
                                      int use_motion, const float *vertex_weights, const int64_t weight_strides[4],
                                      int b, int h, int w, int C, int ver_dim, double sigma, int normalize,
                                      float *loss_seg, float *loss_vertex, float *precision, float *recall,
                                      void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    const KpArgs kp = {hcoords, ver_dim / 2, hcoords_f64 != 0, use_motion != 0};
    return seg_vertex_losses(seg_pred, seg_strides, mask, mask_elem_size, mask_strides, vertex_pred, pred_strides,
                             nullptr, nullptr, &kp, vertex_weights, weight_strides, b, h, w, C, ver_dim, sigma,
                             normalize, loss_seg, loss_vertex, precision, recall, workspace, workspace_bytes, stream);
}

int pvnet_seg_vertex_losses_backward(const float *seg_pred, const int64_t seg_strides[4], const void *mask,
                                     int mask_elem_size, const int64_t mask_strides[3], const float *vertex_pred,
                                     const int64_t pred_strides[4], const float *vertex,
                                     const int64_t vertex_strides[4], const float *vertex_weights,
                                     const int64_t weight_strides[4], int b, int h, int w, int C, int ver_dim,
                                     double sigma, int normalize, const float *grad_loss_seg,
                                     const float *grad_loss_vertex, float *grad_seg, const int64_t grad_seg_strides[4],
                                     float *grad_vertex, const int64_t grad_vertex_strides[4], void *workspace,
                                     size_t workspace_bytes, pvnet_stream_t stream)
{
    return seg_vertex_losses_backward(seg_pred, seg_strides, mask, mask_elem_size, mask_strides, vertex_pred,
                                      pred_strides, vertex, vertex_strides, nullptr, vertex_weights, weight_strides, b,
                                      h, w, C, ver_dim, sigma, normalize, grad_loss_seg, grad_loss_vertex, grad_seg,
                                      grad_seg_strides, grad_vertex, grad_vertex_strides, workspace, workspace_bytes,
                                      stream);
}

int pvnet_seg_vertex_losses_keypoints_backward(
    const float *seg_pred, const int64_t seg_strides[4], const void *mask, int mask_elem_size,
    const int64_t mask_strides[3], const float *vertex_pred, const int64_t pred_strides[4], const void *hcoords,
    int hcoords_f64, int use_motion, const float *vertex_weights, const int64_t weight_strides[4], int b, int h, int w,
    int C, int ver_dim, double sigma, int normalize, const float *grad_loss_seg, const float *grad_loss_vertex,
    float *grad_seg, const int64_t grad_seg_strides[4], float *grad_vertex, const int64_t grad_vertex_strides[4],
    void *workspace, size_t workspace_bytes, pvnet_stream_t stream)
{
    const KpArgs kp = {hcoords, ver_dim / 2, hcoords_f64 != 0, use_motion != 0};
    return seg_vertex_losses_backward(seg_pred, seg_strides, mask, mask_elem_size, mask_strides, vertex_pred,
                                      pred_strides, nullptr, nullptr, &kp, vertex_weights, weight_strides, b, h, w, C,
                                      ver_dim, sigma, normalize, grad_loss_seg, grad_loss_vertex, grad_seg,
                                      grad_seg_strides, grad_vertex, grad_vertex_strides, workspace, workspace_bytes,
                                      stream);
}

int pvnet_vertex_targets(const void *mask, int mask_elem_size, const int64_t mask_strides[3], const void *hcoords,
                         int hcoords_f64, int b, int h, int w, int K, int use_motion, float *vertex_out,
                         pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && K >= 1, "non-positive dimension (b=%d, h=%d, w=%d, K=%d)", b, h, w, K);
    PV_CHECK_ARG(b <= 65535, "batch %d above 65535", b);
    PV_CHECK_ARG(mask && mask_strides && hcoords && vertex_out, "null pointer (mask, mask_strides, hcoords, vertex_out)");
    PV_CHECK_ARG(mask_elem_size == 1 || mask_elem_size == 4 || mask_elem_size == 8, "mask_elem_size %d is not 1, 4 or 8",
                 mask_elem_size);
    PV_CHECK_ARG(mask_strides[2] == 1, "unit stride along w is not 1 (mask %lld)", (long long)mask_strides[2]);
    PV_CHECK_ARG((long long)h * ((w + 3) / 4) <= 0x7fffffffLL - LS_QPB, "image of %d x %d pixels too large", h, w);
    VtArgs a = {};
    a.mask = mask, a.m_b = mask_strides[0], a.m_h = mask_strides[1], a.out = vertex_out;
    a.h = h, a.w = w, a.qw = (w + 3) / 4, a.nquads = h * a.qw;
    a.mvec = aligned(mask, 4 * mask_elem_size) && strides_ok(mask_strides, 2);
    a.ovec = aligned(vertex_out, 16) && w % 4 == 0;
    const KpArgs kp = {hcoords, K, hcoords_f64 != 0, use_motion != 0};
    const dim3 grid(ls_chunks(h, w), b);
    cudaStream_t st = (cudaStream_t)stream;
    if (mask_elem_size == 8)
        k_vertex_targets<long long><<<grid, LS_THREADS, 0, st>>>(a, kp);
    else if (mask_elem_size == 4)
        k_vertex_targets<int><<<grid, LS_THREADS, 0, st>>>(a, kp);
    else
        k_vertex_targets<unsigned char><<<grid, LS_THREADS, 0, st>>>(a, kp);
    PV_LAUNCHED(mask_elem_size == 8 ? "k_vertex_targets<int64>"
                : mask_elem_size == 4 ? "k_vertex_targets<int32>" : "k_vertex_targets<uint8>");
    return PVNET_OK;
}

}  // extern "C"
