/*
 * pvnet_oracle.c -- CPU restatement of the reference's RANSAC voting kernels.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in pvnet_b200/ may include, link, load or
 * call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it, and only as the checker or the
 * timed CPU baseline -- never as the product path.
 *
 * What is restated (paths relative to the reference project):
 *   pvo_generate_hypothesis   lib/ransac_voting_gpu_layer/src/ransac_voting_kernel.cu:11-49
 *   pvo_voting_for_hypothesis lib/ransac_voting_gpu_layer/src/ransac_voting_kernel.cu:88-126
 *   pvo_generate_hypothesis_vp / pvo_voting_for_hypothesis_vp
 *                             lib/ransac_voting_gpu_layer/src/ransac_voting_kernel.cu:170-230, :263-305
 *   pvo_vote_counts           same predicate, summed over pixels the way
 *                             lib/ransac_voting_gpu_layer/ransac_voting_gpu.py:561 does
 *                             (torch.sum(cur_inlier, 2)) without storing the u8 tensor
 *
 * Floating point.  The reference .cu is built by nvcc with its defaults
 * (-fmad=true, -prec-div=true, -prec-sqrt=true).  The exact rounding sequence
 * below was read off the SASS nvcc 12.9 emits (see DESIGN.md,
 * "FP sequence"):  individually rounded FP32 mul/add, single-rounding fmaf where
 * ptxas contracted, correctly rounded sqrtf and '/', and the `< 1e-6` tests
 * done after promotion to double.  x86-64 fmaf/sqrtf/'/' are correctly rounded,
 * so built with -ffp-contract=off this file is bit-exact to the GPU kernels.
 *
 * Parity pin: tests/test_gpu_reference_layer.py runs the reference .cu itself
 * (compiled verbatim into oracle/_ref by oracle/Makefile) on the GPU and
 * checks it against these functions bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(_OPENMP)
#include <omp.h>
#endif

#define PVO_API __attribute__((visibility("default")))

/* ransac_voting_kernel.cu:11-49.  direct [tn,vn,2], coords [tn,2] (x,y),
 * idxs [hn,vn,2] int32, hypo [hn,vn,2].  hypo is zero-filled first, as the
 * launcher does with at::zeros (ransac_voting_kernel.cu:75); degenerate pairs
 * therefore stay (0,0) (early returns at :42-43). */
PVO_API void pvo_generate_hypothesis(const float *direct, const float *coords,
                                     const int32_t *idxs, float *hypo,
                                     int tn, int vn, int hn)
{
    (void)tn;
    memset(hypo, 0, sizeof(float) * (size_t)hn * vn * 2);
    for (int hi = 0; hi < hn; ++hi) {
        for (int vi = 0; vi < vn; ++vi) {
            const int t0 = idxs[(hi * vn + vi) * 2];
            const int t1 = idxs[(hi * vn + vi) * 2 + 1];
            const float d0x = direct[((size_t)t0 * vn + vi) * 2];
            const float d0y = direct[((size_t)t0 * vn + vi) * 2 + 1];
            const float d1x = direct[((size_t)t1 * vn + vi) * 2];
            const float d1y = direct[((size_t)t1 * vn + vi) * 2 + 1];
            const float cx0 = coords[(size_t)t0 * 2], cy0 = coords[(size_t)t0 * 2 + 1];
            const float cx1 = coords[(size_t)t1 * 2], cy1 = coords[(size_t)t1 * 2 + 1];
            /* source: nx=d_y, ny=-d_x; negations fold into the signs below */
            const float p = d0y * d1x;
            const float q = d0x * d1y;
            const float det_y = p - q;              /* nx1*ny0-nx0*ny1 */
            if ((double)fabsf(det_y) < 1e-6) continue;
            const float det_x = q - p;              /* ny1*nx0-ny0*nx1 */
            if ((double)fabsf(det_x) < 1e-6) continue;
            const float s1 = fmaf(d1y, cx1, -(d1x * cy1));
            const float s0 = fmaf(d0y, cx0, -(d0x * cy0));
            const float y = fmaf(d1y, s0, -(d0y * s1)) / det_y;
            const float x = fmaf(-d1x, s0, d0x * s1) / det_x;
            hypo[(hi * vn + vi) * 2] = x;
            hypo[(hi * vn + vi) * 2 + 1] = y;
        }
    }
}

/* ransac_voting_kernel.cu:107-125, one (hypothesis, keypoint, pixel) test */
static inline int pvo_is_inlier(float nx, float ny, float cx, float cy,
                                float hx, float hy, float thresh)
{
    const float dx = hx - cx;
    const float dy = hy - cy;
    const float norm1 = sqrtf(fmaf(nx, nx, ny * ny));
    const float norm2 = sqrtf(fmaf(dx, dx, dy * dy));
    if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) return 0;
    const float num = fmaf(dx, nx, dy * ny);
    const float den = norm1 * norm2;
    const float ang = num / den;
    return ang > thresh;
}

/* ransac_voting_kernel.cu:88-126.  inliers [hn,vn,tn] u8 is only ever SET to 1
 * (the caller zero-fills it, ransac_voting_gpu.py:557). */
PVO_API void pvo_voting_for_hypothesis(const float *direct, const float *coords,
                                       const float *hypo, uint8_t *inliers,
                                       int tn, int vn, int hn, float thresh)
{
#pragma omp parallel for collapse(2) schedule(static)
    for (int hi = 0; hi < hn; ++hi) {
        for (int vi = 0; vi < vn; ++vi) {
            const float hx = hypo[(hi * vn + vi) * 2];
            const float hy = hypo[(hi * vn + vi) * 2 + 1];
            uint8_t *row = inliers + ((size_t)hi * vn + vi) * tn;
            for (int ti = 0; ti < tn; ++ti) {
                if (pvo_is_inlier(direct[((size_t)ti * vn + vi) * 2],
                                  direct[((size_t)ti * vn + vi) * 2 + 1],
                                  coords[(size_t)ti * 2], coords[(size_t)ti * 2 + 1],
                                  hx, hy, thresh))
                    row[ti] = 1;
            }
        }
    }
}

/* counts[hi,vi] = sum_t inlier(hi,vi,t)  (ransac_voting_gpu.py:557-561 without
 * the [hn,vn,tn] tensor).  Same predicate, same result as summing the above. */
PVO_API void pvo_vote_counts(const float *direct, const float *coords,
                             const float *hypo, int32_t *counts,
                             int tn, int vn, int hn, float thresh)
{
#pragma omp parallel for collapse(2) schedule(static)
    for (int hi = 0; hi < hn; ++hi) {
        for (int vi = 0; vi < vn; ++vi) {
            const float hx = hypo[(hi * vn + vi) * 2];
            const float hy = hypo[(hi * vn + vi) * 2 + 1];
            int32_t c = 0;
            for (int ti = 0; ti < tn; ++ti) {
                c += pvo_is_inlier(direct[((size_t)ti * vn + vi) * 2],
                                   direct[((size_t)ti * vn + vi) * 2 + 1],
                                   coords[(size_t)ti * 2], coords[(size_t)ti * 2 + 1],
                                   hx, hy, thresh);
            }
            counts[hi * vn + vi] = c;
        }
    }
}

/* ransac_voting_kernel.cu:170-230.  hypo [hn,vn,3] homogeneous intersection of the two pixels' lines;
 * rounding sequence as nvcc compiles the reference (SASS): see exact_vp_hypothesis in
 * pvnet_b200/csrc/vote.cu for the line-by-line mapping. */
PVO_API void pvo_generate_hypothesis_vp(const float *direct, const float *coords, const int32_t *idxs,
                                        float *hypo, int tn, int vn, int hn)
{
    (void)tn;
    for (int hi = 0; hi < hn; ++hi) {
        for (int vi = 0; vi < vn; ++vi) {
            const int t0 = idxs[(hi * vn + vi) * 2], t1 = idxs[(hi * vn + vi) * 2 + 1];
            const float dx0 = direct[((size_t)t0 * vn + vi) * 2], dy0 = direct[((size_t)t0 * vn + vi) * 2 + 1];
            const float dx1 = direct[((size_t)t1 * vn + vi) * 2], dy1 = direct[((size_t)t1 * vn + vi) * 2 + 1];
            const float cx0 = coords[(size_t)t0 * 2], cy0 = coords[(size_t)t0 * 2 + 1];
            const float cx1 = coords[(size_t)t1 * 2], cy1 = coords[(size_t)t1 * 2 + 1];
            const float lz0 = fmaf(dx0, cy0, -(dy0 * cx0));
            const float lz1 = fmaf(dx1, cy1, -(dy1 * cx1));
            float z = fmaf(dx0, dy1, -(dy0 * dx1));
            float x = fmaf(dx1, lz0, -(dx0 * lz1));
            float y = fmaf(dy1, lz0, -(dy0 * lz1));
            const float vx0 = dx0 * fmaf(-cx0, z, x), vx1 = dx1 * fmaf(-cx1, z, x);
            const float vy0 = dy0 * fmaf(-cy0, z, y), vy1 = dy1 * fmaf(-cy1, z, y);
            if (vx0 < 0.f && vx1 < 0.f && vy0 < 0.f && vy1 < 0.f) {
                x = -x;
                y = -y;
                z = -z;
            }
            if (fminf(vx0 * vx1, vy0 * vy1) < 0.f) x = y = z = 0.f;
            hypo[(hi * vn + vi) * 3] = x;
            hypo[(hi * vn + vi) * 3 + 1] = y;
            hypo[(hi * vn + vi) * 3 + 2] = z;
        }
    }
}

/* ransac_voting_kernel.cu:263-305; inliers [hn,vn,tn] u8 only SET */
PVO_API void pvo_voting_for_hypothesis_vp(const float *direct, const float *coords, const float *hypo,
                                          uint8_t *inliers, int tn, int vn, int hn, float thresh)
{
#pragma omp parallel for collapse(2) schedule(static)
    for (int hi = 0; hi < hn; ++hi) {
        for (int vi = 0; vi < vn; ++vi) {
            const float hx = hypo[(hi * vn + vi) * 3], hy = hypo[(hi * vn + vi) * 3 + 1], hz = hypo[(hi * vn + vi) * 3 + 2];
            uint8_t *row = inliers + ((size_t)hi * vn + vi) * tn;
            for (int ti = 0; ti < tn; ++ti) {
                const float dx = direct[((size_t)ti * vn + vi) * 2], dy = direct[((size_t)ti * vn + vi) * 2 + 1];
                const float fx = fmaf(-coords[(size_t)ti * 2], hz, hx), fy = fmaf(-coords[(size_t)ti * 2 + 1], hz, hy);
                const float norm1 = sqrtf(fmaf(dx, dx, dy * dy)), norm2 = sqrtf(fmaf(fx, fx, fy * fy));
                if ((double)norm1 < 1e-6 || (double)norm2 < 1e-6) continue;
                const float vx = fx * dx, vy = fy * dy;
                const float ang = (vx + vy) / (norm2 * norm1);
                if (fminf(vx, vy) < 0.f) continue;
                if (fabsf(ang) > thresh) row[ti] = 1;
            }
        }
    }
}

PVO_API int pvo_num_threads(void)
{
#if defined(_OPENMP)
    return omp_get_max_threads();
#else
    return 1;
#endif
}

PVO_API void pvo_set_num_threads(int n)
{
#if defined(_OPENMP)
    omp_set_num_threads(n);
#else
    (void)n;
#endif
}
