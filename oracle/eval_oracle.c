/*
 * eval_oracle.c -- CPU restatement of the reference's nearest-point kernel.
 *
 * TEST INFRASTRUCTURE ONLY, like pvnet_oracle.c: nothing in pvnet_b200/ includes, links, loads or calls it;
 * oracle/eval_oracle.py binds it for the tests and benchmarks/eval_metrics.py.
 *
 *   pvo_find_nearest_point_idx   lib/utils/extend_utils/src/nearest_neighborhood.cu:48-117
 *                                (findNearestPoint{3D,2D}IdxKernel, exclude_self = 0)
 *
 * Floating point: the rounding sequence nvcc 12.9 emits for the reference kernel on sm_90a (SASS, DESIGN.md §2
 * "FP sequence"): dy*dy rounded, then fma(dx,dx,.), then fma(dz,dz,.); the FSETP.GEU update is `d < best`, so a
 * NaN never wins and ties keep the lowest index.  Built with -ffp-contract=off (oracle/eval.mk) the fmaf calls
 * are the only fused operations, so this file is bit-exact to the reference kernel.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#define PVO_API __attribute__((visibility("default")))

/* ref [b,pn1,dim], que [b,pn2,dim], idxs [b,pn2]; dim 2 or 3 */
PVO_API void pvo_find_nearest_point_idx(const float *ref, const float *que, int32_t *idxs,
                                        int b, int pn1, int pn2, int dim)
{
#pragma omp parallel for collapse(2) schedule(static)
    for (int bi = 0; bi < b; ++bi) {
        for (int qi = 0; qi < pn2; ++qi) {
            const float *q = que + ((size_t)bi * pn2 + qi) * dim;
            const float *r = ref + (size_t)bi * pn1 * dim;
            float best = 3.402823466e+38F;      /* FLT_MAX */
            int32_t bidx = 0;
            for (int k = 0; k < pn1; ++k) {
                const float dx = r[(size_t)k * dim] - q[0];
                const float dy = r[(size_t)k * dim + 1] - q[1];
                float d = fmaf(dx, dx, dy * dy);
                if (dim == 3) {
                    const float dz = r[(size_t)k * dim + 2] - q[2];
                    d = fmaf(dz, dz, d);
                }
                if (d < best) {
                    best = d;
                    bidx = k;
                }
            }
            idxs[(size_t)bi * pn2 + qi] = bidx;
        }
    }
}
