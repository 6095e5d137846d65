/* extend_oracle.c -- TEST INFRASTRUCTURE ONLY: farthest point sampling and binary mesh rasterisation restated in C
 * from the semantics of the reference's lib/utils/extend_utils/src/{farthest_point_sampling,mesh_rasterization}.cpp
 * (DESIGN.md §11), one statement per rounded operation.  Built by oracle/extend.mk with -ffp-contract=off, so no
 * product or sum is fused, as in the reference's own binary.
 *
 *   pvo_farthest_point_sampling(pts [b,pn,3], start [b] or NULL (init_center), b, pn, sn, idxs [b,sn])
 *   pvo_mesh_binary_rasterization(tris [b,tn,3,2], b, tn, h, w, mask [b,h,w])     (mask is overwritten)
 */
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define API __attribute__((visibility("default")))

static float sqdist(const float *p, float cx, float cy, float cz)
{
    const float dx = p[0] - cx, dy = p[1] - cy, dz = p[2] - cz;
    const float xx = dx * dx, yy = dy * dy, zz = dz * dz;
    const float s = xx + yy;
    return s + zz;
}

/* the first index of the largest min_dist > 0 among unselected points, 0 if there is none */
static int argmax(const float *min_dist, const unsigned char *sel, int pn)
{
    int best = 0;
    float bd = 0.f;
    for (int i = 0; i < pn; ++i)
        if (!sel[i] && min_dist[i] > bd) {
            best = i;
            bd = min_dist[i];
        }
    return best;
}

static void fps_one(const float *pts, const int32_t *start, int pn, int sn, int32_t *idxs)
{
    float *md = malloc(sizeof(float) * (size_t)pn);
    unsigned char *sel = calloc((size_t)pn, 1);
    int cur;
    if (start) {
        int s = *start % pn;
        cur = s < 0 ? s + pn : s;
        for (int i = 0; i < pn; ++i) md[i] = FLT_MAX;
    } else {
        float hi[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX}, lo[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
        for (int i = 0; i < pn; ++i)
            for (int k = 0; k < 3; ++k) {
                const float v = pts[(size_t)i * 3 + k];
                hi[k] = (hi[k] < v) ? v : hi[k];          /* std::max(hi, v) */
                lo[k] = (v < lo[k]) ? v : lo[k];          /* std::min(lo, v) */
            }
        float c[3];
        for (int k = 0; k < 3; ++k) {
            const float s = hi[k] + lo[k];
            c[k] = s * 0.5f;                              /* (max + min) * (1.f / 2.f) */
        }
        for (int i = 0; i < pn; ++i) {
            const float d = sqdist(pts + (size_t)i * 3, c[0], c[1], c[2]);
            md[i] = (FLT_MAX < d) ? FLT_MAX : d;          /* std::min(d, FLT_MAX) */
        }
        cur = argmax(md, sel, pn);
    }
    for (int r = 0; r < sn; ++r) {
        sel[cur] = 1;
        idxs[r] = cur;
        if (r == sn - 1) break;
        const float *c = pts + (size_t)cur * 3;
        const float cx = c[0], cy = c[1], cz = c[2];
        for (int i = 0; i < pn; ++i) {
            if (sel[i]) continue;
            const float d = sqdist(pts + (size_t)i * 3, cx, cy, cz);
            if (d < md[i]) md[i] = d;
        }
        cur = argmax(md, sel, pn);
    }
    free(md);
    free(sel);
}

API void pvo_farthest_point_sampling(const float *pts, const int32_t *start, int b, int pn, int sn, int32_t *idxs)
{
#pragma omp parallel for schedule(dynamic)
    for (int i = 0; i < b; ++i)
        fps_one(pts + (size_t)i * pn * 3, start ? start + i : NULL, pn, sn, idxs + (size_t)i * sn);
}

static int same_side(float x0, float y0, float x1, float y1, float tx0, float ty0, float tx1, float ty1)
{
    const float dx = x1 - x0, dy = y1 - y0;
    const float nx = -dy, ny = dx;
    const float dx0 = tx0 - x0, dy0 = ty0 - y0, dx1 = tx1 - x0, dy1 = ty1 - y0;
    const float a0 = dx0 * nx, b0 = dy0 * ny, a1 = dx1 * nx, b1 = dy1 * ny;
    const float val0 = a0 + b0, val1 = a1 + b1;
    const float prod = val0 * val1;
    return prod >= 0.f;
}

static void raster_one(const float *t, int tn, int h, int w, unsigned char *mask)
{
    for (int ti = 0; ti < tn; ++ti) {
        const float *v = t + (size_t)ti * 6;
        const float x0 = v[0], y0 = v[1], x1 = v[2], y1 = v[3], x2 = v[4], y2 = v[5];
        float minx = x0, maxx = x0, miny = y0, maxy = y0;  /* std::min({..}) / std::max({..}) */
        if (x1 < minx) minx = x1;
        if (x2 < minx) minx = x2;
        if (maxx < x1) maxx = x1;
        if (maxx < x2) maxx = x2;
        if (y1 < miny) miny = y1;
        if (y2 < miny) miny = y2;
        if (maxy < y1) maxy = y1;
        if (maxy < y2) maxy = y2;
        minx = (0.f < minx) ? minx : 0.f;
        miny = (0.f < miny) ? miny : 0.f;
        const float wl = (float)(w - 2), hl = (float)(h - 2);
        maxx = (maxx < wl) ? maxx : wl;
        maxy = (maxy < hl) ? maxy : hl;
        const float ex = maxx + 1.f, ey = maxy + 1.f;
        /* where int() would be undefined the triangle covers no in-range pixel */
        if (!(minx < 2147483648.f) || !(miny < 2147483648.f) || !(ex >= -2147483648.f) || !(ey >= -2147483648.f))
            continue;
        const int begx = (int)minx, endx = (int)ex, begy = (int)miny, endy = (int)ey;
        for (int yi = begy; yi <= endy; ++yi)
            for (int xi = begx; xi <= endx; ++xi) {
                const float px = (float)xi, py = (float)yi;
                if (same_side(x0, y0, x1, y1, x2, y2, px, py) && same_side(x1, y1, x2, y2, x0, y0, px, py) &&
                    same_side(x2, y2, x0, y0, x1, y1, px, py))
                    mask[(size_t)yi * w + xi] = 1;
            }
    }
}

API void pvo_mesh_binary_rasterization(const float *tris, int b, int tn, int h, int w, unsigned char *mask)
{
#pragma omp parallel for schedule(dynamic)
    for (int i = 0; i < b; ++i) {
        unsigned char *m = mask + (size_t)i * h * w;
        memset(m, 0, (size_t)h * w);
        raster_one(tris + (size_t)i * tn * 6, tn, h, w, m);
    }
}
