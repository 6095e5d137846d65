// render.cu -- depth and flat-shaded RGB of a triangle mesh at a batch of poses: the reference's OpenGL render
// backend (lib/utils/opengl_render_backend.py `render`, flat shading, no texture) on the device (DESIGN.md §24).
//
// Conventions: output pixel (r, c) samples the image point (c + 0.5, r + 0.5) in OpenCV pixel coordinates, where
// u = fx X/Z + s Y/Z + cx and v = fy Y/Z + cy -- what the reference's y-down projection, the yz flip of its view
// matrix, GL's viewport transform and the row flip on readback give together.  Vertices, poses, K and the clip
// planes are fp32 as the reference hands them to GL; the geometry is fp64, one rounded __d*_rn intrinsic per
// operation in a fixed order, so oracle/render_oracle.py restates it bit for bit.
//
// Per (pose, face): camera-space vertices V_i = R X_i + t and homogeneous image points h_i = K V_i.  The edge
// opposite vertex i has the vector c_i = h_j x h_k (j, k the next two vertices), computed with the lower vertex
// index first and negated for the other orientation, so faces that share an edge get exactly opposite edge values.
// At p = (c + 0.5, r + 0.5, 1): E_i = c_i . p, S = E_0 + E_1 + E_2, and lambda_i = E_i / S are the
// perspective-correct barycentrics; Z = sum lambda_i Z_i.  The pixel is covered when S != 0, every E_i is 0 or has
// S's sign, and near <= Z <= far: a per-fragment test that handles faces crossing the camera plane with no
// clipping step.  The covering face with the smallest (fp32(Z), face index) wins, through a 64-bit atomicMin on
// bits(fp32(Z)) << 32 | face; Z >= near > 0, so the float bits order like the depths.
//
// Launches: the keys are set to all ones (cudaMemsetAsync); k_render_raster takes the flattened (pose, face)
// pairs, a warp per face walking its pixel box, boxes above RD_BIG pixels deferred to the whole CTA; k_render_resolve
// writes depth and RGB per pixel, recomputing the winner's barycentrics with the same face_setup/face_fragment.
#include "common.cuh"

#include <cmath>

namespace {

constexpr int RD_WARPS = 8;
constexpr int RD_THREADS = RD_WARPS * 32;
constexpr int RD_BIG = 1024;                      // box pixels above which a face is shared by the CTA's warps
constexpr int RD_RESOLVE_THREADS = 256;
constexpr unsigned long long RD_EMPTY = ~0ull;    // no face covers the pixel

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }
// (a0 b0 + a1 b1) + a2 b2
__device__ __forceinline__ double dot3(const double *a, const double *b)
{
    return da(da(dm(a[0], b[0]), dm(a[1], b[1])), dm(a[2], b[2]));
}
__device__ __forceinline__ void cross3(const double *a, const double *b, double *o)
{
    o[0] = ds(dm(a[1], b[2]), dm(a[2], b[1]));
    o[1] = ds(dm(a[2], b[0]), dm(a[0], b[2]));
    o[2] = ds(dm(a[0], b[1]), dm(a[1], b[0]));
}

struct Face {
    double c[3][3];                               // edge vectors, c[i] opposite vertex i
    double z[3];                                  // camera-space depths
    double V[3][3];                               // camera-space vertices (the shading reads them)
    double h[3][3];                               // homogeneous image points K V_i (the box reads them)
    int vi[3];
};

// The face's camera-space vertices, edge vectors and depths.  false: an index outside [0, nv), a repeated index, a
// non-finite h_i, or D = c_0 . h_0 (the determinant of the h_i) zero or non-finite: such a face covers nothing.
// pose: [3,4] fp32 row-major (R | t); Km: [3,3] fp32 (K[1,0] and the third row are not read, as GL's projection
// built from K does not read them).
__device__ __forceinline__ bool face_setup(const float *__restrict__ verts, const int32_t *__restrict__ faces, int f,
                                           int nv, const float *__restrict__ pose, const float *__restrict__ Km,
                                           Face &F)
{
    double (&h)[3][3] = F.h;
    const double fx = Km[0], sk = Km[1], cx = Km[2], fy = Km[4], cy = Km[5];
    for (int i = 0; i < 3; ++i) {
        const int v = __ldg(faces + static_cast<size_t>(f) * 3 + i);
        if (v < 0 || v >= nv) return false;
        F.vi[i] = v;
        const double x = __ldg(verts + static_cast<size_t>(v) * 3), y = __ldg(verts + static_cast<size_t>(v) * 3 + 1),
                     z = __ldg(verts + static_cast<size_t>(v) * 3 + 2);
#pragma unroll
        for (int r = 0; r < 3; ++r)
            F.V[i][r] = da(da(da(dm((double)pose[r * 4], x), dm((double)pose[r * 4 + 1], y)),
                              dm((double)pose[r * 4 + 2], z)),
                           (double)pose[r * 4 + 3]);
        h[i][0] = da(da(dm(fx, F.V[i][0]), dm(sk, F.V[i][1])), dm(cx, F.V[i][2]));
        h[i][1] = da(dm(fy, F.V[i][1]), dm(cy, F.V[i][2]));
        h[i][2] = F.V[i][2];
        F.z[i] = F.V[i][2];
        if (!(isfinite(h[i][0]) && isfinite(h[i][1]) && isfinite(h[i][2]))) return false;
    }
    if (F.vi[0] == F.vi[1] || F.vi[1] == F.vi[2] || F.vi[0] == F.vi[2]) return false;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const int j = (i + 1) % 3, k = (i + 2) % 3;
        if (F.vi[j] < F.vi[k]) {
            cross3(h[j], h[k], F.c[i]);
        } else {
            cross3(h[k], h[j], F.c[i]);
            F.c[i][0] = -F.c[i][0];
            F.c[i][1] = -F.c[i][1];
            F.c[i][2] = -F.c[i][2];
        }
    }
    const double D = dot3(F.c[0], h[0]);
    return isfinite(D) && D != 0.0;
}

// The covering test at pixel (col, row); on true, lam and Z hold the barycentrics and the depth.
__device__ __forceinline__ bool face_fragment(const Face &F, int col, int row, double nearp, double farp,
                                              double lam[3], double &Z)
{
    const double px = col + 0.5, py = row + 0.5;
    double E[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) E[i] = da(da(dm(F.c[i][0], px), dm(F.c[i][1], py)), F.c[i][2]);
    const double S = da(da(E[0], E[1]), E[2]);
    if (S > 0.0) {
        if (!(E[0] >= 0.0 && E[1] >= 0.0 && E[2] >= 0.0)) return false;
    } else if (S < 0.0) {
        if (!(E[0] <= 0.0 && E[1] <= 0.0 && E[2] <= 0.0)) return false;
    } else {
        return false;                              // S == 0 or NaN
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) lam[i] = dd(E[i], S);
    Z = da(da(dm(lam[0], F.z[0]), dm(lam[1], F.z[1])), dm(lam[2], F.z[2]));
    return Z >= nearp && Z <= farp;
}

struct Box {
    int bx, ex, by, ey;                           // inclusive
};

// A conservative pixel box.  When every vertex has Z >= near, every covered point projects into the hull of the
// projected vertices: their box, widened to the pixels whose centres could round onto it plus one pixel.  A face
// with a vertex nearer than near gets the whole image.  false: no pixel can be covered -- the box misses the image,
// or every vertex is nearer than near * (1 - 2^-20), below which no covered depth (a convex combination of the
// vertex depths, a few ulps off) reaches near.
__device__ __forceinline__ bool face_box(const Face &F, int h, int w, double nearp, Box &B)
{
    const double zmin = fmin(fmin(F.z[0], F.z[1]), F.z[2]), zmax = fmax(fmax(F.z[0], F.z[1]), F.z[2]);
    if (zmax < nearp * (1.0 - 0x1p-20)) return false;
    if (zmin < nearp) {
        B.bx = 0;
        B.by = 0;
        B.ex = w - 1;
        B.ey = h - 1;
        return true;
    }
    double u0 = INFINITY, u1 = -INFINITY, v0 = INFINITY, v1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double u = F.h[i][0] / F.h[i][2], v = F.h[i][1] / F.h[i][2];
        u0 = fmin(u0, u);
        u1 = fmax(u1, u);
        v0 = fmin(v0, v);
        v1 = fmax(v1, v);
    }
    const double bx = fmax(floor(u0 - 0.5) - 1.0, 0.0), ex = fmin(ceil(u1 - 0.5) + 1.0, w - 1.0);
    const double by = fmax(floor(v0 - 0.5) - 1.0, 0.0), ey = fmin(ceil(v1 - 0.5) + 1.0, h - 1.0);
    if (!(bx <= ex && by <= ey)) return false;
    B.bx = static_cast<int>(bx);
    B.ex = static_cast<int>(ex);
    B.by = static_cast<int>(by);
    B.ey = static_cast<int>(ey);
    return true;
}

__device__ __forceinline__ void raster_pixel(const Face &F, int f, int col, int row, int w, double nearp,
                                             double farp, unsigned long long *__restrict__ keys)
{
    double lam[3], Z;
    if (!face_fragment(F, col, row, nearp, farp, lam, Z)) return;
    const unsigned long long key =
        (static_cast<unsigned long long>(__float_as_uint(__double2float_rn(Z))) << 32) | static_cast<uint32_t>(f);
    unsigned long long *k = keys + static_cast<size_t>(row) * w + col;
    if (*k > key) atomicMin(k, key);             // keys only decrease: a key at or below ours makes the atomic a no-op
}

struct Scene {
    const float *verts;
    const int32_t *faces;
    const float *colors;                          // [nv,3] or NULL (0.5 grey)
    const float *poses;                           // [b,3,4]
    const float *K;                               // [3,3] or [b,3,3]
    int kstride;                                  // 0 or 9
    int nv, nf, h, w;
    double nearp, farp;
};

// grid: ceil(b * nf / RD_WARPS) CTAs; warp w of CTA c takes pair c * RD_WARPS + w of the flattened (pose, face)
// pairs.  Faces whose box has more than RD_BIG pixels are handled after the others by the whole CTA, its warps
// taking every RD_WARPS-th row.
__global__ void __launch_bounds__(RD_THREADS)
    k_render_raster(Scene s, int total, unsigned long long *__restrict__ keys)
{
    __shared__ int s_big[RD_WARPS];
    __shared__ int s_nbig;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_nbig = 0;
    __syncthreads();
    const int t = blockIdx.x * RD_WARPS + warp;
    const size_t hw = static_cast<size_t>(s.h) * s.w;
    if (t < total) {
        const int img = t / s.nf, f = t - img * s.nf;
        Face F;
        Box B;
        if (face_setup(s.verts, s.faces, f, s.nv, s.poses + static_cast<size_t>(img) * 12,
                       s.K + static_cast<size_t>(img) * s.kstride, F) &&
            face_box(F, s.h, s.w, s.nearp, B)) {
            const int bw = B.ex - B.bx + 1;
            const long long npix = static_cast<long long>(bw) * (B.ey - B.by + 1);
            if (npix > RD_BIG) {
                if (lane == 0) s_big[atomicAdd(&s_nbig, 1)] = t;
            } else {
                unsigned long long *k = keys + img * hw;
                for (int p = lane; p < npix; p += 32)
                    raster_pixel(F, f, B.bx + p % bw, B.by + p / bw, s.w, s.nearp, s.farp, k);
            }
        }
    }
    __syncthreads();
    for (int i = 0; i < s_nbig; ++i) {
        const int tb = s_big[i];
        const int img = tb / s.nf, f = tb - img * s.nf;
        Face F;
        Box B;
        face_setup(s.verts, s.faces, f, s.nv, s.poses + static_cast<size_t>(img) * 12,
                   s.K + static_cast<size_t>(img) * s.kstride, F);
        face_box(F, s.h, s.w, s.nearp, B);
        unsigned long long *k = keys + img * hw;
        for (int row = B.by + warp; row <= B.ey; row += RD_WARPS)
            for (int col = B.bx + lane; col <= B.ex; col += 32) raster_pixel(F, f, col, row, s.w, s.nearp, s.farp, k);
    }
}

// np.round(fp32(x) * 255) to uint8: fp32 multiply, round half to even, clamped to [0, 255] (NaN gives 0)
__device__ __forceinline__ uint8_t to_u8(double x)
{
    const float r = rintf(__fmul_rn(__double2float_rn(x), 255.f));
    return r >= 255.f ? 255 : (r > 0.f ? static_cast<uint8_t>(r) : 0);
}

// flat shading (opengl_render_backend.py:50-75 with u_light_eye_pos at the camera): light_w * sum lambda_i c_i
__device__ __forceinline__ void shade(const Face &F, const double lam[3], const float *__restrict__ colors,
                                      double ambient, uint8_t *__restrict__ out)
{
    // the unit face normal turned toward the camera (n . V < 0), as cross(dFdx, dFdy) of a visible plane is
    double d1[3], d2[3], m[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        d1[r] = ds(F.V[1][r], F.V[0][r]);
        d2[r] = ds(F.V[2][r], F.V[0][r]);
    }
    cross3(d1, d2, m);
    if (dot3(m, F.V[0]) > 0.0) {
        m[0] = -m[0];
        m[1] = -m[1];
        m[2] = -m[2];
    }
    const double mn = __dsqrt_rn(dot3(m, m));
    double n[3], L[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) n[r] = dd(m[r], mn);
    // L = normalize(sum lambda_i v_L,i), v_L,i = -V_i / |V_i|
    double u[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double vn = __dsqrt_rn(dot3(F.V[i], F.V[i]));
#pragma unroll
        for (int r = 0; r < 3; ++r) u[i][r] = -dd(F.V[i][r], vn);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) L[r] = da(da(dm(lam[0], u[0][r]), dm(lam[1], u[1][r])), dm(lam[2], u[2][r]));
    const double ln = __dsqrt_rn(dot3(L, L));
#pragma unroll
    for (int r = 0; r < 3; ++r) L[r] = dd(L[r], ln);
    const double dt = dot3(L, n);
    double lw = da(ambient, dt > 0.0 ? dt : 0.0);
    lw = lw > 1.0 ? 1.0 : lw;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        double c[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) c[i] = colors ? __ldg(colors + static_cast<size_t>(F.vi[i]) * 3 + ch) : 0.5;
        out[ch] = to_u8(dm(lw, da(da(dm(lam[0], c[0]), dm(lam[1], c[1])), dm(lam[2], c[2]))));
    }
}

// one thread per output pixel of the batch
__global__ void __launch_bounds__(RD_RESOLVE_THREADS)
    k_render_resolve(Scene s, long long npix, double ambient, uchar4 bg, const unsigned long long *__restrict__ keys,
                     float *__restrict__ depth, uint8_t *__restrict__ rgb)
{
    const long long i = static_cast<long long>(blockIdx.x) * RD_RESOLVE_THREADS + threadIdx.x;
    if (i >= npix) return;
    const unsigned long long key = keys[i];
    if (key == RD_EMPTY) {
        if (depth) depth[i] = 0.f;
        if (rgb) {
            rgb[i * 3] = bg.x;
            rgb[i * 3 + 1] = bg.y;
            rgb[i * 3 + 2] = bg.z;
        }
        return;
    }
    if (depth) depth[i] = __uint_as_float(static_cast<uint32_t>(key >> 32));
    if (!rgb) return;
    const long long hw = static_cast<long long>(s.h) * s.w;
    const int img = static_cast<int>(i / hw), p = static_cast<int>(i - img * hw);
    const int row = p / s.w, col = p - row * s.w, f = static_cast<int>(static_cast<uint32_t>(key));
    Face F;
    double lam[3], Z;
    // the winner passed both calls in the raster pass; they are pure functions of the same inputs
    face_setup(s.verts, s.faces, f, s.nv, s.poses + static_cast<size_t>(img) * 12,
               s.K + static_cast<size_t>(img) * s.kstride, F);
    face_fragment(F, col, row, s.nearp, s.farp, lam, Z);
    uint8_t c[3];
    shade(F, lam, s.colors, ambient, c);
    rgb[i * 3] = c[0];
    rgb[i * 3 + 1] = c[1];
    rgb[i * 3 + 2] = c[2];
}

uint8_t host_u8(float x)
{
    volatile float g = x * 255.f;                 // one rounded fp32 multiply
    const float r = rintf(g);
    return r >= 255.f ? 255 : (r > 0.f ? static_cast<uint8_t>(r) : 0);
}

}  // namespace

extern "C" {

int pvnet_render_workspace_bytes(int b, int h, int w, size_t *bytes)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1, "non-positive dimension (b=%d, h=%d, w=%d)", b, h, w);
    PV_CHECK_ARG(bytes, "null pointer");
    *bytes = static_cast<size_t>(b) * h * w * sizeof(unsigned long long);
    return PVNET_OK;
}

int pvnet_render_mesh(const float *verts, const int32_t *faces, const float *colors, int nv, int nf, const float *poses,
                      const float *K, int k_per_image, int b, int h, int w, float near_clip, float far_clip,
                      float ambient, const float *bg, float *depth, uint8_t *rgb, void *workspace,
                      size_t workspace_bytes, pvnet_stream_t stream)
{
    PV_CHECK_ARG(b >= 1 && h >= 1 && w >= 1 && nv >= 0 && nf >= 0,
                 "bad dimension (b=%d, h=%d, w=%d, nv=%d, nf=%d)", b, h, w, nv, nf);
    PV_CHECK_ARG(static_cast<long long>(h) * w <= INT32_MAX, "image %dx%d too large", h, w);
    PV_CHECK_ARG(static_cast<long long>(b) * nf <= INT32_MAX - RD_WARPS, "b * nf too large");
    PV_CHECK_ARG(static_cast<long long>(b) * h * w <= static_cast<long long>(INT32_MAX) * RD_RESOLVE_THREADS,
                 "b * h * w too large");
    PV_CHECK_ARG(std::isfinite(near_clip) && std::isfinite(far_clip) && near_clip > 0.f && near_clip < far_clip,
                 "clip planes must satisfy 0 < near < far (got %g, %g)", near_clip, far_clip);
    PV_CHECK_ARG(poses && K && (nf == 0 || faces) && (nv == 0 || verts), "null pointer");
    PV_CHECK_ARG(depth || rgb, "null pointer: neither depth nor rgb requested");
    size_t need = 0;
    pvnet_render_workspace_bytes(b, h, w, &need);
    PV_CHECK_ARG(workspace && workspace_bytes >= need, "workspace %zu bytes < %zu", workspace_bytes, need);
    unsigned long long *keys = static_cast<unsigned long long *>(workspace);
    const cudaStream_t st = (cudaStream_t)stream;
    PV_CUDA(cudaMemsetAsync(keys, 0xff, need, st));
    Scene s;
    s.verts = verts;
    s.faces = faces;
    s.colors = colors;
    s.poses = poses;
    s.K = K;
    s.kstride = k_per_image ? 9 : 0;
    s.nv = nv;
    s.nf = nf;
    s.h = h;
    s.w = w;
    s.nearp = near_clip;
    s.farp = far_clip;
    const int total = b * nf;
    if (total > 0) {
        k_render_raster<<<(total + RD_WARPS - 1) / RD_WARPS, RD_THREADS, 0, st>>>(s, total, keys);
        PV_LAUNCHED("k_render_raster");
    }
    const long long npix = static_cast<long long>(b) * h * w;
    const uchar4 bgc = make_uchar4(bg ? host_u8(bg[0]) : 0, bg ? host_u8(bg[1]) : 0, bg ? host_u8(bg[2]) : 0, 0);
    k_render_resolve<<<static_cast<unsigned>((npix + RD_RESOLVE_THREADS - 1) / RD_RESOLVE_THREADS),
                       RD_RESOLVE_THREADS, 0, st>>>(s, npix, ambient, bgc, keys, depth, rgb);
    PV_LAUNCHED("k_render_resolve");
    return PVNET_OK;
}

}  // extern "C"
