// pnp.cu -- uncertainty-driven PnP on the device (SURVEY.md section 8 row f-1): the consumer of the
// keypoints + covariances the voting layers produce, so that POSES are what leaves the GPU.
//
// Reference (per image, on the host after a device->host copy, tools/train_linemod.py:210-218):
//   lib/utils/evaluation_utils.py:170-181            weights = inv(sqrtm(cov)) per keypoint (zeros if cov[0,0] < 1e-6 / NaN)
//   lib/utils/extend_utils/extend_utils.py:84-88      P3P (OpenCV) on the 4 points with the largest wxx + wxy
//   lib/utils/extend_utils/src/uncertainty_pnp.cpp:20-37,61-92
//                                                      Ceres LM over (angle-axis, t) of sum_i |W_i (proj(R X_i + t) - x_i)|^2
//
// Here: one WARP per image, everything in fp64.  Lane i owns keypoint i (K <= 32): its weight
// matrix, residual and Jacobian rows; the 6x6 normal equations are summed over the warp through a
// 7 KB slice of shared memory and solved redundantly by every lane (Cholesky, fully unrolled in
// registers), so the loop has no divergence.  Rotation is kept as a matrix and updated on the manifold (R <- exp(dw) R), which has the
// same minimiser as the reference's angle-axis parametrisation; damping follows Ceres'
// Levenberg-Marquardt strategy (diagonal scaling, radius /= max(1/3, 1 - (2 rho - 1)^3) on success,
// shrink by 2, 4, 8.. on failure) but iterates until it has taken a step with max |delta| < 1e-9 instead of Ceres'
// function_tolerance 1e-6, i.e. to the minimiser the reference approximates.  Where Gauss-Newton converges
// quadratically the next step would be ~1e-11; on large-residual problems it converges only linearly and a last
// step below 1e-9 can leave a few 1e-8.  It also stops when max |J^T r| < 1e-14 (an absolute threshold), and when
// all 12 damping tries of one iteration fail to lower the cost (status 0 in both cases); a step below 1e-9 counts
// as convergence however heavily it was damped.
// Initialisation: Grunert's P3P quartic (roots by Durand-Kerner, fp32 then fp64, + fp64 Newton polish of the real
// ones) on the first three of the four selected points, the fourth picks the solution -- OpenCV's SOLVEPNP_P3P
// contract.
#include "common.cuh"

#include <cmath>

namespace {

// Most images converge in 4-12 iterations.  A P3P start whose first, nearly undamped step overshoots in depth
// (t_z 1.2 -> 3.2 on one 5-point image of the tests) then crawls back along a curved valley and needs ~240; the
// cap leaves room for twice that.  An image that reaches it returns a non-converged pose with status bit 2.
constexpr int PNP_MAX_ITERS = 500;

__device__ __forceinline__ double warp_sum_all(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct Vec3 {
    double x, y, z;
};
__device__ __forceinline__ Vec3 operator-(Vec3 a, Vec3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ Vec3 operator*(Vec3 a, double s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ double dot(Vec3 a, Vec3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ Vec3 cross(Vec3 a, Vec3 b)
{
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__device__ __forceinline__ Vec3 unit(Vec3 a) { return a * (1.0 / sqrt(dot(a, a))); }

// orthonormal frame of a triangle: columns e1, e2, e3 (row-major 3x3)
__device__ __forceinline__ void tri_frame(Vec3 p0, Vec3 p1, Vec3 p2, double (&F)[9])
{
    const Vec3 e1 = unit(p1 - p0);
    const Vec3 e3 = unit(cross(e1, p2 - p0));
    const Vec3 e2 = cross(e3, e1);
    F[0] = e1.x; F[1] = e2.x; F[2] = e3.x;
    F[3] = e1.y; F[4] = e2.y; F[5] = e3.y;
    F[6] = e1.z; F[7] = e2.z; F[8] = e3.z;
}

// one Durand-Kerner sweep over the four roots (zr + i zi) of the monic z^4 + f3 z^3 + f2 z^2 + f1 z + f0; returns
// the largest |correction| (|re| + |im|)
template <typename T>
__device__ __forceinline__ T durand_kerner_sweep(T (&zr)[4], T (&zi)[4], T f3, T f2, T f1, T f0)
{
    T move = T(0);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        // p(z) by Horner (monic)
        T vr = zr[k] + f3, vi = zi[k];
        T tr = vr * zr[k] - vi * zi[k] + f2, ti = vr * zi[k] + vi * zr[k];
        vr = tr * zr[k] - ti * zi[k] + f1;
        vi = tr * zi[k] + ti * zr[k];
        tr = vr * zr[k] - vi * zi[k] + f0;
        ti = vr * zi[k] + vi * zr[k];
        T dr = T(1), di = T(0);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (j == k) continue;
            const T er = zr[k] - zr[j], ei = zi[k] - zi[j];
            const T xr = dr * er - di * ei, xi = dr * ei + di * er;
            dr = xr;
            di = xi;
        }
        const T den = dr * dr + di * di;
        if (den > T(0)) {
            const T inv = T(1) / den;
            const T qr = (tr * dr + ti * di) * inv, qi = (ti * dr - tr * di) * inv;
            zr[k] -= qr;
            zi[k] -= qi;
            move = fmax(move, fabs(qr) + fabs(qi));
        }
    }
    return move;
}

// all roots of c4 z^4 + .. + c0 by Durand-Kerner: fp32 sweeps from a circle bring the four estimates near the roots
// cheaply, then fp64 sweeps on all four at once separate them.  P3P's quartics have their roots clustered near
// v = 1 with gaps ~1e-2, while rounding the coefficients to fp32 moves such a cluster by about as much: the fp32
// estimates alone can sit on the wrong root, and polishing them one at a time (Newton) merges neighbours and loses
// real roots.  The simultaneous fp64 iteration keeps the four apart; it stops when the largest correction is below
// 1e-10 of the root bound (2-3 sweeps for most quartics, up to 64 for near-double roots, whose corrections stall at
// the rounding floor).  The real roots (|im| <= 1e-6 max(1, |re|)) are then Newton-polished on the real polynomial
// and kept where the quartic vanishes to 1e-9 of its terms' magnitude.
__device__ int quartic_real_roots(const double (&c)[5], double (&out)[4])
{
    if (!(fabs(c[4]) > 1e-300)) return 0;
    const double a3 = c[3] / c[4], a2 = c[2] / c[4], a1 = c[1] / c[4], a0 = c[0] / c[4];
    const float f3 = (float)a3, f2 = (float)a2, f1 = (float)a1, f0 = (float)a0;
    float zr[4], zi[4];
    // start on a circle of the Cauchy bound's size, off the real axis
    const float rad = 1.0f + fmaxf(fmaxf(fabsf(f3), fabsf(f2)), fmaxf(fabsf(f1), fabsf(f0)));
    if (!(rad < 1e18f)) return 0;
    {
        float pr = 1.0f, pi = 0.0f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            zr[k] = pr * rad * 0.5f;
            zi[k] = pi * rad * 0.5f;
            const float nr = pr * 0.4f - pi * 0.9f, ni = pr * 0.9f + pi * 0.4f;
            pr = nr;
            pi = ni;
        }
    }
    for (int it = 0; it < 48; ++it)
        if (durand_kerner_sweep(zr, zi, f3, f2, f1, f0) < 2e-6f * rad) break;
    double wr[4], wi[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        wr[k] = zr[k];
        wi[k] = zi[k];
    }
    for (int it = 0; it < 64; ++it)
        if (durand_kerner_sweep(wr, wi, a3, a2, a1, a0) < 1e-10 * (double)rad) break;
    int n = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (!(fabs(wi[k]) <= 1e-6 * fmax(1.0, fabs(wr[k])))) continue;
        double v = wr[k];
        for (int it = 0; it < 12; ++it) {
            const double p = (((v + a3) * v + a2) * v + a1) * v + a0;
            const double d = ((4.0 * v + 3.0 * a3) * v + 2.0 * a2) * v + a1;
            if (d == 0.0) break;
            const double st = p / d;
            v -= st;
            if (fabs(st) < 1e-15 * fmax(1.0, fabs(v))) break;
        }
        const double resid = (((v + a3) * v + a2) * v + a1) * v + a0;
        const double scale = ((fabs(v) + fabs(a3)) * fabs(v) + fabs(a2)) * fabs(v) * fabs(v) + fabs(a1 * v) + fabs(a0);
        if (fabs(resid) <= 1e-9 * fmax(scale, 1e-300)) out[n++] = v;
    }
    return n;
}

// exp of a rotation vector (Rodrigues), row-major
__device__ void so3_exp(double wx, double wy, double wz, double (&E)[9])
{
    const double th2 = wx * wx + wy * wy + wz * wz;
    double a, b;                                   // E = I + a [w]x + b [w]x^2
    if (th2 < 1e-16) {
        a = 1.0 - th2 / 6.0;
        b = 0.5 - th2 / 24.0;
    } else {
        const double th = sqrt(th2);
        a = sin(th) / th;
        b = (1.0 - cos(th)) / th2;
    }
    E[0] = 1.0 - b * (wy * wy + wz * wz);
    E[1] = -a * wz + b * wx * wy;
    E[2] = a * wy + b * wx * wz;
    E[3] = a * wz + b * wx * wy;
    E[4] = 1.0 - b * (wx * wx + wz * wz);
    E[5] = -a * wx + b * wy * wz;
    E[6] = -a * wy + b * wx * wz;
    E[7] = a * wx + b * wy * wz;
    E[8] = 1.0 - b * (wx * wx + wy * wy);
}

// solve the SPD system A x = rhs (6x6, row-major, full storage) by Cholesky; false if not positive definite
__device__ bool chol6(const double (&A)[36], const double (&rhs)[6], double (&x)[6])
{
    double L[36];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = 0; j <= i; ++j) {
            double s = A[i * 6 + j];
#pragma unroll
            for (int k = 0; k < j; ++k) s -= L[i * 6 + k] * L[j * 6 + k];
            if (i == j) {
                if (!(s > 0.0)) return false;
                L[i * 6 + i] = sqrt(s);
            } else {
                L[i * 6 + j] = s / L[j * 6 + j];
            }
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double s = rhs[i];
#pragma unroll
        for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * y[k];
        y[i] = s / L[i * 6 + i];
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * x[k];
        x[i] = s / L[i * 6 + i];
    }
    return true;
}

struct PnpState {
    double R[9], t[3];
};

// this lane's weighted residual (and optionally its 2x6 Jacobian wrt (dw, dt), left perturbation)
__device__ __forceinline__ void lane_residual(const PnpState &s, bool active, Vec3 X, double u, double v, double wxx,
                                              double wxy, double wyy, double fx, double fy, double cx, double cy,
                                              double &r0, double &r1, double (*J)[6])
{
    r0 = r1 = 0.0;
    if (J)
        for (int j = 0; j < 6; ++j) J[0][j] = J[1][j] = 0.0;
    if (!active) return;
    const double rx = s.R[0] * X.x + s.R[1] * X.y + s.R[2] * X.z;        // R X
    const double ry = s.R[3] * X.x + s.R[4] * X.y + s.R[5] * X.z;
    const double rz = s.R[6] * X.x + s.R[7] * X.y + s.R[8] * X.z;
    const double px = rx + s.t[0], py = ry + s.t[1], pz = rz + s.t[2];
    const double iz = 1.0 / pz;
    const double dx = fx * px * iz + cx - u, dy = fy * py * iz + cy - v;
    r0 = wxx * dx + wxy * dy;
    r1 = wxy * dx + wyy * dy;
    if (!J) return;
    // d(proj)/d(p): [fx/z, 0, -fx px/z^2; 0, fy/z, -fy py/z^2];  dp/dw = -[R X]x, dp/dt = I
    const double a0 = fx * iz, a2 = -fx * px * iz * iz, b1 = fy * iz, b2 = -fy * py * iz * iz;
    // -[RX]x = [[0, rz, -ry], [-rz, 0, rx], [ry, -rx, 0]]
    const double ju[6] = {a2 * ry, a0 * rz - a2 * rx, -a0 * ry, a0, 0.0, a2};
    const double jv[6] = {-b1 * rz + b2 * ry, -b2 * rx, b1 * rx, 0.0, b1, b2};
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        J[0][j] = wxx * ju[j] + wxy * jv[j];
        J[1][j] = wxy * ju[j] + wyy * jv[j];
    }
}

// evaluation_utils.py:170-181 for one keypoint
__device__ __forceinline__ void cov_to_weight(double c00, double c01, double c10, double c11, double &wxx, double &wxy,
                                              double &wyy)
{
    wxx = wxy = wyy = 0.0;
    if (c00 < 1e-6 || isnan(c00) || isnan(c01) || isnan(c10) || isnan(c11)) return;
    const double o = 0.5 * (c01 + c10);
    const double det = c00 * c11 - o * o;
    if (!(det > 0.0)) return;
    const double sd = sqrt(det);
    const double nrm = sqrt(c00 + c11 + 2.0 * sd);
    const double r00 = (c00 + sd) / nrm, r01 = o / nrm, r11 = (c11 + sd) / nrm;        // sqrtm(cov)
    const double rdet = r00 * r11 - r01 * r01;
    wxx = r11 / rdet;
    wxy = -r01 / rdet;
    wyy = r00 / rdet;
}

// Sum 28 per-lane doubles (21 upper-triangle entries of J^T J, 6 of J^T r, the cost) over the warp through
// this warp's slice of shared memory: lanes write rows, the first 28 lanes add one column each, everyone
// reads the totals back.  (28 butterfly reductions of doubles cost ~10x more issue slots.)
constexpr int PNP_NRED = 28;
__device__ __forceinline__ void warp_reduce28(double (&v)[PNP_NRED], double *sm /* [33][PNP_NRED] */, int lane)
{
#pragma unroll
    for (int i = 0; i < PNP_NRED; ++i) sm[lane * PNP_NRED + i] = v[i];
    __syncwarp();
    if (lane < PNP_NRED) {
        double s = 0.0;
        for (int r = 0; r < 32; ++r) s += sm[r * PNP_NRED + lane];
        sm[32 * PNP_NRED + lane] = s;
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < PNP_NRED; ++i) v[i] = sm[32 * PNP_NRED + i];
    __syncwarp();
}

// Where each image's camera comes from: one K passed by value for the whole batch (pvnet_uncertainty_pnp), or a
// device array [b,3,3] with one K per image (pvnet_uncertainty_pnp_per_image_k).  Either way the solver reads
// fx = K[0,0], cx = K[0,2], fy = K[1,1], cy = K[1,2]; skew and the last row are not used.
struct PnpCamera {
    double fx, fy, cx, cy;
    const double *per_image;        // row-major [b,3,3] on the device, or null: every image uses (fx, fy, cx, cy)
};

// status bit 4: the image's K has a zero focal length (the rule pvnet_uncertainty_pnp applies to its host K); the
// image is not solved and its pose is NaN
constexpr int PNP_STATUS_BAD_CAMERA = 4;

// status bit 8 (pvnet_uncertainty_pnp_instances): row j of image b with j >= num[b] holds no instance; it is not
// solved and its pose is NaN
constexpr int PNP_STATUS_NO_INSTANCE = 8;

// The solve of one image by one warp: keypoint row `img` of kp / cov / wgt, pose and info row `img` of the outputs,
// camera row `cam_row` of cam.per_image (when not null).  s_red, s_cam: the CTA's reduction slices and camera slots
// in shared memory, one per warp.
__device__ __forceinline__ void pnp_solve(const float *__restrict__ kp, const float *__restrict__ cov,
                                          const float *__restrict__ wgt, const float *__restrict__ pts3d,
                                          const PnpCamera &cam, int cam_row, int img, int K,
                                          double (*s_red)[33 * PNP_NRED], double (*s_cam)[4],
                                          double *__restrict__ out_pose, int *__restrict__ out_info)
{
    const int lane = threadIdx.x & 31;
    // this image's (fx, fy, cx, cy) in this warp's slot of shared memory, read where they are used: held in
    // registers through the LM loop they would push the kernel (at the 255-register limit) into spilling
    double *cm = s_cam[threadIdx.x >> 5];
    if (lane == 0) {
        const double *k = cam.per_image ? cam.per_image + (size_t)cam_row * 9 : nullptr;
        cm[0] = k ? k[0] : cam.fx;
        cm[1] = k ? k[4] : cam.fy;
        cm[2] = k ? k[2] : cam.cx;
        cm[3] = k ? k[5] : cam.cy;
    }
    __syncwarp();
    const double &fx = cm[0], &fy = cm[1], &cx = cm[2], &cy = cm[3];
    if (!(fx != 0.0 && fy != 0.0)) {                // warp-uniform: the whole warp leaves
        if (lane == 0) {
            for (int i = 0; i < 12; ++i) out_pose[(size_t)img * 12 + i] = __longlong_as_double(0x7ff8000000000000ll);
            if (out_info) {
                out_info[img * 2] = PNP_STATUS_BAD_CAMERA;
                out_info[img * 2 + 1] = 0;
            }
        }
        return;
    }
    double *sm = s_red[threadIdx.x >> 5];
    const bool active = lane < K;
    const int li = active ? lane : 0;
    const double u = kp[((size_t)img * K + li) * 2], v = kp[((size_t)img * K + li) * 2 + 1];
    const Vec3 X = {pts3d[li * 3], pts3d[li * 3 + 1], pts3d[li * 3 + 2]};
    double wxx, wxy, wyy;
    if (wgt) {
        wxx = wgt[((size_t)img * K + li) * 3];
        wxy = wgt[((size_t)img * K + li) * 3 + 1];
        wyy = wgt[((size_t)img * K + li) * 3 + 2];
    } else {
        const float *c = cov + ((size_t)img * K + li) * 4;
        cov_to_weight(c[0], c[1], c[2], c[3], wxx, wxy, wyy);
    }
    if (!active) wxx = wxy = wyy = 0.0;

    // ---- the four most confident points: argsort(wxx + wxy)[-4:], ascending (extend_utils.py:84)
    const double key = wxx + wxy;
    int rank = 0;                                   // how many points sort after this one
    for (int j = 0; j < K; ++j) {
        const double kj = __shfl_sync(0xffffffffu, key, j);
        if (j != lane && (kj > key || (kj == key && j > lane))) ++rank;
    }
    if (!active) rank = 64;
    int sel[4];
    for (int r = 0; r < 4; ++r) {                   // sel[0..3] = ascending order = ranks 3,2,1,0
        const unsigned m = __ballot_sync(0xffffffffu, rank == 3 - r);
        sel[r] = m ? __ffs(m) - 1 : 0;
    }
    Vec3 P[4];
    double U[4], V[4];
    for (int r = 0; r < 4; ++r) {
        P[r].x = __shfl_sync(0xffffffffu, X.x, sel[r]);
        P[r].y = __shfl_sync(0xffffffffu, X.y, sel[r]);
        P[r].z = __shfl_sync(0xffffffffu, X.z, sel[r]);
        U[r] = __shfl_sync(0xffffffffu, u, sel[r]);
        V[r] = __shfl_sync(0xffffffffu, v, sel[r]);
    }

    // ---- P3P (every lane computes the same thing)
    PnpState st;
    bool have_init = false;
    {
        Vec3 f[3];
        for (int r = 0; r < 3; ++r) f[r] = unit(Vec3{(U[r] - cx) / fx, (V[r] - cy) / fy, 1.0});
        const Vec3 d12 = P[1] - P[2], d02 = P[0] - P[2], d01 = P[0] - P[1];
        const double a2 = dot(d12, d12), b2 = dot(d02, d02), c2 = dot(d01, d01);
        const double ca = dot(f[1], f[2]), cb = dot(f[0], f[2]), cg = dot(f[0], f[1]);
        if (b2 > 0.0 && a2 > 0.0 && c2 > 0.0) {
            const double q = (a2 - c2) / b2, p = (a2 + c2) / b2;
            double co[5];
            co[4] = (q - 1) * (q - 1) - 4 * c2 / b2 * ca * ca;
            co[3] = 4 * (q * (1 - q) * cb - (1 - p) * ca * cg + 2 * c2 / b2 * ca * ca * cb);
            co[2] = 2 * (q * q - 1 + 2 * q * q * cb * cb + 2 * (b2 - c2) / b2 * ca * ca - 4 * p * ca * cb * cg +
                         2 * (b2 - a2) / b2 * cg * cg);
            co[1] = 4 * (-q * (1 + q) * cb + 2 * a2 / b2 * cg * cg * cb - (1 - p) * ca * cg);
            co[0] = (1 + q) * (1 + q) - 4 * a2 / b2 * cg * cg;
            double roots[4];
            const int nr = quartic_real_roots(co, roots);
            double best = 1e300;
            double FP[9];
            tri_frame(P[0], P[1], P[2], FP);
            for (int i = 0; i < nr; ++i) {
                const double vv = roots[i];
                const double den = 2 * (cg - vv * ca);
                if (!(fabs(den) > 1e-14) || !(vv > 0.0)) continue;
                const double uu = ((q - 1) * vv * vv - 2 * q * cb * vv + 1 + q) / den;
                const double s1sq = b2 / (1 + vv * vv - 2 * vv * cb);
                if (!(uu > 0.0) || !(s1sq > 0.0)) continue;
                const double s1 = sqrt(s1sq);
                const Vec3 Q0 = f[0] * s1, Q1 = f[1] * (uu * s1), Q2 = f[2] * (vv * s1);
                double FQ[9], Rc[9];
                tri_frame(Q0, Q1, Q2, FQ);
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c)
                        Rc[r * 3 + c] = FQ[r * 3] * FP[c * 3] + FQ[r * 3 + 1] * FP[c * 3 + 1] + FQ[r * 3 + 2] * FP[c * 3 + 2];
                const double tx = Q0.x - (Rc[0] * P[0].x + Rc[1] * P[0].y + Rc[2] * P[0].z);
                const double ty = Q0.y - (Rc[3] * P[0].x + Rc[4] * P[0].y + Rc[5] * P[0].z);
                const double tz = Q0.z - (Rc[6] * P[0].x + Rc[7] * P[0].y + Rc[8] * P[0].z);
                const double x4 = Rc[0] * P[3].x + Rc[1] * P[3].y + Rc[2] * P[3].z + tx;
                const double y4 = Rc[3] * P[3].x + Rc[4] * P[3].y + Rc[5] * P[3].z + ty;
                const double z4 = Rc[6] * P[3].x + Rc[7] * P[3].y + Rc[8] * P[3].z + tz;
                const double eu = fx * x4 / z4 + cx - U[3], ev = fy * y4 / z4 + cy - V[3];
                const double e = eu * eu + ev * ev;
                if (e < best) {
                    best = e;
                    for (int j = 0; j < 9; ++j) st.R[j] = Rc[j];
                    st.t[0] = tx;
                    st.t[1] = ty;
                    st.t[2] = tz;
                    have_init = true;
                }
            }
        }
    }
    if (!have_init) {
        for (int j = 0; j < 9; ++j) st.R[j] = (j % 4 == 0) ? 1.0 : 0.0;
        st.t[0] = st.t[1] = 0.0;
        st.t[2] = 1.0;
    }

    // ---- Levenberg-Marquardt (extend_utils.py:90-94: with exactly 4 points the P3P pose is the answer)
    int iters = 0, status = have_init ? 0 : 1;      // bit 0: P3P found no solution
    if (K > 4) {
        double radius = 1e4, decrease = 2.0;       // Ceres: initial_trust_region_radius 1e4
        double r0, r1, J[2][6];
        lane_residual(st, active, X, u, v, wxx, wxy, wyy, fx, fy, cx, cy, r0, r1, J);
        double cost = 0.5 * warp_sum_all(r0 * r0 + r1 * r1);
        for (; iters < PNP_MAX_ITERS; ++iters) {
            double A[36], g[6];
            {
                double red[PNP_NRED];
                int q = 0;
#pragma unroll
                for (int i = 0; i < 6; ++i)
#pragma unroll
                    for (int j = i; j < 6; ++j) red[q++] = J[0][i] * J[0][j] + J[1][i] * J[1][j];
#pragma unroll
                for (int i = 0; i < 6; ++i) red[21 + i] = J[0][i] * r0 + J[1][i] * r1;
                red[27] = 0.0;
                warp_reduce28(red, sm, lane);
                q = 0;
#pragma unroll
                for (int i = 0; i < 6; ++i)
#pragma unroll
                    for (int j = i; j < 6; ++j) {
                        A[i * 6 + j] = red[q];
                        A[j * 6 + i] = red[q++];
                    }
#pragma unroll
                for (int i = 0; i < 6; ++i) g[i] = red[21 + i];
            }
            double gmax = 0.0;
            for (int i = 0; i < 6; ++i) gmax = fmax(gmax, fabs(g[i]));
            if (gmax < 1e-14) break;
            bool stepped = false, converged = false;
            for (int tries = 0; tries < 12 && !stepped; ++tries) {
                double Ad[36], rhs[6], d[6];
                for (int i = 0; i < 36; ++i) Ad[i] = A[i];
                for (int i = 0; i < 6; ++i) {
                    const double dd = fmin(fmax(A[i * 6 + i], 1e-12), 1e64);      // Ceres clamps the Jacobi scaling
                    Ad[i * 6 + i] += dd / radius;
                    rhs[i] = -g[i];
                }
                if (!chol6(Ad, rhs, d)) {
                    radius /= decrease;
                    decrease *= 2.0;
                    continue;
                }
                double dn = 0.0;
                for (int i = 0; i < 6; ++i) dn = fmax(dn, fabs(d[i]));
                PnpState cand;
                double E[9];
                so3_exp(d[0], d[1], d[2], E);
                for (int r = 0; r < 3; ++r)
                    for (int c = 0; c < 3; ++c)
                        cand.R[r * 3 + c] = E[r * 3] * st.R[c] + E[r * 3 + 1] * st.R[3 + c] + E[r * 3 + 2] * st.R[6 + c];
                for (int i = 0; i < 3; ++i) cand.t[i] = st.t[i] + d[3 + i];
                if (dn < 1e-9) {                    // the next Gauss-Newton step would be ~50x smaller: take this one, stop
                    st = cand;                      // (cost differences are below rounding here: rho would be noise)
                    converged = true;
                    break;
                }
                double c0, c1, Jc[2][6];
                lane_residual(cand, active, X, u, v, wxx, wxy, wyy, fx, fy, cx, cy, c0, c1, Jc);
                const double new_cost = 0.5 * warp_sum_all(c0 * c0 + c1 * c1);
                // model decrease: -g.d - 0.5 d^T A d
                double md = 0.0;
                for (int i = 0; i < 6; ++i) {
                    double Adi = 0.0;
                    for (int j = 0; j < 6; ++j) Adi += A[i * 6 + j] * d[j];
                    md -= d[i] * (g[i] + 0.5 * Adi);
                }
                const double rho = (cost - new_cost) / md;
                if (new_cost <= cost && md > 0.0 && rho > 1e-3) {
                    st = cand;
                    r0 = c0;
                    r1 = c1;
                    for (int i = 0; i < 6; ++i) {
                        J[0][i] = Jc[0][i];
                        J[1][i] = Jc[1][i];
                    }
                    const double tmp = 2.0 * rho - 1.0;
                    radius = fmin(radius / fmax(1.0 / 3.0, 1.0 - tmp * tmp * tmp), 1e16);
                    decrease = 2.0;
                    cost = new_cost;
                    stepped = true;
                } else {
                    radius /= decrease;
                    decrease *= 2.0;
                }
            }
            if (converged || !stepped) break;
        }
        if (iters >= PNP_MAX_ITERS) status |= 2;
    }
    if (lane == 0) {
        double *o = out_pose + (size_t)img * 12;
        for (int r = 0; r < 3; ++r) {
            o[r * 4] = st.R[r * 3];
            o[r * 4 + 1] = st.R[r * 3 + 1];
            o[r * 4 + 2] = st.R[r * 3 + 2];
            o[r * 4 + 3] = st.t[r];
        }
        if (out_info) {
            out_info[img * 2] = status;
            out_info[img * 2 + 1] = iters;
        }
    }
}

// one warp per image
__global__ void __launch_bounds__(128)
    k_uncertainty_pnp(const float *__restrict__ kp, const float *__restrict__ cov, const float *__restrict__ wgt,
                      const float *__restrict__ pts3d, PnpCamera cam, int nb, int K,
                      double *__restrict__ out_pose, int *__restrict__ out_info)
{
    __shared__ double s_red[4][33 * PNP_NRED];
    const int img = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (img >= nb) return;
    __shared__ double s_cam[4][4];
    pnp_solve(kp, cov, wgt, pts3d, cam, img, img, K, s_red, s_cam, out_pose, out_info);
}

// One warp per (image, instance) row v = bi * L + j of [b,L] keypoints.  A row with j < num[bi] is solved with camera
// bi by k_uncertainty_pnp's code; the others leave at once with a NaN pose and status PNP_STATUS_NO_INSTANCE.
__global__ void __launch_bounds__(128)
    k_uncertainty_pnp_instances(const float *__restrict__ kp, const float *__restrict__ cov,
                                const float *__restrict__ wgt, const float *__restrict__ pts3d, PnpCamera cam,
                                const int *__restrict__ num, int L, int nrows, int K, double *__restrict__ out_pose,
                                int *__restrict__ out_info)
{
    __shared__ double s_red[4][33 * PNP_NRED];
    __shared__ double s_cam[4][4];
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (row >= nrows) return;
    const int bi = row / L, j = row - bi * L;
    if (j >= num[bi]) {                             // warp-uniform
        if ((threadIdx.x & 31) == 0) {
            for (int i = 0; i < 12; ++i) out_pose[(size_t)row * 12 + i] = __longlong_as_double(0x7ff8000000000000ll);
            if (out_info) {
                out_info[row * 2] = PNP_STATUS_NO_INSTANCE;
                out_info[row * 2 + 1] = 0;
            }
        }
        return;
    }
    pnp_solve(kp, cov, wgt, pts3d, cam, bi, row, K, s_red, s_cam, out_pose, out_info);
}

// covariance -> (wxx, wxy, wyy), thread per keypoint
__global__ void k_cov_to_weights(const float *__restrict__ cov, int n, float *__restrict__ wgt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double wxx, wxy, wyy;
    cov_to_weight(cov[i * 4], cov[i * 4 + 1], cov[i * 4 + 2], cov[i * 4 + 3], wxx, wxy, wyy);
    wgt[i * 3] = (float)wxx;
    wgt[i * 3 + 1] = (float)wxy;
    wgt[i * 3 + 2] = (float)wyy;
}

}  // namespace

extern "C" {

int pvnet_covariance_to_weights(const float *cov, int n, float *weights, pvnet_stream_t stream)
{
    PV_CHECK_ARG(cov && weights, "null pointer");
    PV_CHECK_ARG(n >= 1, "non-positive count");
    k_cov_to_weights<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(cov, n, weights);
    PV_LAUNCHED("k_cov_to_weights");
    return PVNET_OK;
}

static int launch_uncertainty_pnp(const float *points_2d, const float *cov, const float *weights_2d,
                                  const float *points_3d, PnpCamera cam, int b, int pn, double *out_pose,
                                  int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(points_2d && points_3d && out_pose, "null pointer");
    PV_CHECK_ARG((cov != nullptr) != (weights_2d != nullptr), "pass exactly one of cov / weights_2d");
    PV_CHECK_ARG(b >= 1, "non-positive batch");
    PV_CHECK_ARG(pn >= 4 && pn <= 32, "point count %d outside [4,32] (one warp per image)", pn);
    // one warp per CTA: the solve is a serial fp64 chain, so images should sit on different SMs, not share
    // one SM's fp64 pipe (4 warps per CTA doubled the time at batch 16)
    const int warps_per_cta = b <= 592 ? 1 : 4;
    k_uncertainty_pnp<<<(b + warps_per_cta - 1) / warps_per_cta, 32 * warps_per_cta, 0, (cudaStream_t)stream>>>(
        points_2d, cov, weights_2d, points_3d, cam, b, pn, out_pose, out_info);
    PV_LAUNCHED("k_uncertainty_pnp");
    return PVNET_OK;
}

int pvnet_uncertainty_pnp(const float *points_2d, const float *cov, const float *weights_2d, const float *points_3d,
                          const double camera_matrix[9], int b, int pn, double *out_pose, int32_t *out_info,
                          pvnet_stream_t stream)
{
    PV_CHECK_ARG(camera_matrix, "null pointer");
    const double fx = camera_matrix[0], fy = camera_matrix[4], cx = camera_matrix[2], cy = camera_matrix[5];
    PV_CHECK_ARG(fx != 0.0 && fy != 0.0, "zero focal length");
    return launch_uncertainty_pnp(points_2d, cov, weights_2d, points_3d, PnpCamera{fx, fy, cx, cy, nullptr}, b, pn,
                                  out_pose, out_info, stream);
}

int pvnet_uncertainty_pnp_per_image_k(const float *points_2d, const float *cov, const float *weights_2d,
                                      const float *points_3d, const double *camera_matrices, int b, int pn,
                                      double *out_pose, int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(camera_matrices, "null pointer");
    return launch_uncertainty_pnp(points_2d, cov, weights_2d, points_3d, PnpCamera{0.0, 0.0, 0.0, 0.0, camera_matrices},
                                  b, pn, out_pose, out_info, stream);
}

int pvnet_uncertainty_pnp_instances(const float *points_2d, const float *cov, const float *weights_2d,
                                    const float *points_3d, const double *camera_matrices, const int32_t *num, int L,
                                    int b, int pn, double *out_pose, int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(points_2d && points_3d && out_pose && camera_matrices && num, "null pointer");
    PV_CHECK_ARG((cov != nullptr) != (weights_2d != nullptr), "pass exactly one of cov / weights_2d");
    PV_CHECK_ARG(b >= 1, "non-positive batch");
    PV_CHECK_ARG(L >= 1 && L <= 32 && b * L <= 1024, "instance count %d outside 1..32 or b*L = %d above 1024", L,
                 b * L);
    PV_CHECK_ARG(pn >= 4 && pn <= 32, "point count %d outside [4,32] (one warp per image)", pn);
    const int rows = b * L;
    const int warps_per_cta = rows <= 592 ? 1 : 4;      // launch_uncertainty_pnp's rule, over the rows
    k_uncertainty_pnp_instances<<<(rows + warps_per_cta - 1) / warps_per_cta, 32 * warps_per_cta, 0,
                                  (cudaStream_t)stream>>>(points_2d, cov, weights_2d, points_3d,
                                                          PnpCamera{0.0, 0.0, 0.0, 0.0, camera_matrices}, num, L, rows,
                                                          pn, out_pose, out_info);
    PV_LAUNCHED("k_uncertainty_pnp_instances");
    return PVNET_OK;
}

}  // extern "C"
