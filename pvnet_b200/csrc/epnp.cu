// epnp.cu -- EPnP on the device: the reference's `pnp(..., method=cv2.SOLVEPNP_EPNP)` (lib/utils/evaluation_utils.py:
// 19-52) for a whole batch, one warp per image, everything in fp64.
//
// The algorithm is Lepetit, Moreno-Noguer and Fua, "EPnP: An Accurate O(n) Solution to the PnP Problem" (IJCV 81(2),
// 2009); oracle/epnp_oracle.py restates it step for step in numpy:
//   1. control points: c0 = centroid; c1..c3 = c0 + sqrt(lambda_k / n) v_k from the PCA of the centred object points
//      (a cyclic one-sided Jacobi from the identity, whose eigenvector signs are the ones OpenCV's output shows: with
//      noisy image points the pose depends on which control points are used);
//   2. barycentric coordinates alpha of every point (closed form: the v_k are orthonormal);
//   3. M^T M (12x12) of the 2n x 12 system, from 40 per-point moments summed over the warp (ten per pass);
//   4. its four smallest eigenvectors, by a parallel cyclic Jacobi in shared memory;
//   5. L (6x10) and rho (6);
//   6. betas by three linearisations (N = 1, 2, 3), each followed by 5 Gauss-Newton steps;
//   7. per N: camera control points, sign fix (the first point in front of the camera), R and t by the SVD
//      Procrustes fit (a reflection made a rotation by negating its third row), mean reprojection error in pixels;
//   8. the N with the smallest error (strict <, N = 1 first).
// Lanes stride over the points for every sum; the warp sums are xor butterflies, which give every lane the same
// value and the same value from run to run.  Everything after the sums runs redundantly in every lane (or, for the
// 12x12 Jacobi, lane-parallel in this warp's slice of shared memory).  No workspace, no allocation, no host sync.
#include "common.cuh"

#include <cmath>

namespace {

constexpr int EPNP_MAX_POINTS = 4096;
constexpr int EPNP_GN_STEPS = 5;
constexpr int EPNP_PCA_SWEEPS = 30;          // 3x3 Jacobi sweeps (converges in 4-6)
constexpr int EPNP_SWEEPS_12 = 20;           // 12x12 Jacobi sweeps (converges in 6-9)
constexpr double EPNP_PCA_DEGENERATE = 1e-10;  // status 1: smallest PCA eigenvalue <= this x the largest
constexpr int EPNP_STATUS_DEGENERATE = 1;
constexpr int EPNP_STATUS_BAD_CAMERA = 4;
constexpr int EPNP_WARPS = 4;                // warps per CTA at most

__device__ __forceinline__ double wsum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double dot3(const double *a, const double *b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// PCA of the symmetric PSD 3x3 A: cyclic one-sided Jacobi on its rows from V = I; every rotation leaves the larger
// row norm in the lower index.  lam descending, V rows = unit eigenvectors (oracle/epnp_oracle.py pca3).
__device__ void pca3(const double (&A0)[9], double (&lam)[3], double (&V)[9])
{
    double A[9], W[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        A[i] = A0[i];
        W[i] = (i % 4 == 0) ? 1.0 : 0.0;
    }
    double w[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = dot3(A + 3 * i, A + 3 * i);
    for (int sweep = 0; sweep < EPNP_PCA_SWEEPS; ++sweep) {
        bool changed = false;
#pragma unroll
        for (int pr = 0; pr < 3; ++pr) {
            const int i = pr == 2 ? 1 : 0, j = pr == 0 ? 1 : 2;
            const double a = w[i], b = w[j];
            double p = dot3(A + 3 * i, A + 3 * j);
            if (!(fabs(p) > 2.2e-15 * sqrt(a * b))) continue;
            p *= 2.0;
            const double beta = a - b, gamma = hypot(p, beta);
            double c, s;
            if (beta < 0) {
                s = sqrt((gamma - beta) * 0.5 / gamma);
                c = p / (gamma * s * 2.0);
            } else {
                c = sqrt((gamma + beta) / (gamma * 2.0));
                s = p / (gamma * c * 2.0);
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double ai = A[3 * i + k], aj = A[3 * j + k], vi = W[3 * i + k], vj = W[3 * j + k];
                A[3 * i + k] = c * ai + s * aj;
                A[3 * j + k] = -s * ai + c * aj;
                W[3 * i + k] = c * vi + s * vj;
                W[3 * j + k] = -s * vi + c * vj;
            }
            w[i] = dot3(A + 3 * i, A + 3 * i);
            w[j] = dot3(A + 3 * j, A + 3 * j);
            changed = true;
        }
        if (!changed) break;
    }
    double l[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) l[i] = sqrt(dot3(A + 3 * i, A + 3 * i));
    // stable descending order of three values
    int o[3] = {0, 1, 2};
    if (l[o[1]] > l[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
    if (l[o[2]] > l[o[1]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
    if (l[o[1]] > l[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        lam[r] = l[o[r]];
#pragma unroll
        for (int k = 0; k < 3; ++k) V[3 * r + k] = W[3 * o[r] + k];
    }
}

// Eigenvectors of the symmetric 3x3 S by cyclic two-sided Jacobi: columns of E, eigenvalues descending in d.
__device__ void sym3_eig(const double (&S0)[9], double (&d)[3], double (&E)[9])
{
    double S[9], Q[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        S[i] = S0[i];
        Q[i] = (i % 4 == 0) ? 1.0 : 0.0;
    }
    const double scale = fabs(S[0]) + fabs(S[4]) + fabs(S[8]);
    for (int sweep = 0; sweep < EPNP_PCA_SWEEPS; ++sweep) {
        bool changed = false;
#pragma unroll
        for (int pr = 0; pr < 3; ++pr) {
            const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2;
            const double apq = S[3 * p + q];
            if (!(fabs(apq) > fmax(2.2e-16 * sqrt(fabs(S[4 * p] * S[4 * q])), 1e-17 * scale))) continue;
            const double th = (S[4 * q] - S[4 * p]) / (2.0 * apq);
            const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(1.0 + th * th));
            const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
#pragma unroll
            for (int k = 0; k < 3; ++k) {               // S <- S J (columns p, q)
                const double kp = S[3 * k + p], kq = S[3 * k + q];
                S[3 * k + p] = c * kp - s * kq;
                S[3 * k + q] = s * kp + c * kq;
                const double qp = Q[3 * k + p], qq = Q[3 * k + q];
                Q[3 * k + p] = c * qp - s * qq;
                Q[3 * k + q] = s * qp + c * qq;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {               // S <- J^T S (rows p, q)
                const double pk = S[3 * p + k], qk = S[3 * q + k];
                S[3 * p + k] = c * pk - s * qk;
                S[3 * q + k] = s * pk + c * qk;
            }
            changed = true;
        }
        if (!changed) break;
    }
    int o[3] = {0, 1, 2};
    if (S[4 * o[1]] > S[4 * o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
    if (S[4 * o[2]] > S[4 * o[1]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
    if (S[4 * o[1]] > S[4 * o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        d[r] = S[4 * o[r]];
#pragma unroll
        for (int k = 0; k < 3; ++k) E[3 * k + r] = Q[3 * k + o[r]];
    }
}

// Least squares min |A x - b| of a 6 x NC system by Householder QR (A and b are overwritten).
template <int NC>
__device__ void lsq6(double (&A)[6][NC], double (&b)[6], double (&x)[NC])
{
    double diag[NC];
#pragma unroll
    for (int k = 0; k < NC; ++k) {
        double nrm = 0.0;
#pragma unroll
        for (int i = k; i < 6; ++i) nrm += A[i][k] * A[i][k];
        nrm = sqrt(nrm);
        const double alpha = A[k][k] > 0 ? -nrm : nrm;     // R[k][k]
        diag[k] = alpha;
        if (nrm == 0.0) continue;
        // v = a_k - alpha e_k, stored in place; H = I - 2 v v^T / (v^T v)
        A[k][k] -= alpha;
        double vtv = 0.0;
#pragma unroll
        for (int i = k; i < 6; ++i) vtv += A[i][k] * A[i][k];
#pragma unroll
        for (int j = k + 1; j < NC; ++j) {
            double s = 0.0;
#pragma unroll
            for (int i = k; i < 6; ++i) s += A[i][k] * A[i][j];
            s = 2.0 * s / vtv;
#pragma unroll
            for (int i = k; i < 6; ++i) A[i][j] -= s * A[i][k];
        }
        double s = 0.0;
#pragma unroll
        for (int i = k; i < 6; ++i) s += A[i][k] * b[i];
        s = 2.0 * s / vtv;
#pragma unroll
        for (int i = k; i < 6; ++i) b[i] -= s * A[i][k];
    }
#pragma unroll
    for (int k = NC - 1; k >= 0; --k) {
        double s = b[k];
#pragma unroll
        for (int j = k + 1; j < NC; ++j) s -= A[k][j] * x[j];
        x[k] = diag[k] != 0.0 ? s / diag[k] : 0.0;
    }
}

// per-warp shared memory: the 12x12 Jacobi, then L and rho
struct EpnpShared {
    double A[144], V[144];
    double c[12], s[12];
    int partner[12];
    double L[60], rho[6];
    int idx[4];
};

// the four smallest eigenvectors of the symmetric 12x12 in sh.A (columns of sh.V after the call): parallel cyclic
// Jacobi in the round-robin order, six disjoint rotations per round, eleven rounds per sweep
__device__ void jacobi12(EpnpShared &sh, int lane)
{
    for (int e = lane; e < 144; e += 32) sh.V[e] = (e % 13 == 0) ? 1.0 : 0.0;
    __syncwarp();
    // an off-diagonal entry is left alone below eps of its diagonal pair or 1e-17 of the trace: the second rule ends
    // the sweeps where rounding keeps refilling entries next to the (near-)zero eigenvalues
    double scale = 0.0;
    for (int i = 0; i < 12; ++i) scale += fabs(sh.A[13 * i]);
    for (int sweep = 0; sweep < EPNP_SWEEPS_12; ++sweep) {
        bool rotated = false;
        for (int round = 0; round < 11; ++round) {
            if (lane < 6) {
                const int a = lane == 0 ? 0 : 1 + (lane - 1 + round) % 11;
                const int b = 1 + (10 - lane + round) % 11;
                const int p = a < b ? a : b, q = a < b ? b : a;
                const double app = sh.A[13 * p], aqq = sh.A[13 * q], apq = sh.A[12 * p + q];
                double c = 1.0, s = 0.0;
                if (fabs(apq) > fmax(2.2e-16 * sqrt(fabs(app * aqq)), 1e-17 * scale)) {
                    const double th = (aqq - app) / (2.0 * apq);
                    const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(1.0 + th * th));
                    c = 1.0 / sqrt(1.0 + t * t);
                    s = t * c;
                    rotated = rotated || s != 0.0;
                }
                sh.partner[p] = q;
                sh.partner[q] = p;
                sh.c[p] = c;
                sh.c[q] = c;
                sh.s[p] = -s;                       // column p of J: c at p, -s at q; column q: s at p, c at q
                sh.s[q] = s;
            }
            __syncwarp();
            double na[5], nv[5];
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const int e = lane + 32 * k;
                if (e < 144) {
                    const int r = e / 12, col = e % 12, pr = sh.partner[r], pc = sh.partner[col];
                    const double cr = sh.c[r], sr = sh.s[r], cc = sh.c[col], sc = sh.s[col];
                    na[k] = cr * (cc * sh.A[12 * r + col] + sc * sh.A[12 * r + pc]) +
                            sr * (cc * sh.A[12 * pr + col] + sc * sh.A[12 * pr + pc]);
                    nv[k] = cc * sh.V[12 * r + col] + sc * sh.V[12 * r + pc];
                }
            }
            __syncwarp();
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const int e = lane + 32 * k;
                if (e < 144) {
                    sh.A[e] = na[k];
                    sh.V[e] = nv[k];
                }
            }
            __syncwarp();
        }
        if (!__any_sync(0xffffffffu, rotated)) break;
    }
    if (lane == 0) {                                // indices of the four smallest eigenvalues, ascending
        bool used[12];
        for (int i = 0; i < 12; ++i) used[i] = false;
        for (int k = 0; k < 4; ++k) {
            int m = -1;
            for (int i = 0; i < 12; ++i)
                if (!used[i] && (m < 0 || sh.A[13 * i] < sh.A[13 * m] || sh.A[13 * m] != sh.A[13 * m])) m = i;
            used[m] = true;
            sh.idx[k] = m;
        }
    }
    __syncwarp();
}

__device__ __forceinline__ double vv(const EpnpShared &sh, int k, int i) { return sh.V[12 * i + sh.idx[k]]; }

// Gauss-Newton on the six distance equations L q(beta) = rho (all four betas)
__device__ void gauss_newton(const EpnpShared &sh, double (&be)[4])
{
#pragma unroll 1
    for (int it = 0; it < EPNP_GN_STEPS; ++it) {
        double J[6][4], r[6], dx[4];
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const double *l = sh.L + 10 * i;
            J[i][0] = 2 * l[0] * be[0] + l[1] * be[1] + l[3] * be[2] + l[6] * be[3];
            J[i][1] = l[1] * be[0] + 2 * l[2] * be[1] + l[4] * be[2] + l[7] * be[3];
            J[i][2] = l[3] * be[0] + l[4] * be[1] + 2 * l[5] * be[2] + l[8] * be[3];
            J[i][3] = l[6] * be[0] + l[7] * be[1] + l[8] * be[2] + 2 * l[9] * be[3];
            r[i] = sh.rho[i] - (l[0] * be[0] * be[0] + l[1] * be[0] * be[1] + l[2] * be[1] * be[1] +
                                l[3] * be[0] * be[2] + l[4] * be[1] * be[2] + l[5] * be[2] * be[2] +
                                l[6] * be[0] * be[3] + l[7] * be[1] * be[3] + l[8] * be[2] * be[3] +
                                l[9] * be[3] * be[3]);
        }
        lsq6<4>(J, r, dx);
#pragma unroll
        for (int k = 0; k < 4; ++k) be[k] += dx[k];
    }
}

// the linearised betas of linearisation N (1: b11 b12 b13 b14; 2: b11 b12 b22; 3: b11 b12 b22 b13 b23)
template <int NC>
__device__ void linearised(const EpnpShared &sh, const int (&cols)[NC], double (&x)[NC])
{
    double A[6][NC], b[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
#pragma unroll
        for (int j = 0; j < NC; ++j) A[i][j] = sh.L[10 * i + cols[j]];
        b[i] = sh.rho[i];
    }
    lsq6<NC>(A, b, x);
}

__device__ __noinline__ void betas(const EpnpShared &sh, int N, double (&be)[4])
{
    if (N == 1) {
        const int cols[4] = {0, 1, 3, 6};
        double x[4];
        linearised<4>(sh, cols, x);
        const double b0 = sqrt(fabs(x[0])), sg = x[0] < 0 ? -1.0 : 1.0;
        be[0] = b0;
        be[1] = sg * x[1] / b0;
        be[2] = sg * x[2] / b0;
        be[3] = sg * x[3] / b0;
        return;
    }
    double x[5] = {0, 0, 0, 0, 0};
    if (N == 2) {
        const int cols[3] = {0, 1, 2};
        double y[3];
        linearised<3>(sh, cols, y);
        x[0] = y[0];
        x[1] = y[1];
        x[2] = y[2];
    } else {
        const int cols[5] = {0, 1, 2, 3, 4};
        linearised<5>(sh, cols, x);
    }
    double b0, b1;
    if (x[0] < 0) {
        b0 = sqrt(-x[0]);
        b1 = x[2] < 0 ? sqrt(-x[2]) : 0.0;
    } else {
        b0 = sqrt(x[0]);
        b1 = x[2] > 0 ? sqrt(x[2]) : 0.0;
    }
    if (x[1] < 0) b0 = -b0;
    be[0] = b0;
    be[1] = b1;
    be[2] = N == 3 ? x[3] / b0 : 0.0;
    be[3] = 0.0;
}

// R from the cross-covariance H = U S V^T: U V^T, a reflection's third row negated (oracle/epnp_oracle.py procrustes)
__device__ __noinline__ void procrustes(const double (&H)[9], double (&R)[9])
{
    double HtH[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) HtH[3 * i + j] = H[i] * H[j] + H[3 + i] * H[3 + j] + H[6 + i] * H[6 + j];
    double d[3], E[9];
    sym3_eig(HtH, d, E);
    double v0[3] = {E[0], E[3], E[6]}, v1[3] = {E[1], E[4], E[7]};
    const double v2[3] = {v0[1] * v1[2] - v0[2] * v1[1], v0[2] * v1[0] - v0[0] * v1[2], v0[0] * v1[1] - v0[1] * v1[0]};
    double u0[3], u1[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        u0[i] = dot3(H + 3 * i, v0);
        u1[i] = dot3(H + 3 * i, v1);
    }
    const double n0 = 1.0 / sqrt(dot3(u0, u0));
#pragma unroll
    for (int i = 0; i < 3; ++i) u0[i] *= n0;
    const double pr = dot3(u0, u1);
#pragma unroll
    for (int i = 0; i < 3; ++i) u1[i] -= pr * u0[i];
    const double n1 = 1.0 / sqrt(dot3(u1, u1));
#pragma unroll
    for (int i = 0; i < 3; ++i) u1[i] *= n1;
    const double u2[3] = {u0[1] * u1[2] - u0[2] * u1[1], u0[2] * u1[0] - u0[0] * u1[2], u0[0] * u1[1] - u0[1] * u1[0]};
    const double det = H[0] * (H[4] * H[8] - H[5] * H[7]) - H[1] * (H[3] * H[8] - H[5] * H[6]) +
                       H[2] * (H[3] * H[7] - H[4] * H[6]);
    const double sg = det < 0 ? -1.0 : 1.0;         // U V^T is a reflection where det(H) < 0
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) R[3 * i + j] = u0[i] * v0[j] + u1[i] * v1[j] + sg * u2[i] * v2[j];
    if (sg < 0) {
        R[6] = -R[6];
        R[7] = -R[7];
        R[8] = -R[8];
    }
}

struct EpnpCamera {
    double fx, fy, cx, cy;
    const double *per_image;        // row-major [b,3,3] on the device, or null: every image uses (fx, fy, cx, cy)
};

__global__ void __launch_bounds__(32 * EPNP_WARPS)
    k_epnp(const float *__restrict__ kp, const float *__restrict__ pts3d, EpnpCamera cam, int nb, int n,
           double *__restrict__ out_pose, int *__restrict__ out_info)
{
    __shared__ EpnpShared s_all[EPNP_WARPS];
    const int img = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (img >= nb) return;
    EpnpShared &sh = s_all[threadIdx.x >> 5];
    double fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy;
    if (cam.per_image) {
        const double *k = cam.per_image + (size_t)img * 9;
        fx = k[0];
        cx = k[2];
        fy = k[4];
        cy = k[5];
    }
    if (!(fx != 0.0 && fy != 0.0)) {                // warp-uniform: the whole warp leaves
        if (lane == 0) {
            for (int i = 0; i < 12; ++i) out_pose[(size_t)img * 12 + i] = __longlong_as_double(0x7ff8000000000000ll);
            if (out_info) {
                out_info[img * 2] = EPNP_STATUS_BAD_CAMERA;
                out_info[img * 2 + 1] = 0;
            }
        }
        return;
    }
    const float *x2 = kp + (size_t)img * n * 2;
    int status = 0;

    // ---- 1. control points
    double c0[3] = {0, 0, 0};
    for (int i = lane; i < n; i += 32)
#pragma unroll
        for (int k = 0; k < 3; ++k) c0[k] += pts3d[3 * i + k];
#pragma unroll
    for (int k = 0; k < 3; ++k) c0[k] = wsum(c0[k]) / n;
    double A[9];
    {
        double a6[6] = {0, 0, 0, 0, 0, 0};
        for (int i = lane; i < n; i += 32) {
            const double d0 = pts3d[3 * i] - c0[0], d1 = pts3d[3 * i + 1] - c0[1], d2 = pts3d[3 * i + 2] - c0[2];
            a6[0] += d0 * d0;
            a6[1] += d0 * d1;
            a6[2] += d0 * d2;
            a6[3] += d1 * d1;
            a6[4] += d1 * d2;
            a6[5] += d2 * d2;
        }
#pragma unroll
        for (int k = 0; k < 6; ++k) a6[k] = wsum(a6[k]);
        A[0] = a6[0]; A[1] = a6[1]; A[2] = a6[2];
        A[3] = a6[1]; A[4] = a6[3]; A[5] = a6[4];
        A[6] = a6[2]; A[7] = a6[4]; A[8] = a6[5];
    }
    double lam[3], V[9], sk[3];
    pca3(A, lam, V);
    if (!(lam[2] > EPNP_PCA_DEGENERATE * lam[0])) status |= EPNP_STATUS_DEGENERATE;
#pragma unroll
    for (int k = 0; k < 3; ++k) sk[k] = sqrt(fmax(lam[k], EPNP_PCA_DEGENERATE * lam[0]) / n);

    // ---- 2-3. barycentric coordinates and the moments of M^T M
    // one moment kind per pass, so that only ten sums are live: m = 0: alpha_j alpha_k; 1: x du; 2: x dv;
    // 3: x (du^2 + dv^2), with du = cx - u, dv = cy - v
#pragma unroll 1
    for (int m = 0; m < 4; ++m) {
        double S[10];
#pragma unroll
        for (int k = 0; k < 10; ++k) S[k] = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double d[3] = {pts3d[3 * i] - c0[0], pts3d[3 * i + 1] - c0[1], pts3d[3 * i + 2] - c0[2]};
            double al[4];
            al[1] = dot3(V, d) / sk[0];
            al[2] = dot3(V + 3, d) / sk[1];
            al[3] = dot3(V + 6, d) / sk[2];
            al[0] = 1.0 - (al[1] + al[2] + al[3]);
            const double du = cx - (double)x2[2 * i], dv = cy - (double)x2[2 * i + 1];
            const double w = m == 0 ? 1.0 : m == 1 ? du : m == 2 ? dv : du * du + dv * dv;
            int q = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int k = j; k < 4; ++k, ++q) S[q] += m == 0 ? al[j] * al[k] : al[j] * al[k] * w;
        }
#pragma unroll
        for (int k = 0; k < 10; ++k) S[k] = wsum(S[k]);
        for (int e = lane; e < 144; e += 32) {
            const int r = e / 12, c = e % 12, j = r / 3, k = c / 3, a = r % 3, b = c % 3;
            const int jj = j < k ? j : k, kk = j < k ? k : j;
            const int q = jj * 4 - jj * (jj - 1) / 2 + (kk - jj);     // index of (jj, kk) in the j <= k order
            double Sq = 0.0;
#pragma unroll
            for (int t = 0; t < 10; ++t) Sq = t == q ? S[t] : Sq;
            const int kind = (a == 2 && b == 2) ? 3 : (a == 2 || b == 2) ? (a + b == 2 ? 1 : 2) : (a == b ? 0 : -1);
            if (m == 0 && kind == -1) sh.A[e] = 0.0;
            if (kind != m) continue;
            sh.A[e] = m == 0 ? (a == 0 ? fx * fx : fy * fy) * Sq : m == 1 ? fx * Sq : m == 2 ? fy * Sq : Sq;
        }
    }
    __syncwarp();

    // ---- 4. null-space basis
    jacobi12(sh, lane);

    // ---- 5. L and rho over the control-point pairs (0,1),(0,2),(0,3),(1,2),(1,3),(2,3)
    if (lane < 6) {
        const int pa = lane < 3 ? 0 : (lane < 5 ? 1 : 2);
        const int pb = lane < 3 ? lane + 1 : (lane < 5 ? lane - 1 : 3);
        double dv4[4][3];
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int c = 0; c < 3; ++c) dv4[k][c] = vv(sh, k, 3 * pa + c) - vv(sh, k, 3 * pb + c);
        double *l = sh.L + 10 * lane;
        l[0] = dot3(dv4[0], dv4[0]);
        l[1] = 2.0 * dot3(dv4[0], dv4[1]);
        l[2] = dot3(dv4[1], dv4[1]);
        l[3] = 2.0 * dot3(dv4[0], dv4[2]);
        l[4] = 2.0 * dot3(dv4[1], dv4[2]);
        l[5] = dot3(dv4[2], dv4[2]);
        l[6] = 2.0 * dot3(dv4[0], dv4[3]);
        l[7] = 2.0 * dot3(dv4[1], dv4[3]);
        l[8] = 2.0 * dot3(dv4[2], dv4[3]);
        l[9] = dot3(dv4[3], dv4[3]);
        double ca[3], cb[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            ca[c] = pa == 0 ? c0[c] : c0[c] + sk[pa - 1] * V[3 * (pa - 1) + c];
            cb[c] = c0[c] + sk[pb - 1] * V[3 * (pb - 1) + c];
        }
        const double e[3] = {ca[0] - cb[0], ca[1] - cb[1], ca[2] - cb[2]};
        sh.rho[lane] = dot3(e, e);
    }
    __syncwarp();

    // Procrustes moments Q_k = A V_k / s_k, and the first point's barycentric coordinates (sign fix)
    double Q[9], al0[4];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) Q[3 * k + c] = dot3(V + 3 * k, A + 3 * c) / sk[k];
    {
        const double d[3] = {pts3d[0] - c0[0], pts3d[1] - c0[1], pts3d[2] - c0[2]};
        al0[1] = dot3(V, d) / sk[0];
        al0[2] = dot3(V + 3, d) / sk[1];
        al0[3] = dot3(V + 6, d) / sk[2];
        al0[0] = 1.0 - (al0[1] + al0[2] + al0[3]);
    }

    // ---- 6-8. three linearisations, Gauss-Newton, pose and error; keep the best
    double best_err = 0.0, best[12];
    int best_n = 0;
#pragma unroll 1
    for (int N = 1; N <= 3; ++N) {
        double be[4];
        betas(sh, N, be);
        gauss_newton(sh, be);
        double ccs[4][3];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                ccs[j][c] = be[0] * vv(sh, 0, 3 * j + c) + be[1] * vv(sh, 1, 3 * j + c) + be[2] * vv(sh, 2, 3 * j + c) +
                            be[3] * vv(sh, 3, 3 * j + c);
        if (al0[0] * ccs[0][2] + al0[1] * ccs[1][2] + al0[2] * ccs[2][2] + al0[3] * ccs[3][2] < 0) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c = 0; c < 3; ++c) ccs[j][c] = -ccs[j][c];
        }
        double H[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                H[3 * r + c] = (ccs[1][r] - ccs[0][r]) * Q[c] + (ccs[2][r] - ccs[0][r]) * Q[3 + c] +
                               (ccs[3][r] - ccs[0][r]) * Q[6 + c];
        double R[9], t[3];
        procrustes(H, R);
#pragma unroll
        for (int r = 0; r < 3; ++r) t[r] = ccs[0][r] - dot3(R + 3 * r, c0);
        double err = 0.0;
        for (int i = lane; i < n; i += 32) {
            const double p[3] = {pts3d[3 * i], pts3d[3 * i + 1], pts3d[3 * i + 2]};
            const double X = dot3(R, p) + t[0], Y = dot3(R + 3, p) + t[1], Z = dot3(R + 6, p) + t[2];
            const double eu = fx * X / Z + cx - (double)x2[2 * i], ev = fy * Y / Z + cy - (double)x2[2 * i + 1];
            err += sqrt(eu * eu + ev * ev);
        }
        err = wsum(err) / n;
        if (N == 1 || err < best_err) {
            best_err = err;
            best_n = N;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                best[4 * r] = R[3 * r];
                best[4 * r + 1] = R[3 * r + 1];
                best[4 * r + 2] = R[3 * r + 2];
                best[4 * r + 3] = t[r];
            }
        }
    }
    if (lane == 0) {
        for (int i = 0; i < 12; ++i) out_pose[(size_t)img * 12 + i] = best[i];
        if (out_info) {
            out_info[img * 2] = status;
            out_info[img * 2 + 1] = best_n;
        }
    }
}

}  // namespace

extern "C" {

static int launch_epnp(const float *points_2d, const float *points_3d, EpnpCamera cam, int b, int pn,
                       double *out_pose, int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(points_2d && points_3d && out_pose, "null pointer");
    PV_CHECK_ARG(b >= 1, "non-positive batch");
    PV_CHECK_ARG(pn >= 4 && pn <= EPNP_MAX_POINTS, "point count %d outside [4,%d]", pn, EPNP_MAX_POINTS);
    // one warp per CTA up to a few images per SM (the solve is a serial fp64 chain per warp), four beyond
    const int warps_per_cta = b <= 592 ? 1 : EPNP_WARPS;
    k_epnp<<<(b + warps_per_cta - 1) / warps_per_cta, 32 * warps_per_cta, 0, (cudaStream_t)stream>>>(
        points_2d, points_3d, cam, b, pn, out_pose, out_info);
    PV_LAUNCHED("k_epnp");
    return PVNET_OK;
}

int pvnet_epnp(const float *points_2d, const float *points_3d, const double camera_matrix[9], int b, int pn,
               double *out_pose, int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(camera_matrix, "null pointer");
    const double fx = camera_matrix[0], fy = camera_matrix[4], cx = camera_matrix[2], cy = camera_matrix[5];
    PV_CHECK_ARG(fx != 0.0 && fy != 0.0, "zero focal length");
    return launch_epnp(points_2d, points_3d, EpnpCamera{fx, fy, cx, cy, nullptr}, b, pn, out_pose, out_info, stream);
}

int pvnet_epnp_per_image_k(const float *points_2d, const float *points_3d, const double *camera_matrices, int b,
                           int pn, double *out_pose, int32_t *out_info, pvnet_stream_t stream)
{
    PV_CHECK_ARG(camera_matrices, "null pointer");
    return launch_epnp(points_2d, points_3d, EpnpCamera{0.0, 0.0, 0.0, 0.0, camera_matrices}, b, pn, out_pose,
                       out_info, stream);
}

}  // extern "C"
