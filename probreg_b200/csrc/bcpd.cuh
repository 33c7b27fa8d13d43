// bcpd.cuh -- device code of the BCPD registration loop (CombinedBCPD, probreg/bcpd.py:82-156) resident on the H100.
//
// One iteration, given the similarity s, R, t, the displacement v, the mixing weights alpha, diag(Sigma) and sigma2 of the last one:
//   E-step      T(y) = s R (y + v) + t (bcpd_move_kernel), per-source exponents la_m = -log2(alpha_m (1 - w) exp(-s^2 Sigma_mm D / 2 sigma2))
//               (bcpd_la_*: also what cpd_bcpd_estep runs), the weighted pair passes of kernels.cuh -> nu_d, nu, px
//   precision   A = lmd G^-1 + ratio diag(nu),  ratio = (s / sigma2)^2 (bcpd.py:129), FP64, with Sigma := I beside it (bcpd_system_kernel)
//   covariance  Sigma = A^-1 by cuSOLVER's LU and a solve against the identity (the host code in host_bcpd.inl)
//   displacement  v = ratio Sigma r,  r_m = R^T (px_m - nu_m t) / s - nu_m y_m   (== nu (T^-1(x_hat) - y) without dividing by nu)
//   weights     alpha_m = exp(psi(k + nu_m) - psi(k M + n_p)),  sigma2_m = sum nu_m Sigma_mm / n_p
//   similarity  S_xu = sum (px_m - nu_m xbar)(u_m - ubar)^T / n_p,  tr S_uu = sum nu_m |u_m - ubar|^2 / n_p + D sigma2_m,
//               Procrustes with the reference's sign fix, s = tr(R S_xu) / tr S_uu, t = xbar - s R ubar       (bcpd.py:138-150)
//   sigma2      (sum nu_d |x|^2 - 2 sum px . yhat + sum nu |yhat|^2) / (n_p D) + s^2 sigma2_m, yhat = T_prev(u)  (bcpd.py:151-155)
//               -- evaluated in the targets' centred frame (x - cx, yhat - cx): the same value, since sum nu_d = sum nu and
//               sum_n nu_d x_n = sum_m px_m, without the centroid offset in the cancellation.
// All vectors are in the library's internal (Z-order) source order; the M x M matrices are row-major in that order.
// The low-rank loop (cpd_bcpd_lowrank_begin) replaces the precision, covariance and displacement steps by the K x K algebra at the
// end of this file.
#pragma once
#include "kernels.cuh"
#include "lowrank.cuh"

namespace cpd {

// Loop state of a handle's BCPD registration (device memory; the host reads it back only on request)
struct BcpdState {
    double rot[9];        // similarity of the current transformation: y -> scale rot (y + v) + t   (rot 3 x 3 row-major)
    double t[3];
    double scale;         // scale, sigma2, w: contiguous, read as one triple by bcpd_la_kernel
    double sigma2;
    double w;
    double lmd, k;
    double n_p;           // of the last E-step
    double sigma2_m;      // sum nu Sigma_mm / n_p of the last M-step
};

// la_m = -log2(alpha_m) - log2(1 - w) + scale^2 / (2 sigma2) D log2(e) Sigma_mm (FP64; +inf for alpha_m = 0) and per-block minima.
// ssw = {scale, sigma2, w}.
__global__ void __launch_bounds__(THREADS)
bcpd_la_kernel(const double* __restrict__ alpha, const double* __restrict__ sdiag, long long m, const double* __restrict__ ssw, int dim,
               double* __restrict__ la, double* __restrict__ part_min) {
    __shared__ double sh[THREADS / 32];
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    const double scale = ssw[0], sigma2 = ssw[1], w = ssw[2];
    double v = INFINITY;
    if (i < m) {
        const double kf = scale * scale / (2.0 * sigma2) * (double)dim * LOG2E, l1w = -log2(1.0 - w);
        const double a = alpha[i];
        v = (a > 0.0 ? -log2(a) : INFINITY) + l1w + kf * sdiag[i];
        la[i] = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < THREADS / 32; ++k) v = fmin(v, sh[k]);
        part_min[blockIdx.x] = v;
    }
}
// la_min over the block minima, then the constants finalize1 reads (cpd_bcpd_estep's comment in cpd_b200.cu explains them):
//   log2c[0] = log2(w / N) + la_min + (D/2) log2(2 pi sigma2)  (-inf when w = 0),  log2c[1] = min(0, -la_min - (D/2) log2(2 pi sigma2)),
//   log2c[2] = la_min.   One warp.
__global__ void __launch_bounds__(32)
bcpd_la_finish_kernel(const double* __restrict__ part_min, int nb, const double* __restrict__ ssw, int dim, long long n_global,
                      double* __restrict__ log2c) {
    double v = INFINITY;
    for (int b = threadIdx.x; b < nb; b += 32) v = fmin(v, part_min[b]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (threadIdx.x == 0) {
        const double sigma2 = ssw[1], w = ssw[2];
        const double half_d_log2 = 0.5 * (double)dim * log2(2.0 * 3.14159265358979323846 * sigma2);
        log2c[0] = (w > 0.0) ? log2(w / (double)n_global) + v + half_d_log2 : -INFINITY;
        log2c[1] = fmin(0.0, -v - half_d_log2);
        log2c[2] = v;
    }
}
// the float32 exponents the pair passes read: out[k] = min(la[perm[k]] - la_min, 1e30) (perm == null: already in internal order);
// +inf (a zero weight) becomes 1e30, a weight of exactly 0 in the passes
__global__ void __launch_bounds__(THREADS)
bcpd_la_apply_kernel(const double* __restrict__ la, const int* __restrict__ perm, long long m, const double* __restrict__ log2c,
                     float* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < m) out[k] = (float)fmin(la[perm ? perm[k] : k] - log2c[2], 1.0e30);
}

// ts_m = s R (y_m + v_m) + t in the caller's frame (y = yc + cy)
__global__ void __launch_bounds__(THREADS)
bcpd_move_kernel(const BcpdState* __restrict__ bc, const double* __restrict__ yc, double c0, double c1, double c2,
                 const double* __restrict__ v, long long m, double* __restrict__ ts) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const double u[3] = {yc[3 * i] + c0 + v[3 * i], yc[3 * i + 1] + c1 + v[3 * i + 1], yc[3 * i + 2] + c2 + v[3 * i + 2]};
        const double s = bc->scale;
#pragma unroll
        for (int a = 0; a < 3; ++a)
            ts[3 * i + a] = s * (bc->rot[3 * a] * u[0] + bc->rot[3 * a + 1] * u[1] + bc->rot[3 * a + 2] * u[2]) + bc->t[a];
    }
}

// A = lmd G^-1 + ratio diag(nu) (FP64, row-major) and S = I, the right-hand side the solve overwrites with Sigma = A^-1.
// Rows on grid.x (grid.y is limited to 65535).
__global__ void __launch_bounds__(THREADS)
bcpd_system_kernel(const float* __restrict__ ginv, const double* __restrict__ nu, const BcpdState* __restrict__ bc, long long m,
                   double* __restrict__ A, double* __restrict__ S) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;
    const long long i = blockIdx.x;
    if (j < m) {
        const double r = bc->scale / bc->sigma2, ratio = r * r;
        A[i * m + j] = bc->lmd * (double)ginv[i * m + j] + (i == j ? ratio * nu[i] : 0.0);
        S[i * m + j] = (i == j) ? 1.0 : 0.0;
    }
}

// r_i = R^T (px_i - nu_i t) / s - nu_i y_i, px = pxc + nu cx, y = yc + cy; element a is stored at r[a * stride_a + i * stride_i]
__device__ __forceinline__ void bcpd_rhs_point(const BcpdState* __restrict__ bc, const DevState* __restrict__ st, const double* __restrict__ nu,
                                               const double* __restrict__ pxc, const double* __restrict__ yc, long long i, double* __restrict__ r,
                                               long long stride_a, long long stride_i) {
    const double n = nu[i];
    double q[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) q[a] = pxc[3 * i + a] + n * (st->cx[a] - bc->t[a]);
    const double inv_s = 1.0 / bc->scale;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double rt = bc->rot[a] * q[0] + bc->rot[3 + a] * q[1] + bc->rot[6 + a] * q[2];      // (R^T q)_a
        r[a * stride_a + i * stride_i] = rt * inv_s - n * (yc[3 * i + a] + st->cy[a]);
    }
}
// r (m x 3, point-major) for the dense M-step
__global__ void __launch_bounds__(THREADS)
bcpd_rhs_kernel(const BcpdState* __restrict__ bc, const DevState* __restrict__ st, const double* __restrict__ nu,
                const double* __restrict__ pxc, const double* __restrict__ yc, long long m, double* __restrict__ r) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) bcpd_rhs_point(bc, st, nu, pxc, yc, i, r, 1, 3);
}

// v_i = ratio sum_j Sigma_ij r_j (one warp per row, FP64) and sdiag_i = Sigma_ii
__global__ void __launch_bounds__(THREADS)
bcpd_disp_kernel(const double* __restrict__ S, const double* __restrict__ r, const BcpdState* __restrict__ bc, long long m,
                 double* __restrict__ v, double* __restrict__ sdiag) {
    const long long i = (long long)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    const double* row = S + i * m;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (long long j = lane; j < m; j += 32) {
        const double g = row[j];
        a0 += g * r[3 * j]; a1 += g * r[3 * j + 1]; a2 += g * r[3 * j + 2];
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    if (lane == 0) {
        const double q = bc->scale / bc->sigma2, ratio = q * q;
        v[3 * i] = ratio * a0; v[3 * i + 1] = ratio * a1; v[3 * i + 2] = ratio * a2;
        sdiag[i] = row[i];
    }
}

// First moment pass, per-block partials of BCPD_KA sums (u~ = yc + v: the deformed source centred on cy;
// yhat~ = T_prev(u) - cx = s R (u~ + cy) + t - cx):
//   [0] nu  [1..3] pxc  [4..6] nu u~  [7] nu Sigma_mm  [8] pxc . yhat~  [9] nu |yhat~|^2
constexpr int BCPD_KA = 10, BCPD_KB = 10;
__global__ void __launch_bounds__(THREADS)
bcpd_moments_a_kernel(const BcpdState* __restrict__ bc, const DevState* __restrict__ st, const double* __restrict__ nu,
                      const double* __restrict__ pxc, const double* __restrict__ yc, const double* __restrict__ v,
                      const double* __restrict__ sdiag, long long m, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double acc[BCPD_KA];
#pragma unroll
    for (int k = 0; k < BCPD_KA; ++k) acc[k] = 0.0;
    if (i < m) {
        const double n = nu[i];
        double u[3], yh[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) u[a] = yc[3 * i + a] + v[3 * i + a];
        const double s = bc->scale;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double ru = bc->rot[3 * a] * (u[0] + st->cy[0]) + bc->rot[3 * a + 1] * (u[1] + st->cy[1]) + bc->rot[3 * a + 2] * (u[2] + st->cy[2]);
            yh[a] = s * ru + bc->t[a] - st->cx[a];
        }
        acc[0] = n;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double p = pxc[3 * i + a];
            acc[1 + a] = p;
            acc[4 + a] = n * u[a];
            acc[8] += p * yh[a];
            acc[9] += n * yh[a] * yh[a];
        }
        acc[7] = n * sdiag[i];
    }
    block_reduce_store<BCPD_KA>(acc, part + (size_t)blockIdx.x * BCPD_KA);
}

// psi(x), x > 0: the recurrence psi(x) = psi(x + 1) - 1/x up to x >= 10, then the asymptotic series to x^-14 (truncation below
// 1e-17 there)
__device__ inline double bcpd_digamma(double x) {
    double acc = 0.0;
    while (x < 10.0) { acc -= 1.0 / x; x += 1.0; }
    const double r = 1.0 / x, r2 = r * r;
    const double series = r2 * (1.0 / 12 - r2 * (1.0 / 120 - r2 * (1.0 / 252 - r2 * (1.0 / 240 - r2 * (1.0 / 132 - r2 * (691.0 / 32760 - r2 / 12))))));
    return acc + log(x) - 0.5 * r - series;
}

// the new mixing weights alpha_m = exp(psi(k + nu_m) - psi(k M + n_p)) (bcpd.py:137); n_p = sums_a[0]
__global__ void __launch_bounds__(THREADS)
bcpd_alpha_kernel(const BcpdState* __restrict__ bc, const double* __restrict__ sums_a, const double* __restrict__ nu, long long m,
                  double* __restrict__ alpha) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const double k = bc->k;
        alpha[i] = exp(bcpd_digamma(k + nu[i]) - bcpd_digamma(k * (double)m + sums_a[0]));
    }
}

// Second moment pass (needs the means of the first): per-block partials of
//   [0..8] (pxc - nu xbar~)(u~ - ubar~)^T (row-major 3 x 3)  [9] nu |u~ - ubar~|^2
__global__ void __launch_bounds__(THREADS)
bcpd_moments_b_kernel(const double* __restrict__ sums_a, const double* __restrict__ nu, const double* __restrict__ pxc,
                      const double* __restrict__ yc, const double* __restrict__ v, long long m, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double acc[BCPD_KB];
#pragma unroll
    for (int k = 0; k < BCPD_KB; ++k) acc[k] = 0.0;
    if (i < m) {
        const double n_p = sums_a[0], n = nu[i];
        double dx[3], du[3];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            dx[a] = pxc[3 * i + a] - n * (sums_a[1 + a] / n_p);
            du[a] = yc[3 * i + a] + v[3 * i + a] - sums_a[4 + a] / n_p;
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
            for (int b = 0; b < 3; ++b) acc[3 * a + b] = dx[a] * du[b];
            acc[9] += n * du[a] * du[a];
        }
    }
    block_reduce_store<BCPD_KB>(acc, part + (size_t)blockIdx.x * BCPD_KB);
}

// The similarity and sigma2 of bcpd.py:138-155 from the reduced sums (one thread, FP64):
//   sums_a (BCPD_KA), sums_b (BCPD_KB), sums_t[4] = sum nu_d |x - cx|^2 (tgt_moments_api_kernel's last column).
__global__ void __launch_bounds__(32)
bcpd_mstep_kernel(BcpdState* bc, const DevState* __restrict__ st, const double* __restrict__ sums_a, const double* __restrict__ sums_b,
                  const double* __restrict__ sums_t, int dim) {
    if (threadIdx.x != 0) return;
    const int n = dim;
    const double n_p = sums_a[0];
    const double sigma2_m = sums_a[7] / n_p;
    double xbar[3], ubar[3], Sxu[3][3];
    for (int a = 0; a < 3; ++a) {
        xbar[a] = st->cx[a] + sums_a[1 + a] / n_p;
        ubar[a] = st->cy[a] + sums_a[4 + a] / n_p;
        for (int b = 0; b < 3; ++b) Sxu[a][b] = (a < n && b < n) ? sums_b[3 * a + b] / n_p : 0.0;
    }
    const double tr_suu = sums_b[9] / n_p + n * sigma2_m;
    double U[3][3], sv[3], V[3][3], UVt[3][3], rot[3][3];
    jacobi_svd(n, Sxu, U, sv, V);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { double t = 0; for (int k = 0; k < n; ++k) t += U[i][k] * V[j][k]; UVt[i][j] = t; }
    const double dt = det_n(n, UVt);                                                     // bcpd.py:141-142
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double t = 0;
            for (int k = 0; k < n; ++k) t += U[i][k] * (k == n - 1 ? dt : 1.0) * V[j][k];
            rot[i][j] = (i < n && j < n) ? t : (i == j ? 1.0 : 0.0);                      // bcpd.py:143
        }
    double tr_rsxu = 0.0;                                                                // trace(rot S_xu), bcpd.py:144
    for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) tr_rsxu += rot[i][j] * Sxu[j][i];
    const double scale = tr_rsxu / tr_suu;
    const double sigma2 = (sums_t[4] - 2.0 * sums_a[8] + sums_a[9]) / (n_p * n) + scale * scale * sigma2_m;
    for (int a = 0; a < 3; ++a) {
        const double ru = rot[a][0] * ubar[0] + rot[a][1] * ubar[1] + rot[a][2] * ubar[2];
        bc->t[a] = (a < n) ? xbar[a] - scale * ru : 0.0;
        for (int b = 0; b < 3; ++b) bc->rot[3 * a + b] = rot[a][b];
    }
    bc->scale = scale;
    bc->sigma2 = sigma2;
    bc->n_p = n_p;
    bc->sigma2_m = sigma2_m;
}

// out[i][j] = in[perm[i]][perm[j]] (m x m float32, row-major): G^-1 from the caller's point order into the internal one
__global__ void __launch_bounds__(THREADS)
bcpd_gather2d_kernel(const float* __restrict__ in, const int* __restrict__ perm, long long m, float* __restrict__ out) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;
    const long long i = blockIdx.x;
    if (j < m) out[i * m + j] = in[(long long)perm[i] * m + perm[j]];
}
// x[k] = value (k < count)
__global__ void __launch_bounds__(THREADS)
bcpd_fill_kernel(double* __restrict__ x, long long count, double value) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < count) x[k] = value;
}

// ---- the low-rank M-step (cpd_bcpd_lowrank_begin) ---------------------------------------------------------------------------------
// With G ~= Qt Qt^T (Qt = Q L of the set-up, lowrank.cuh: [K][ld], K columns) the displacement is v = Qt w with the prior
// w ~ N(0, I / lmd).  The posterior of w given the E-step is Gaussian with precision ratio (c I + St):
//     c = lmd / ratio,   St = Qt^T diag(nu) Qt,   C = (c I + St)^-1      (symmetric positive definite, eigenvalues of C^-1 >= c)
//     v = Qt C Rt,   Rt = Qt^T r      (r of bcpd_rhs_point: nu (T^-1(x_hat) - y) without dividing by nu)
//     diag Sigma_v = diag(Qt C Qt^T) / ratio = sum_k Qt[k][i] (C Qt^T)[k][i] / ratio      (FP64, >= 0, no M x M buffer)
// At K = M with Qt of full rank this is (lmd G^-1 + ratio diag(nu))^-1: the dense loop's Sigma.  No G^-1, no Bc^-1, no division by
// nu: a source no target explains keeps a finite v, and a column the pivoted Cholesky dropped (zero in Qt) gives St a zero row and
// column, where C = 1 / c.  Mixing weights, similarity and sigma2 follow with the dense loop's kernels.

// r in the [3][m] layout lr_inner_narrow_kernel reads
__global__ void __launch_bounds__(THREADS)
bcpd_lr_rhs_kernel(const BcpdState* __restrict__ bc, const DevState* __restrict__ st, const double* __restrict__ nu,
                   const double* __restrict__ pxc, const double* __restrict__ yc, long long m, double* __restrict__ r) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) bcpd_rhs_point(bc, st, nu, pxc, yc, i, r, m, 1);
}
// Msys = c I + St (row-major K x K), c = lmd / ratio from the loop state, and E = I, the right-hand side the solve overwrites with C
__global__ void __launch_bounds__(THREADS)
bcpd_lr_system_kernel(const double* __restrict__ St, const BcpdState* __restrict__ bc, int K, double* __restrict__ Msys, double* __restrict__ E) {
    const long long e = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (e < (long long)K * K) {
        const double q = bc->scale / bc->sigma2, c = bc->lmd / (q * q);
        const bool diag = e / K == e % K;
        Msys[e] = St[e] + (diag ? c : 0.0);
        E[e] = diag ? 1.0 : 0.0;
    }
}
// w[k][d] = sum_b C[k][b] Rt[b][d]   (K x 3; Rt as lr_merge_kernel leaves it, [K][3])
__global__ void __launch_bounds__(THREADS)
bcpd_lr_coef_kernel(const double* __restrict__ C, const double* __restrict__ Rt, int K, double* __restrict__ w) {
    const int e = blockIdx.x * THREADS + threadIdx.x;
    if (e < 3 * K) {
        const int k = e / 3, d = e % 3;
        double s = 0.0;
        for (int b = 0; b < K; ++b) s = fma(C[(size_t)k * K + b], Rt[(size_t)b * 3 + d], s);
        w[e] = s;
    }
}
// v_i = sum_k Qt[k][i] w[k]  (m x 3, point-major) and sdiag_i = sum_k Qt[k][i] CQ[k][i] / ratio, CQ = C Qt^T (lr_rotate_kernel)
__global__ void __launch_bounds__(THREADS)
bcpd_lr_disp_kernel(const double* __restrict__ Qt, const double* __restrict__ CQ, long long ld, int K, const double* __restrict__ w,
                    const BcpdState* __restrict__ bc, long long m, double* __restrict__ v, double* __restrict__ sdiag) {
    __shared__ double sw[3 * LR_MAX_RANK];
    for (int e = threadIdx.x; e < 3 * K; e += THREADS) sw[e] = w[e];
    __syncthreads();
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, sd = 0.0;
        for (int k = 0; k < K; ++k) {
            const double q = Qt[(long long)k * ld + i];
            a0 = fma(q, sw[3 * k], a0); a1 = fma(q, sw[3 * k + 1], a1); a2 = fma(q, sw[3 * k + 2], a2);
            sd = fma(q, CQ[(long long)k * ld + i], sd);
        }
        const double r = bc->scale / bc->sigma2;
        v[3 * i] = a0; v[3 * i + 1] = a1; v[3 * i + 2] = a2;
        sdiag[i] = sd / (r * r);
    }
}

}  // namespace cpd
