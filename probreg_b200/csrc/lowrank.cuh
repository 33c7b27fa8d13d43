// lowrank.cuh -- non-rigid CPD with a rank-K factorisation of the RBF Gram matrix
// (BASELINE configuration 5: N = M = 50k, K = 200).
//
// Reference: NonRigidCPD._maximization_step (probreg/cpd.py:284-303) solves the dense M x M system
//     (diag(p1) G + lmd sigma2 I) W = px - diag(p1) Y,        G_ij = exp(-|y_i - y_j|^2 / (2 beta))   (cc/math_utils.cc:17-19)
// -- 2/3 M^3 flops and 12 M^2 bytes per iteration (10^14 flops, 30 GB at M = 50k).  The reference has no low-rank path;
// this one follows the low-rank construction of the CPD paper (Myronenko & Song 2010, "fast implementation"), with the
// eigen-decomposition replaced by a randomised range finder that only needs products G X, which the pair kernel forms on
// the fly (G is never stored):
//     G ~= Q Bc Q^T,   Q (M x K) orthonormal columns,  Bc = Q^T G Q (K x K)
//     W  = (F - diag(p1) Q Z) / c,     c = lmd sigma2,  F = px - diag(p1) Y
//     Z  = Bc Q^T W  solves the K x K system  (c I + Bc S) Z = Bc R,   S = Q^T diag(p1) Q,  R = Q^T F
//     T  = Y + G W ~= Y + Q Z
// (Woodbury written without Bc^-1, so numerically rank-deficient Q -- zero columns -- is harmless.)
// The iteration runs on the factor Qt = Q L, Bc ~= L L^T, whose K x K system is symmetric positive definite and is
// solved by one CTA (lr_spd_form in host_nonrigid.inl, lr_pchol_kernel / lr_spd_solve_kernel below); the unsymmetric system above
// with cuSOLVER's LU remains for K > LR_SPD_MAX_RANK and as the cross-check (CPD_B200_LR_CORE=lu).
// Parity: against the dense device path / the numpy oracle at small M (tests); at K = M the two coincide up to rounding.
//
// Layout: Q, X, GQ are FP64 "column-major" [K][ld]: row k holds column k of the matrix, i contiguous -- every kernel below
// then reads them coalesced along i.  All arrays are in the library's internal (Z-order) source order.
#pragma once
#include "kernels.cuh"

namespace cpd {

#ifndef CPD_LR_COLS
#define CPD_LR_COLS 16
#endif
constexpr int LR_COLS = CPD_LR_COLS;   // columns of X handled per CTA of lr_gram_apply_kernel (tunable: -DCPD_LR_COLS=...)
constexpr int LR_JT = 256;        // j-points per shared-memory tile (== THREADS)
constexpr int LR_SLICES = 8;      // i-slices of lr_inner_kernel (partials merged in fixed order)
constexpr int LR_TILE = 32;       // output tile edge of lr_inner_kernel (2 x 2 outputs per thread)
constexpr int LR_CHUNK = 64;      // i-points per shared-memory chunk of lr_inner_kernel
constexpr int LR_MAX_RANK = 1024;

// ---- the kernel function of the G X products (a template parameter of both product kernels) ----------------------------------
//   LR_GAUSS  G_ij = exp(-|y_i - y_j|^2 / (2 beta))     (non-rigid CPD)   points a = y sqrt(log2(e) / (2 beta)),  G = 2^-u
//   LR_IMQ    G_ij = (|y_i - y_j|^2 + c)^(-1/2)         (BCPD, cc/math_utils.cc:37-39)
//                                                                         points a = y / sqrt(c),  G = c^(-1/2) G',  G' = (1 + u)^(-1/2)
// with u = |a_i - a_j|^2 in the scaled frame of lr_pack_kernel.  Both tile values lie in (0, 1], so the digits of the tensor-core
// product (gram_i8.cuh) are the same for both; the factor c^(-1/2) of the IMQ is applied to each FP64 output (`gscale`).
// The IMQ tile value is MUFU's rsqrt.approx.ftz.f32 of fl(1 + u): relative error <= 2^-22.9 (PTX ISA), on top of the one rounding
// of 1 + u (2^-24 relative); it is clamped to 1 so that G' = 1 keeps the digits (128, 0, 0).  The CPU emulation uses 1 / sqrtf.
constexpr int LR_GAUSS = 0, LR_IMQ = 1;
__device__ __forceinline__ float lr_rsqrt(float x) {
#ifdef CPD_HOST_EMU
    return 1.0f / sqrtf(x);
#else
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
#endif
}
template <int KIND>
__device__ __forceinline__ float lr_kernel_value(float u) {
    if constexpr (KIND == LR_GAUSS) return ex2(-u);
    else return fminf(lr_rsqrt(__fadd_rn(1.0f, u)), 1.0f);
}

// float32 coordinates scaled by sb (sqrt(log2(e) / (2 beta)) or 1 / sqrt(c), see above).  The cast to float32 comes first,
// like the pybind11/Eigen cast of the reference (cc/types.h:19); padding records are far away (G == 0; G' < 1e-18 for the IMQ,
// and their X entries are zero).
__global__ void __launch_bounds__(THREADS)
lr_pack_kernel(const double* __restrict__ yc, double c0, double c1, double c2, long long m, long long mpad, float sb,
               float4* __restrict__ pts) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) pts[i] = make_float4(sb * (float)(yc[3 * i] + c0), sb * (float)(yc[3 * i + 1] + c1), sb * (float)(yc[3 * i + 2] + c2), 0.0f);
    else if (i < mpad) pts[i] = make_float4(FAR_COORD, FAR_COORD, FAR_COORD, 0.0f);
}

// counter-based uniform(-1, 1) test matrix of the range finder: X[k][i] = u(seed, k, i)   (splitmix64 finaliser)
__global__ void __launch_bounds__(THREADS)
lr_random_kernel(double* __restrict__ X, long long m, long long ld, int rank, unsigned long long seed) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    const int k = blockIdx.y;
    if (i < m && k < rank) {
        unsigned long long z = seed + 0x9e3779b97f4a7c15ull * (unsigned long long)((long long)k * m + i + 1);
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        z ^= z >> 31;
        X[(long long)k * ld + i] = (double)(z >> 11) * (2.0 / 9007199254740992.0) - 1.0;
    }
}

// out[c][i] = sum_j G_ij X[c][j]  for the LR_COLS columns c0 .. c0+LR_COLS of this CTA's column group (blockIdx.y):
// the pair kernel of the E-step with a weight per column instead of the normalisation.  One i-point per thread,
// j-points and the X tile staged through shared memory, FP32 pair arithmetic and 32-term FP32 partial sums, FP64 beyond.
// KIND: LR_GAUSS or LR_IMQ (gscale = c^(-1/2) multiplies the FP64 outputs of the IMQ; unused for the Gaussian).
template <int KIND>
__global__ void __launch_bounds__(THREADS)
lr_gram_apply_kernel(const float4* __restrict__ pts, long long m, long long mpad, const double* __restrict__ X, long long ld, int rank,
                     double* __restrict__ out, long long i_begin, long long i_end /* rows of this launch: all, or one rank's share */,
                     double gscale) {
    __shared__ float4 sp[LR_JT];
    __shared__ __align__(16) float sx[LR_JT][LR_COLS];
    const long long i = i_begin + (long long)blockIdx.x * THREADS + threadIdx.x;
    const int c0 = blockIdx.y * LR_COLS;
    const float4 t = pts[i < i_end ? i : i_end - 1];
    double acc[LR_COLS];
#pragma unroll
    for (int c = 0; c < LR_COLS; ++c) acc[c] = 0.0;
    for (long long j0 = 0; j0 < mpad; j0 += LR_JT) {
        __syncthreads();
        const long long j = j0 + threadIdx.x;
        sp[threadIdx.x] = pts[j];                                  // j < mpad always (mpad is a multiple of LR_JT)
#pragma unroll
        for (int c = 0; c < LR_COLS; ++c) sx[threadIdx.x][c] = (j < m && c0 + c < rank) ? (float)X[(long long)(c0 + c) * ld + j] : 0.0f;
        __syncthreads();
#pragma unroll 1
        for (int g = 0; g < LR_JT; g += 32) {
            float a[LR_COLS];
#pragma unroll
            for (int c = 0; c < LR_COLS; ++c) a[c] = 0.0f;
#pragma unroll 4
            for (int jj = 0; jj < 32; ++jj) {
                const float4 b = sp[g + jj];
                const float dx = t.x - b.x, dy = t.y - b.y, dz = t.z - b.z;
                const float e = lr_kernel_value<KIND>(fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
                const float4* xr = reinterpret_cast<const float4*>(sx[g + jj]);
#pragma unroll
                for (int q = 0; q < LR_COLS / 4; ++q) {
                    const float4 xv = xr[q];
                    a[4 * q] = fmaf(e, xv.x, a[4 * q]); a[4 * q + 1] = fmaf(e, xv.y, a[4 * q + 1]);
                    a[4 * q + 2] = fmaf(e, xv.z, a[4 * q + 2]); a[4 * q + 3] = fmaf(e, xv.w, a[4 * q + 3]);
                }
            }
#pragma unroll
            for (int c = 0; c < LR_COLS; ++c) acc[c] += (double)a[c];
        }
    }
    if (i < i_end) {
#pragma unroll
        for (int c = 0; c < LR_COLS; ++c)
            if (c0 + c < rank) {
                if constexpr (KIND == LR_IMQ) out[(long long)(c0 + c) * ld + i] = acc[c] * gscale;
                else out[(long long)(c0 + c) * ld + i] = acc[c];
            }
    }
}

// ---- orthonormalisation of the columns of X (classical Gram-Schmidt, every column projected twice) ---------------------
// part[s][k] = <X_k, X_j> over the s-th of LR_SLICES point slices, for k = k_first .. j (the last one is |X_j|^2).
// One CTA per {k, slice}: a single CTA per k would stream 2 M doubles through one SM, whatever j is;
// consumers add the slices in a fixed order, so the result is reproducible.
__global__ void __launch_bounds__(THREADS)
lr_dots_kernel(const double* __restrict__ X, long long m, long long ld, int j, int k_first, int stride /* rank + 1 */,
               double* __restrict__ part) {
    const int k = k_first + blockIdx.x, slice = blockIdx.y, nsl = gridDim.y;      // nsl <= LR_SLICES, chosen by the host from m
    const long long per = (m + nsl - 1) / nsl;
    const long long i_lo = per * slice, i_hi = (i_lo + per < m) ? i_lo + per : m;
    const double* a = X + (long long)k * ld;
    const double* b = X + (long long)j * ld;
    double v[1] = {0.0};
    for (long long i = i_lo + threadIdx.x; i < i_hi; i += THREADS) v[0] += a[i] * b[i];
    block_reduce_store<1>(v, part + (size_t)slice * stride + k);
}
__device__ __forceinline__ double lr_sum_slices(const double* __restrict__ part, int stride, int nsl, int k) {
    double s = 0.0;
    for (int sl = 0; sl < nsl; ++sl) s += part[(size_t)sl * stride + k];
    return s;
}
// X_j -= sum_{k<j} coef[k] X_k,   coef[k] = sum over slices of part[.][k]
__global__ void __launch_bounds__(THREADS)
lr_project_kernel(double* __restrict__ X, long long m, long long ld, int j, int stride, int nsl, const double* __restrict__ part) {
    __shared__ double sc[LR_MAX_RANK];
    for (int k = threadIdx.x; k < j; k += THREADS) sc[k] = lr_sum_slices(part, stride, nsl, k);
    __syncthreads();
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        double x = X[(long long)j * ld + i];
        for (int k = 0; k < j; ++k) x -= sc[k] * X[(long long)k * ld + i];
        X[(long long)j * ld + i] = x;
    }
}
// X_j *= 1/|X_j|; a column that has (numerically) nothing left outside the span of its predecessors becomes zero.
// n0 = |X_j|^2 before the projections (slices of part0), n2 = after (slices of part2).
__global__ void __launch_bounds__(THREADS)
lr_scale_kernel(double* __restrict__ X, long long m, long long ld, int j, int stride, int nsl, const double* __restrict__ part0,
                const double* __restrict__ part2) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    const double n0 = lr_sum_slices(part0, stride, nsl, j), n2 = lr_sum_slices(part2, stride, nsl, j);
    const double s = (n2 > 1e-280 && n2 > 1e-28 * n0) ? 1.0 / sqrt(n2) : 0.0;
    if (i < m) X[(long long)j * ld + i] *= s;
}

// ---- blocked orthonormalisation (block classical Gram-Schmidt with re-orthogonalisation, panels of LR_PANEL columns) --------------
// Per panel P = X[j0 .. j0+np):   (a) P -= Q Q^T P  against the finished columns Q = X[0 .. j0)      (lr_panel_* below)
//                                 (b) P <- P T, T = R^-1 from the Cholesky factor of the panel's Gram matrix  (lr_panel_chol / _apply)
//                                 (c), (d): both once more.
// (b) leaves the columns normalised and orthogonal to ~eps / (relative pivot); (c) removes what (b) amplified along Q, at unit
// scale; (d) starts from a Gram matrix I + O(1e-6) and ends at rounding level -- the same O(eps) orthogonality as projecting every
// column twice on its own (lr_orthonormalise_columnwise), with 16 launches per 16 columns instead of 96 and each finished column
// read 4 times per PANEL instead of 4 times per COLUMN (the column-wise version moved 32 GB at M = 50k, K = 200).
// Rank decisions (a dropped column becomes exactly zero and stays zero in every later product, like before):
//   * nothing left after (a): norm^2 <= 1e-28 of the norm^2 the column arrived with -- the rule of the column-wise version;
//   * the same rule once more at (d), on what is left after the panel's own projections (lr_panel_chol_kernel).
constexpr int LR_PANEL = 16;
constexpr int LR_UPD_KC = 128;     // finished columns per shared-memory chunk of lr_panel_update_kernel

// X[j0+p][i] -= sum_{k<nk} C[k][p] X[k][i]      (C row-major [nk][np]: the merged output of lr_inner_kernel)
__global__ void __launch_bounds__(THREADS)
lr_panel_update_kernel(double* __restrict__ X, long long m, long long ld, int j0, int np, int nk, const double* __restrict__ C /* [nk][np] */) {
    __shared__ double sc[LR_UPD_KC][LR_PANEL];
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double acc[LR_PANEL];
#pragma unroll
    for (int p = 0; p < LR_PANEL; ++p) acc[p] = 0.0;
    for (int k0 = 0; k0 < nk; k0 += LR_UPD_KC) {
        const int kc = (nk - k0 < LR_UPD_KC) ? nk - k0 : LR_UPD_KC;
        __syncthreads();
        for (int e = threadIdx.x; e < kc * LR_PANEL; e += THREADS) {
            const int k = e / LR_PANEL, pp = e % LR_PANEL;
            sc[k][pp] = pp < np ? C[(size_t)(k0 + k) * np + pp] : 0.0;
        }
        __syncthreads();
        if (i < m) {
#pragma unroll 8
            for (int k = 0; k < kc; ++k) {
                const double q = X[(long long)(k0 + k) * ld + i];
#pragma unroll
                for (int p = 0; p < LR_PANEL; ++p) acc[p] = fma(sc[k][p], q, acc[p]);
            }
        }
    }
    if (i < m) {
#pragma unroll
        for (int p = 0; p < LR_PANEL; ++p)
            if (p < np) X[(long long)(j0 + p) * ld + i] -= acc[p];
    }
}

// part[blk][a][b] = sum over the block's points of X[j0+a][i] X[j0+b][i]   (a, b < LR_PANEL; rows >= np count as zero).
// One CTA per LR_GRAM_PTS points (grid-stride beyond that), thread (a, b): 256 threads = the 16 x 16 outputs.
constexpr int LR_GRAM_PTS = 256;
constexpr int LR_GRAM_BLOCKS = 1024;   // most CTAs of lr_panel_gram_kernel (beyond 262144 points they stride)
__global__ void __launch_bounds__(THREADS)
lr_panel_gram_kernel(const double* __restrict__ X, long long m, long long ld, int j0, int np, double* __restrict__ part) {
    __shared__ double sp[LR_PANEL][LR_GRAM_PTS + 1];           // + 1: the 16 rows a warp reads in one step fall into distinct banks
    const int a = threadIdx.x / LR_PANEL, b = threadIdx.x % LR_PANEL;
    double acc = 0.0;
    for (long long i0 = (long long)blockIdx.x * LR_GRAM_PTS; i0 < m; i0 += (long long)gridDim.x * LR_GRAM_PTS) {
        __syncthreads();
        for (int e = threadIdx.x; e < LR_PANEL * LR_GRAM_PTS; e += THREADS) {
            const int r = e / LR_GRAM_PTS, ii = e % LR_GRAM_PTS;
            sp[r][ii] = (r < np && i0 + ii < m) ? X[(long long)(j0 + r) * ld + i0 + ii] : 0.0;
        }
        __syncthreads();
#pragma unroll 8
        for (int ii = 0; ii < LR_GRAM_PTS; ++ii) acc = fma(sp[a][ii], sp[b][ii], acc);
    }
    part[(size_t)blockIdx.x * (LR_PANEL * LR_PANEL) + threadIdx.x] = acc;
}

// One CTA (256 threads): W = sum over blocks of part (fixed order), then T (upper triangular, row-major [LR_PANEL][LR_PANEL]) such
// that P T has orthonormal columns, by a Cholesky factorisation W = R^T R, T = R^-1.
//   mode 2 (arrival): only n0[p] = W[p][p] is stored -- the norm^2 each column of the panel arrived with.
//   mode 1 (step b):  a column with nothing left after (a) (norm^2 <= 1e-28 n0) is dropped.  A column whose pivot is lost in the
//       cancellation (<= 1e-13 of its norm^2: it lies in the span of its panel predecessors up to ~3e-7) is still projected with the
//       computed coefficients -- which removes the predecessors to rounding level -- but scaled by a guess and left out of the
//       factorisation of the later columns; step (d) sees it well separated and measures what is really left.
//       scale2[p] = the square of the factor column p was multiplied with.
//   mode 0 (step d):  scale2 from (b) turns the diagonal of W back into the column's remaining norm^2 in arrival units; the
//       column-wise rule (kept iff that is > 1e-28 n0) decides.  Dropped columns get a zero column in T and stay exactly zero.
// The factorisation is right-looking on one warp (lane = column): 16 steps of a few operations instead of one thread walking
// ~3000 dependent FP64 operations.
constexpr int LR_CHOL_THREADS = 1024;   // 4 threads per Gram entry for the merge of the block partials
__global__ void __launch_bounds__(LR_CHOL_THREADS)
lr_panel_chol_kernel(const double* __restrict__ part, int nblk, int np, double* __restrict__ n0, int mode, double* __restrict__ scale2,
                     double* __restrict__ T) {
    __shared__ double W[LR_PANEL][LR_PANEL + 1], R[LR_PANEL][LR_PANEL + 1], Ti[LR_PANEL][LR_PANEL + 1], diag0[LR_PANEL];
    __shared__ double wsum[4][LR_PANEL * LR_PANEL];
    __shared__ int live[LR_PANEL];          // 1: part of the factorisation, 2: projected and rescaled only, 0: dropped
    const int tid = threadIdx.x, t = tid & 255, a = t / LR_PANEL, b = t % LR_PANEL, lane4 = tid >> 8;
    {   // merge: thread group lane4 takes the blocks lane4, lane4 + 4, ...; the four sums are joined in a fixed order (the merge
        // of one thread per entry would be 196 dependent L2 round trips)
        double s = 0.0;
#pragma unroll 8
        for (int k = lane4; k < nblk; k += 4) s += part[(size_t)k * (LR_PANEL * LR_PANEL) + t];
        wsum[lane4][t] = s;
    }
    __syncthreads();
    if (tid < 256) { W[a][b] = (wsum[0][t] + wsum[1][t]) + (wsum[2][t] + wsum[3][t]); R[a][b] = 0.0; Ti[a][b] = 0.0; }
    __syncthreads();
    if (mode == 2) {
        if (tid < LR_PANEL) n0[tid] = W[tid][tid];
        return;
    }
    if (tid < LR_PANEL) diag0[tid] = W[tid][tid];
    __syncthreads();
    if (tid < 32) {
        const int lane = tid;               // lane = column index b of the row being formed / the Schur update
        for (int p = 0; p < np; ++p) {
            const double wpp = diag0[p], piv = W[p][p], arrived = n0[p];
            int state;
            if (mode == 1) state = !(wpp > 1e-280 && wpp > 1e-28 * arrived) ? 0 : (piv > 1e-13 * wpp ? 1 : 2);
            else state = (wpp > 1e-280 && wpp / scale2[p] > 1e-28 * arrived && piv > 1e-13 * wpp) ? 1 : 0;
            const double rpp = state == 1 ? sqrt(piv) : (state == 2 ? sqrt(1e-20 * wpp) : 0.0);
            if (lane == 0) {
                live[p] = state;
                R[p][p] = rpp;
                if (mode == 1) scale2[p] = state ? 1.0 / (rpp * rpp) : 1.0;
            }
            if (state == 1) {
                if (lane > p && lane < np) R[p][lane] = W[p][lane] / rpp;
                __syncwarp();
                // Schur complement of the trailing block: W[a][b] -= R[p][a] R[p][b] for p < a <= b < np (lane = b)
                if (lane > p && lane < np)
                    for (int aa = p + 1; aa <= lane; ++aa) W[aa][lane] -= R[p][aa] * R[p][lane];
            }
            __syncwarp();
        }
        // T = R^-1 over the kept columns: back substitution, one column per lane (rows of dropped / rescaled-only columns are zero)
        if (lane < np && live[lane]) {
            const int bb = lane;
            Ti[bb][bb] = 1.0 / R[bb][bb];
            for (int aa = bb - 1; aa >= 0; --aa) {
                if (live[aa] != 1) continue;
                double v = 0.0;
                for (int q = aa + 1; q <= bb; ++q) v -= R[aa][q] * Ti[q][bb];
                Ti[aa][bb] = v / R[aa][aa];
            }
        }
    }
    __syncthreads();
    if (tid < 256) T[t] = Ti[a][b];
}

// X[j0+p][i] <- sum_{q<=p} X[j0+q][i] T[q][p]
__global__ void __launch_bounds__(THREADS)
lr_panel_apply_kernel(double* __restrict__ X, long long m, long long ld, int j0, int np, const double* __restrict__ T) {
    __shared__ double st[LR_PANEL][LR_PANEL];
    for (int e = threadIdx.x; e < LR_PANEL * LR_PANEL; e += THREADS) st[e / LR_PANEL][e % LR_PANEL] = T[e];
    __syncthreads();
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        double x[LR_PANEL];
#pragma unroll
        for (int p = 0; p < LR_PANEL; ++p) x[p] = p < np ? X[(long long)(j0 + p) * ld + i] : 0.0;
#pragma unroll
        for (int p = 0; p < LR_PANEL; ++p) {
            if (p < np) {
                double v = 0.0;
#pragma unroll
                for (int q = 0; q <= p; ++q) v = fma(x[q], st[q][p], v);
                X[(long long)(j0 + p) * ld + i] = v;
            }
        }
    }
}

// ---- out[a][b] = sum_i wt_i A[a][i] Bm[b][i]   (a < na, b < nb; wt may be null) -------------------------------------------
// One CTA per {32 x 32 output tile, i-slice}; 2 x 2 outputs per thread; partial per slice, merged by lr_merge_kernel.
__global__ void __launch_bounds__(THREADS)
lr_inner_kernel(const double* __restrict__ A, int na, long long lda, const double* __restrict__ Bm, int nb, long long ldb,
                const double* __restrict__ wt, long long m,
                double* __restrict__ part /* [gridDim.y][na][nb] */) {
    // rows padded by 2 doubles: 16-byte aligned for the two-point LDS.128 of the inner loop, and the 16 rows a quarter-warp reads
    // in one step fall into distinct bank quads (row stride 132 words)
    __shared__ __align__(16) double sa[LR_TILE][LR_CHUNK + 2], sb[LR_TILE][LR_CHUNK + 2];
    const int tiles_b = (nb + LR_TILE - 1) / LR_TILE;
    const int ta0 = (blockIdx.x / tiles_b) * LR_TILE, tb0 = (blockIdx.x % tiles_b) * LR_TILE;
    const int slice = blockIdx.y, nsl = gridDim.y;
    const long long per = (m + nsl - 1) / nsl;
    const long long i_lo = (per * slice < m) ? per * slice : m, i_hi = (i_lo + per < m) ? i_lo + per : m;
    const int ty = threadIdx.x / 16, tx = threadIdx.x % 16;
    double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
    for (long long i0 = i_lo; i0 < i_hi; i0 += LR_CHUNK) {
        __syncthreads();
        for (int e = threadIdx.x; e < LR_TILE * LR_CHUNK; e += THREADS) {
            const int r = e / LR_CHUNK, ii = e % LR_CHUNK;
            const long long i = i0 + ii;
            const bool in = i < i_hi;
            const double w = in ? (wt ? wt[i] : 1.0) : 0.0;
            sa[r][ii] = (in && ta0 + r < na) ? w * A[(long long)(ta0 + r) * lda + i] : 0.0;
            sb[r][ii] = (in && tb0 + r < nb) ? Bm[(long long)(tb0 + r) * ldb + i] : 0.0;
        }
        __syncthreads();
        // two points per shared-memory load: 4 LDS.128 feed 8 DFMA (one LDS.64 per DFMA made the loop shared-memory bound)
#pragma unroll 8
        for (int ii = 0; ii < LR_CHUNK; ii += 2) {
            const double2 a0 = *reinterpret_cast<const double2*>(&sa[ty][ii]), a1 = *reinterpret_cast<const double2*>(&sa[ty + 16][ii]);
            const double2 b0 = *reinterpret_cast<const double2*>(&sb[tx][ii]), b1 = *reinterpret_cast<const double2*>(&sb[tx + 16][ii]);
            acc[0][0] = fma(a0.x, b0.x, acc[0][0]); acc[0][1] = fma(a0.x, b1.x, acc[0][1]);
            acc[1][0] = fma(a1.x, b0.x, acc[1][0]); acc[1][1] = fma(a1.x, b1.x, acc[1][1]);
            acc[0][0] = fma(a0.y, b0.y, acc[0][0]); acc[0][1] = fma(a0.y, b1.y, acc[0][1]);
            acc[1][0] = fma(a1.y, b0.y, acc[1][0]); acc[1][1] = fma(a1.y, b1.y, acc[1][1]);
        }
    }
    double* dst = part + (size_t)slice * na * nb;
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            const int a = ta0 + ty + 16 * u, b = tb0 + tx + 16 * v;
            if (a < na && b < nb) dst[(size_t)a * nb + b] = acc[u][v];
        }
}
// ---- the square, mathematically symmetric case  out = A diag(wt) Bm^T  (S = Q^T diag(w) Q of every M-step, Bc = Q^T (G Q)) --------
// One CTA per {64 x 64 tile of the LOWER triangle (ta >= tb), i-slice}; 4 x 4 outputs per thread: two points cost 8 LDS.128 for 32
// DFMA (12 shared-memory wavefronts against 16 cycles of the FP64 pipe per warp: FP64-bound, where the 2 x 2 tiles of
// lr_inner_kernel are shared-memory bound by 2x).  A thread owns the CONSECUTIVE rows 4 ty .. 4 ty + 3 (a warp: 8 rows), so in the
// last tile row -- the only one with padding, the lower triangle keeps the padded index on the row side -- whole warps have nothing
// to do and skip the arithmetic (n = 200: rows 192..199 of 256, one warp of eight); its columns are strided (tx + 16 v), which keeps
// the shared-memory reads conflict-free.  Partials per slice, joined by lr_merge_sym_kernel.
constexpr int LRS_TILE = 64, LRS_CHUNK = 32;
__global__ void __launch_bounds__(THREADS, 2)
lr_inner_sym_kernel(const double* __restrict__ A, int n, long long lda, const double* __restrict__ Bm, long long ldb,
                    const double* __restrict__ wt, long long m, double* __restrict__ part /* [gridDim.y][n][n], lower tiles only */) {
    __shared__ __align__(16) double sa[LRS_TILE][LRS_CHUNK + 2], sb[LRS_TILE][LRS_CHUNK + 2];   // row stride 68 words: see above
    int ta = 0, tb = (int)blockIdx.x;
    while (tb > ta) { tb -= ta + 1; ++ta; }            // blockIdx.x enumerates (0,0), (1,0), (1,1), (2,0), ...
    const int ta0 = ta * LRS_TILE, tb0 = tb * LRS_TILE;
    const int slice = blockIdx.y, nsl = gridDim.y;
    const long long per = (m + nsl - 1) / nsl;
    const long long i_lo = (per * slice < m) ? per * slice : m, i_hi = (i_lo + per < m) ? i_lo + per : m;
    const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
    const bool warp_has_rows = ta0 + (int)(threadIdx.x >> 5) * 8 < n;
    double acc[4][4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = 0.0;
    for (long long i0 = i_lo; i0 < i_hi; i0 += LRS_CHUNK) {
        __syncthreads();
        for (int e = threadIdx.x; e < LRS_TILE * LRS_CHUNK; e += THREADS) {
            const int r = e / LRS_CHUNK, ii = e % LRS_CHUNK;
            const long long i = i0 + ii;
            const bool in = i < i_hi;
            const double w = in ? (wt ? wt[i] : 1.0) : 0.0;
            sa[r][ii] = (in && ta0 + r < n) ? w * A[(long long)(ta0 + r) * lda + i] : 0.0;
            sb[r][ii] = (in && tb0 + r < n) ? Bm[(long long)(tb0 + r) * ldb + i] : 0.0;
        }
        __syncthreads();
        if (warp_has_rows) {
#pragma unroll 4
            for (int ii = 0; ii < LRS_CHUNK; ii += 2) {
                double2 a[4], b[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) a[u] = *reinterpret_cast<const double2*>(&sa[4 * ty + u][ii]);
#pragma unroll
                for (int v = 0; v < 4; ++v) b[v] = *reinterpret_cast<const double2*>(&sb[tx + 16 * v][ii]);
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u].x, b[v].x, acc[u][v]);
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int v = 0; v < 4; ++v) acc[u][v] = fma(a[u].y, b[v].y, acc[u][v]);
            }
        }
    }
    double* dst = part + (size_t)slice * n * n;
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int a = ta0 + 4 * ty + u, b = tb0 + tx + 16 * v;
            if (a < n && b < n) dst[(size_t)a * n + b] = acc[u][v];
        }
}
// out[a][b] (n x n, exactly symmetric) from the slice partials of lr_inner_sym_kernel: 8 lanes per output take the slices l, l + 8,
// ..., a fixed shuffle tree joins them; tiles above the diagonal are mirrored, diagonal tiles give (x + x^T) / 2.
__global__ void __launch_bounds__(THREADS)
lr_merge_sym_kernel(const double* __restrict__ part, int nsl, int n, double* __restrict__ out) {
    const int e = (blockIdx.x * THREADS + threadIdx.x) >> 3, l = threadIdx.x & 7;
    const bool in = e < n * n;
    const int a = in ? e / n : 0, b = in ? e % n : 0;
    const int ta = a / LRS_TILE, tb = b / LRS_TILE;
    const size_t e_ab = (size_t)a * n + b, e_ba = (size_t)b * n + a;
    double s = 0.0, t = 0.0;
    if (in) {
#pragma unroll 4
        for (int sl = l; sl < nsl; sl += 8) {
            const double* p = part + (size_t)sl * n * n;
            if (ta >= tb) s += p[e_ab];
            if (ta <= tb) t += p[e_ba];
        }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); t += __shfl_xor_sync(0xffffffffu, t, o); }
    if (in && l == 0) out[e] = ta == tb ? 0.5 * (s + t) : (ta > tb ? s : t);
}

// part[blk][a][d] = sum over the block's points of A[a][i] F[d][i]   for a narrow right factor (nd <= 4 rows, e.g. the three
// coordinates of F = px - diag(p1) Y): one warp per row a, lanes over the points -- lr_inner_kernel would pad the 3 columns to a
// 32-wide tile.  Merged by lr_merge_kernel like the other partials ([blk][na][nd]).
constexpr int LR_NARROW_PTS = 1024;
__global__ void __launch_bounds__(THREADS)
lr_inner_narrow_kernel(const double* __restrict__ A, int na, long long lda, const double* __restrict__ F, int nd, long long ldf, long long m,
                       double* __restrict__ part) {
    const int a = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (a >= na) return;
    const long long i_lo = (long long)blockIdx.y * LR_NARROW_PTS, i_hi = (i_lo + LR_NARROW_PTS < m) ? i_lo + LR_NARROW_PTS : m;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long i = i_lo + lane; i < i_hi; i += 32) {
        const double q = A[(long long)a * lda + i];
#pragma unroll
        for (int d = 0; d < 4; ++d)
            if (d < nd) acc[d] = fma(q, F[(long long)d * ldf + i], acc[d]);
    }
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        const double v = warp_sum(acc[d]);
        if (lane == 0 && d < nd) part[((size_t)blockIdx.y * na + a) * nd + d] = v;
    }
}

// out[e] = sum_slices part[s][e]  (fixed order: 8 lanes per output take the slices l, l + 8, ..., then a fixed shuffle tree joins
// them).  The symmetric products have their own pair (lr_inner_sym_kernel / lr_merge_sym_kernel).
__global__ void __launch_bounds__(THREADS)
lr_merge_kernel(const double* __restrict__ part, int nsl, int na, int nb, double* __restrict__ out) {
    const int e = (blockIdx.x * THREADS + threadIdx.x) >> 3, l = threadIdx.x & 7;
    const bool in = e < na * nb;
    double s = 0.0;
    if (in) {
#pragma unroll 4
        for (int sl = l; sl < nsl; sl += 8) s += part[(size_t)sl * na * nb + e];
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (in && l == 0) out[e] = s;
}

// ---- the K x K system of one M-step:  Msys = c I + Bc S  (row-major),  rhs[d][a] = sum_k Bc[a][k] R[k][d],  c = lmd sigma2 ----
__global__ void __launch_bounds__(THREADS)
lr_system_kernel(const double* __restrict__ Bc, const double* __restrict__ S, const double* __restrict__ R /* [K][3] */, int rank,
                 const double* __restrict__ sigma2_ptr, double lmd, double* __restrict__ Msys, double* __restrict__ rhs /* [3][K] */,
                 double* __restrict__ c_out) {
    const int e = blockIdx.x * THREADS + threadIdx.x;
    const double c = lmd * *sigma2_ptr;
    if (e == 0) *c_out = c;
    if (e < rank * rank) {
        const int a = e / rank, b = e % rank;
        double s = (a == b) ? c : 0.0;
        for (int k = 0; k < rank; ++k) s += Bc[(size_t)a * rank + k] * S[(size_t)k * rank + b];
        Msys[e] = s;
    } else if (e < rank * rank + 3 * rank) {
        const int f = e - rank * rank, d = f / rank, a = f % rank;
        double s = 0.0;
        for (int k = 0; k < rank; ++k) s += Bc[(size_t)a * rank + k] * R[(size_t)k * 3 + d];
        rhs[f] = s;
    }
}

// ---- symmetric form of the K x K system: G ~= Q Bc Q^T = Qt Qt^T with Qt = Q L, Bc ~= L L^T (pivoted Cholesky, once, at set-up) -----
// With the (non-orthonormal) factor Qt the Woodbury system of an M-step is symmetric positive definite,
//     (c I + St) Z = Rt,      St = Qt^T diag(p1) Qt,  Rt = Qt^T F,      W = (F - diag(p1) Qt Z) / c,   T = Y + Qt Z,
// against the unsymmetric (c I + Bc S) Z = Bc R of the orthonormal factor.  lr_spd_solve_kernel solves it in ONE CTA: the lower
// triangle of  c I + St  with the three right-hand sides appended as rows K .. K+2 lives in shared memory (packed by rows,
// (K+3)(K+4)/2 doubles: 166 KB at K = 200, plus the panel buffer), a blocked LDL^T factorisation runs over it (see the kernel) -- the
// appended rows come out as the forward substitution -- then the back substitution in registers.  It replaces cuSOLVER's LU of
// the unsymmetric form (getrf is a single 256-thread CTA there, plus laswp and two trsm), which stays selectable with
// CPD_B200_LR_CORE=lu.  (An eigen-decomposition of Bc would serve as well as the Cholesky factor; cusolverDnXsyevd's first call
// in a process is costly, so the factor is computed here.)
constexpr int LR_SPD_THREADS = 512;           // 128 registers per thread: phase 1 keeps an 8 x 8 block in registers
constexpr int LR_SPD_B = 8;                  // columns per panel: two barriers per LR_SPD_B columns
constexpr int LR_SPD_RG = 4;                 // rows per warp pass in the trailing update
constexpr int LR_SPD_MAX_RANK = 228;         // (K+3)(K+4)/2 + LR_SPD_B (K+3) + K doubles <= 227 KB
__host__ __device__ constexpr size_t lr_spd_smem_bytes(int k) {
    return ((size_t)(k + 3) * (k + 4) / 2 + (size_t)LR_SPD_B * (k + 3) + (size_t)k) * sizeof(double);
}
// Blocked LDL^T (no pivoting: the matrix is c I + a positive semi-definite one).  "Unscaled" storage throughout: below the diagonal
// a'_ik = l_ik d_k, on it d_k.  Per panel of LR_SPD_B columns at j0:
//   phase 1, one THREAD per row i >= j0: factor the LR_SPD_B x LR_SPD_B diagonal block (every thread for itself: 36 broadcast loads,
//            ~90 FMAs -- cheaper than a barrier) and run the row through it:  p_c = a_{i,j0+c} - sum_{c'<c} p_c' l_{c c'};  p goes
//            back into the triangle and into the panel buffer (rows >= j0 + B: that is all they ever need from this panel);
//   phase 2, one WARP per row i >= j0 + B, lanes over k:  a_ik -= sum_c p_ic p_kc / d_c  -- LR_SPD_B FMAs per load/store pair.
// The right-hand sides ride along as rows K .. K+2 (phase 2 leaves them as the forward substitution).  Then L = a' / d in place and
// one warp per right-hand side does the back substitution in registers (lane-owned entries, shuffles; no barrier).
__global__ void __launch_bounds__(LR_SPD_THREADS, 1)
lr_spd_solve_kernel(const double* __restrict__ S, const double* __restrict__ R /* [K][3] */, int K, const double* __restrict__ sigma2_ptr,
                    double lmd, double* __restrict__ Zt /* [3][K] */, double* __restrict__ c_out) {
    CPD_DYN_SMEM(smraw);
    constexpr int B = LR_SPD_B, NW = LR_SPD_THREADS / 32;
    double* const tri = reinterpret_cast<double*>(smraw);               // row i at i (i + 1) / 2, entries k <= i
    const int rows = K + 3;
    double* const pan = tri + (size_t)rows * (rows + 1) / 2;            // [B][rows]: the current panel, rows relative to j0 (column-major:
                                                                        // consecutive rows in consecutive banks)
    double* const dinv = pan + (size_t)B * rows;                        // [K]: 1 / d_k
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const double c = lmd * *sigma2_ptr;
    if (tid == 0) *c_out = c;
    for (int i = warp; i < rows; i += NW) {
        double* row = tri + (size_t)i * (i + 1) / 2;
        if (i < K) for (int k = lane; k <= i; k += 32) row[k] = S[(size_t)i * K + k] + (i == k ? c : 0.0);
        else for (int k = lane; k < K; k += 32) row[k] = R[(size_t)k * 3 + (i - K)];
    }
    __syncthreads();
    for (int j0 = 0; j0 < K; j0 += B) {
        const int nb = (K - j0 < B) ? K - j0 : B;
        // phase 1
        if (tid < rows - j0) {
            const int i = j0 + tid;
            double blk[B][B], rd[B], pv[B];
#pragma unroll
            for (int a = 0; a < B; ++a)
#pragma unroll
                for (int b2 = 0; b2 <= a; ++b2) blk[a][b2] = (a < nb) ? tri[(size_t)(j0 + a) * (j0 + a + 1) / 2 + j0 + b2] : (a == b2 ? 1.0 : 0.0);
#pragma unroll
            for (int cc = 0; cc < B; ++cc) {
                const double dc = blk[cc][cc];
                rd[cc] = 1.0 / (dc > 0.0 ? dc : c);            // d >= c in exact arithmetic
#pragma unroll
                for (int a = cc + 1; a < B; ++a) {
                    const double f = blk[a][cc] * rd[cc];
#pragma unroll
                    for (int b2 = cc + 1; b2 <= a; ++b2) blk[a][b2] -= f * blk[b2][cc];
                }
            }
            double* row = tri + (size_t)i * (i + 1) / 2;
            const int have = (tid < nb) ? tid + 1 : nb;        // rows inside the block own the columns up to their diagonal
#pragma unroll
            for (int cc = 0; cc < B; ++cc) {
                double v = 0.0;
                if (cc < have) {
                    v = row[j0 + cc];
#pragma unroll
                    for (int c2 = 0; c2 < cc; ++c2) v -= pv[c2] * (blk[cc][c2] * rd[c2]);
                    if (tid >= nb) row[j0 + cc] = v;          // the block's own rows are being read by everybody: written after the barrier
                }
                pv[cc] = v;
                pan[(size_t)cc * rows + tid] = v;
            }
            if (tid == 0)
#pragma unroll
                for (int cc = 0; cc < B; ++cc) if (cc < nb) dinv[j0 + cc] = rd[cc];
        }
        __syncthreads();
        if (tid < nb) {
            double* row = tri + (size_t)(j0 + tid) * (j0 + tid + 1) / 2;
            for (int cc = 0; cc <= tid; ++cc) row[j0 + cc] = pan[(size_t)cc * rows + tid];
        }
        // phase 2: rows beyond the panel, columns beyond the panel; a warp takes LR_SPD_RG consecutive rows at a time and reuses the
        // eight panel entries of its lanes' columns for all of them (shared-memory wavefronts per FMA: 20 / 8 -> 8 / 8)
        const int k0 = j0 + nb;
        for (int i0 = k0 + LR_SPD_RG * warp; i0 < rows; i0 += LR_SPD_RG * NW) {
            double pi[LR_SPD_RG][B];
            double* row[LR_SPD_RG];
            int kend[LR_SPD_RG];
#pragma unroll
            for (int q = 0; q < LR_SPD_RG; ++q) {
                const int i = i0 + q;
                const bool live = i < rows;
                row[q] = tri + (size_t)(live ? i : i0) * ((live ? i : i0) + 1) / 2;
                kend[q] = live ? (i < K ? i : K - 1) : -1;
#pragma unroll
                for (int cc = 0; cc < B; ++cc) pi[q][cc] = (live && cc < nb) ? pan[(size_t)cc * rows + (i - j0)] * dinv[j0 + cc] : 0.0;
            }
            const int kmax = kend[LR_SPD_RG - 1] >= 0 ? kend[LR_SPD_RG - 1] : (i0 + LR_SPD_RG - 1 < K ? i0 + LR_SPD_RG - 1 : K - 1);
            for (int k = k0 + lane; k <= kmax; k += 32) {
                double pk[B];
#pragma unroll
                for (int cc = 0; cc < B; ++cc) pk[cc] = pan[(size_t)cc * rows + (k - j0)];
#pragma unroll
                for (int q = 0; q < LR_SPD_RG; ++q) {
                    if (k <= kend[q]) {
                        double v = row[q][k];
#pragma unroll
                        for (int cc = 0; cc < B; ++cc) v = fma(-pi[q][cc], pk[cc], v);
                        row[q][k] = v;
                    }
                }
            }
        }
        __syncthreads();
    }
    // L = a' / d in place (strictly lower part of rows < K); the right-hand-side rows become y0 = D^-1 L^-1 b
    for (int i = 1 + warp; i < rows; i += NW) {
        double* row = tri + (size_t)i * (i + 1) / 2;
        const int kend = i < K ? i - 1 : K - 1;
        for (int k = lane; k <= kend; k += 32) row[k] *= dinv[k];
    }
    __syncthreads();
    // back substitution  L^T x = y0: warp d owns right-hand side d; lane l holds the entries 32 t + l
    if (warp < 3) {
        constexpr int T = (LR_SPD_MAX_RANK + 31) / 32;
        const double* rhs = tri + (size_t)(K + warp) * (K + warp + 1) / 2;
        double y[T];
#pragma unroll
        for (int t = 0; t < T; ++t) y[t] = (32 * t + lane < K) ? rhs[32 * t + lane] : 0.0;
#pragma unroll
        for (int t = T - 1; t >= 0; --t) {
#pragma unroll 1
            for (int l = 31; l >= 0; --l) {
                const int j = 32 * t + l;
                if (j >= K) continue;
                const double xj = __shfl_sync(0xffffffffu, y[t], l);
                const double* rowj = tri + (size_t)j * (j + 1) / 2;
#pragma unroll
                for (int tt = 0; tt <= t; ++tt) {
                    const int i = 32 * tt + lane;
                    if (i < j) y[tt] = fma(-rowj[i], xj, y[tt]);
                }
            }
        }
#pragma unroll
        for (int t = 0; t < T; ++t)
            if (32 * t + lane < K) Zt[(size_t)warp * K + 32 * t + lane] = y[t];
    }
}

// Pivoted (diagonal pivoting) Cholesky of the symmetric positive semi-definite core, left-looking, ONE CTA:  Bc ~= L L^T with
//   Lt[j][i] = L_ij  (row j of Lt = column j of L, in the ORIGINAL row order: nothing is permuted, the pivot order is implicit).
// Step j: p = argmax of the remaining diagonal d; stop when d_p <= 1e-14 of the largest diagonal entry of Bc (what is left is
// rounding -- or the float32 noise of the G X products once K reaches into it, where the remaining Schur complement is indefinite:
// a positive semi-definite G has no use for it); L_:j = (Bc_:p - sum_{t<j} L_:t L_pt) / sqrt(d_p); d -= L_:j^2.  A dropped column of
// Q (zero row and column of Bc) has d = 0 and is never picked.  Columns from the stopping point on are zero.
constexpr int LR_PCHOL_THREADS = 1024;
__global__ void __launch_bounds__(LR_PCHOL_THREADS, 1)
lr_pchol_kernel(const double* __restrict__ Bc, int K, double* __restrict__ Lt /* [K][K] */, int* __restrict__ rank_out) {
    __shared__ double d[LR_MAX_RANK], lp[LR_MAX_RANK];      // remaining diagonal; row p of L (columns < j)
    __shared__ double wv[LR_PCHOL_THREADS / 32];
    __shared__ int wi[LR_PCHOL_THREADS / 32];
    __shared__ int piv;
    __shared__ double dpiv, dmax0;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < K; i += LR_PCHOL_THREADS) d[i] = Bc[(size_t)i * K + i];
    for (int e = tid; e < K * K; e += LR_PCHOL_THREADS) Lt[e] = 0.0;
    __syncthreads();
    int rank = 0;
    for (int j = 0; j < K; ++j) {
        // argmax of d (ties: the smaller index), two-level
        double bv = -1.0;
        int bi = 0x7fffffff;
        for (int i = tid; i < K; i += LR_PCHOL_THREADS)
            if (d[i] > bv || (d[i] == bv && i < bi)) { bv = d[i]; bi = i; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if (lane == 0) { wv[warp] = bv; wi[warp] = bi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < LR_PCHOL_THREADS / 32; ++w)
                if (wv[w] > bv || (wv[w] == bv && wi[w] < bi)) { bv = wv[w]; bi = wi[w]; }
            piv = bi; dpiv = bv;
            if (j == 0) dmax0 = bv;
        }
        __syncthreads();
        const int p = piv;
        const double dp = dpiv;
        if (!(dp > 1e-14 * dmax0) || !(dp > 0.0)) break;          // uniform: every thread reads the same shared values
        for (int t = tid; t < j; t += LR_PCHOL_THREADS) lp[t] = Lt[(size_t)t * K + p];
        __syncthreads();
        const double rs = 1.0 / sqrt(dp);
        // one warp per row i: dot product over the finished columns, lanes over t
        for (int i = warp; i < K; i += LR_PCHOL_THREADS / 32) {
            double s = 0.0;
            for (int t = lane; t < j; t += 32) s = fma(Lt[(size_t)t * K + i], lp[t], s);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) {
                // rows already used as pivots have d = 0 by construction (their residual is what rounding left): keep them at zero
                const double l = (d[i] > 0.0 || i == p) ? (Bc[(size_t)i * K + p] - s) * rs : 0.0;
                Lt[(size_t)j * K + i] = l;
                const double dn = d[i] - l * l;
                d[i] = (i == p) ? 0.0 : (dn > 0.0 ? dn : 0.0);
            }
        }
        rank = j + 1;
        __syncthreads();
    }
    if (tid == 0) *rank_out = rank;
}
// Bc <- L L^T: the core that the symmetric form really uses (Bc minus what the pivoted Cholesky left out: rounding, or the indefinite
// float32 noise of the G X products) -- it is what cpd_nonrigid_lowrank_get hands out, so G ~= Q Bc Q^T stays exactly the iteration's G.
__global__ void __launch_bounds__(THREADS)
lr_llt_kernel(const double* __restrict__ Lt, int K, double* __restrict__ Bc) {
    const int e = blockIdx.x * THREADS + threadIdx.x;
    if (e < K * K) {
        const int a = e / K, b = e % K;
        const int lo = a < b ? a : b, hi = a < b ? b : a;        // one summation per unordered pair: exactly symmetric
        double s = 0.0;
        for (int j = 0; j < K; ++j) s = fma(Lt[(size_t)j * K + lo], Lt[(size_t)j * K + hi], s);
        Bc[e] = s;
    }
}
// out[j0 + p][i] = sum_k V[j0 + p][k] Q[k][i]: the columns of Qt = Q L, LR_PANEL at a time (V = Lt of lr_pchol_kernel)
__global__ void __launch_bounds__(THREADS)
lr_rotate_kernel(const double* __restrict__ Q, long long m, long long ld, int K, const double* __restrict__ V, int j0, int np,
                 double* __restrict__ out) {
    __shared__ double sc[LR_UPD_KC][LR_PANEL];
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double acc[LR_PANEL];
#pragma unroll
    for (int p = 0; p < LR_PANEL; ++p) acc[p] = 0.0;
    for (int k0 = 0; k0 < K; k0 += LR_UPD_KC) {
        const int kc = (K - k0 < LR_UPD_KC) ? K - k0 : LR_UPD_KC;
        __syncthreads();
        for (int e = threadIdx.x; e < kc * LR_PANEL; e += THREADS) {
            const int k = e % kc, pp = e / kc;
            sc[k][pp] = pp < np ? V[(size_t)(j0 + pp) * K + k0 + k] : 0.0;
        }
        __syncthreads();
        if (i < m) {
#pragma unroll 8
            for (int k = 0; k < kc; ++k) {
                const double q = Q[(long long)(k0 + k) * ld + i];
#pragma unroll
                for (int p = 0; p < LR_PANEL; ++p) acc[p] = fma(q, sc[k][p], acc[p]);
            }
        }
    }
    if (i < m)
        for (int p = 0; p < np; ++p) out[(long long)(j0 + p) * ld + i] = acc[p];
}

// T_i = y_i + sum_k Q[k][i] Z[k]   (Z arrives as the solution layout of the LU solve: Zt[d][k])
__global__ void __launch_bounds__(THREADS)
lr_apply_kernel(const double* __restrict__ Q, long long m, long long ld, int rank, const double* __restrict__ Zt, const double* __restrict__ yc,
                double c0, double c1, double c2, double* __restrict__ ts) {
    __shared__ double sz[3][LR_MAX_RANK];
    for (int e = threadIdx.x; e < 3 * rank; e += THREADS) sz[e / rank][e % rank] = Zt[e];
    __syncthreads();
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        for (int k = 0; k < rank; ++k) {
            const double q = Q[(long long)k * ld + i];
            a0 += q * sz[0][k]; a1 += q * sz[1][k]; a2 += q * sz[2][k];
        }
        ts[3 * i] = yc[3 * i] + c0 + a0;
        ts[3 * i + 1] = yc[3 * i + 1] + c1 + a1;
        ts[3 * i + 2] = yc[3 * i + 2] + c2 + a2;
    }
}

// W_i = (F_i - p1_i (T_i - y_i)) / c      [T - Y = Q Z]      F arrives as [3][m] (nr_rhs_kernel)
__global__ void __launch_bounds__(THREADS)
lr_w_kernel(const double* __restrict__ F, const double* __restrict__ p1, const double* __restrict__ ts, const double* __restrict__ yc,
            double c0, double c1, double c2, long long m, const double* __restrict__ c_ptr, double* __restrict__ W) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const double inv = 1.0 / *c_ptr, cc[3] = {c0, c1, c2};
#pragma unroll
        for (int d = 0; d < 3; ++d) W[3 * i + d] = (F[(long long)d * m + i] - p1[i] * (ts[3 * i + d] - yc[3 * i + d] - cc[d])) * inv;
    }
}

// out[perm[i]][k] = Q[k][i]: the basis in the caller's point order, row-major M x K
__global__ void __launch_bounds__(THREADS)
lr_export_kernel(const double* __restrict__ Q, const int* __restrict__ perm, long long m, long long ld, int rank, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const long long r = perm[i];
        for (int k = 0; k < rank; ++k) out[r * rank + k] = Q[(long long)k * ld + i];
    }
}
// X[k][i] = in[perm[i]][k]: the inverse of lr_export_kernel (a row-major M x K block in the caller's order -> [K][ld], internal order)
__global__ void __launch_bounds__(THREADS)
lr_import_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long m, long long ld, int rank, double* __restrict__ X) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const long long r = perm[i];
        for (int k = 0; k < rank; ++k) X[(long long)k * ld + i] = in[r * rank + k];
    }
}

}  // namespace cpd
