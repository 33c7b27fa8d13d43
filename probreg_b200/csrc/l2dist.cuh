// l2dist.cuh -- GMMReg (Jian & Vemuri, PAMI 2011; probreg/l2dist_regs.py, cost_functions.py, features.py) on sm_90a: the spherical
// Gaussian-mixture fit that summarises each cloud (sklearn's GaussianMixture(covariance_type="spherical")), the L2 distance between
// two mixtures with its gradient, and the float32 thin-plate-spline kernel matrix.  FP64 throughout (except the TPS matrix, float32
// like the reference), every reduction in a fixed order (no atomics), so two runs on one device are bit-identical.  Host
// orchestration: host_l2dist.inl.
//
// The EM iteration of the fit is one pass over the points (gm_estep_kernel): a CTA owns GM_CHUNK points, phase 1 gives every point
// its log-sum-exp over the K components (the components' constants tiled through shared memory), phase 2 gives every component
// (one thread each) its sums of r {1, x - mu, |x - mu|^2} over the chunk's points, read from shared memory, with the
// responsibilities r = exp(log p - lse) recomputed.  The chunk partials are joined in chunk order (gm_merge_kernel) and one CTA
// forms the M-step and the next iteration's constants (gm_mstep_kernel).
#pragma once
#include "kernels.cuh"

namespace cpd {

constexpr int GM_CHUNK = 512;            // points per CTA of the E-step (two per thread)
constexpr int GM_TILE = 128;             // components per shared-memory tile of phase 1
constexpr int GM_C = 5;                  // per component: {mu (3, centred frame), 1 / (2 var), log w - D/2 log(2 pi var)}
constexpr int GM_S = 5;                  // per component: {sum r, sum r (x - mu) (3), sum r |x - mu|^2}
constexpr int GM_P = 5;                  // per component: {mu (3, caller frame), var, w}
constexpr double GM_LOG_2PI = 1.8378770664093453;
constexpr double GM_NK_EPS = 10.0 * 2.220446049250313e-16;   // sklearn's nk = resp.sum(0) + 10 * eps (_gaussian_mixture.py)

constexpr int L2_SRC = 64;               // sources per CTA of the L2 distance, one per thread
constexpr int L2_TILE = 64;              // targets per shared-memory tile
constexpr int L2_CTAS = 2112;            // CTAs the source x target-chunk grid aims at (16 per SM of a 132-SM H100)

// ---- the spherical GMM fit ------------------------------------------------------------------------------------------------------
// The M-step of component j from its sums S (anchored at a = the mean the E-step used, centred frame) and the next E-step's
// constants; init: one-hot responsibilities at the seed point (S = {1, 0, 0}, a = the seed).  In the caller's frame
// (ac = a + origin), exactly sklearn's _estimate_gaussian_parameters with nk = S0 + 10 eps:
//   mu  = (S1 + ac S0) / nk                                  (= sum r x / nk)
//   var = (S2 / nk - |mu - ac|^2 + 10 eps |ac|^2 / nk) / D + reg   (= (sum r |x|^2 / nk - |mu|^2) / D + reg, without its cancellation)
// The last term is the shrink of nk's 10 eps towards the caller's origin; it matters only for components that hold no points.
__device__ __forceinline__ void gm_component(const double (&S)[GM_S], const double (&a)[3], const double (&org)[3], int dim,
                                             double reg, double (&mu)[3], double& var, double& nk) {
    nk = S[0] + GM_NK_EPS;
    double d2 = 0.0, a2 = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double ac = a[c] + org[c];
        mu[c] = (S[1 + c] + ac * S[0]) / nk;
        const double dl = mu[c] - ac;
        d2 += dl * dl;
        a2 += ac * ac;
    }
    var = (S[4] / nk - d2 + GM_NK_EPS * a2 / nk) / (double)dim + reg;
}

// M-step of every component (one CTA): sums (K x GM_S) and the old constants -> parameters (K x GM_P, caller frame) and the new
// constants.  init != 0: the initialisation from the seed points (pts: centred, internal order; inv: caller -> internal index),
// weights nk / n (unnormalised, as sklearn's _initialize leaves them); else weights nk / sum nk.  lb_sum: the E-step's sum of the
// per-point lse, written as lb_sum / n to out_lb.
__global__ void __launch_bounds__(THREADS)
gm_mstep_kernel(int init, const double* __restrict__ pts, const int* __restrict__ inv, const long long* __restrict__ seeds,
                const double* __restrict__ sums, int K, long long n, int dim, double reg, double o0, double o1, double o2,
                double* __restrict__ cst, double* __restrict__ par, double* __restrict__ scr, const double* __restrict__ lb_sum,
                double* __restrict__ out_lb) {
    const double org[3] = {o0, o1, o2};
    double tot[1] = {0.0};
    for (int j = threadIdx.x; j < K; j += THREADS) {
        double S[GM_S] = {1.0, 0.0, 0.0, 0.0, 0.0}, a[3], mu[3], var, nk;
        if (init) {
            const double* y = pts + 3 * (size_t)inv[seeds[j]];
            a[0] = y[0]; a[1] = y[1]; a[2] = y[2];
        } else {
#pragma unroll
            for (int t = 0; t < GM_S; ++t) S[t] = sums[(size_t)j * GM_S + t];
            a[0] = cst[(size_t)j * GM_C]; a[1] = cst[(size_t)j * GM_C + 1]; a[2] = cst[(size_t)j * GM_C + 2];
        }
        gm_component(S, a, org, dim, reg, mu, var, nk);
        double* p = par + (size_t)j * GM_P;
        p[0] = mu[0]; p[1] = mu[1]; p[2] = mu[2]; p[3] = var; p[4] = nk;
        tot[0] += nk;
    }
    block_reduce_store<1>(tot, scr);
    __syncthreads();                                    // scr[0] (global, written by thread 0) is visible to the block
    const double den = init ? (double)n : scr[0];
    for (int j = threadIdx.x; j < K; j += THREADS) {
        double* p = par + (size_t)j * GM_P;
        double* c = cst + (size_t)j * GM_C;
        const double w = p[4] / den, var = p[3];
        p[4] = w;
        c[0] = p[0] - o0; c[1] = p[1] - o1; c[2] = p[2] - o2;
        c[3] = 0.5 / var;
        c[4] = log(w) - 0.5 * (double)dim * (GM_LOG_2PI + log(var));
    }
    if (threadIdx.x == 0 && out_lb) *out_lb = *lb_sum / (double)n;
}

// log p of a point against a prepared component: log w - D/2 log(2 pi var) - |x - mu|^2 / (2 var)
__device__ __forceinline__ double gm_logp(const double* __restrict__ c, double x0, double x1, double x2) {
    const double d0 = x0 - c[0], d1 = x1 - c[1], d2 = x2 - c[2];
    return c[4] - c[3] * (d0 * d0 + d1 * d1 + d2 * d2);
}

// One EM E-step over a chunk of GM_CHUNK points (centred, internal order).  part: [K][nch][GM_S] component sums of this chunk;
// lbp[chunk]: the chunk's sum of the per-point lse.
__global__ void __launch_bounds__(THREADS, 1)
gm_estep_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ cst, int K, long long nch,
                double* __restrict__ part, double* __restrict__ lbp) {
    __shared__ double sp[GM_CHUNK][4];                 // x, y, z, lse
    __shared__ double tile[GM_TILE * GM_C];
    const long long c0 = (long long)blockIdx.x * GM_CHUNK;
    const int np = (int)min((long long)GM_CHUNK, n - c0);
    // phase 1: thread t owns points t and t + THREADS of the chunk; online log-sum-exp over the components in index order
    double x[2][3], mx[2], s[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int k = threadIdx.x + r * THREADS;
        const long long i = c0 + min(k, np - 1);      // threads past the end repeat the last point and store nothing
        x[r][0] = pts[3 * i]; x[r][1] = pts[3 * i + 1]; x[r][2] = pts[3 * i + 2];
        mx[r] = -INFINITY;
        s[r] = 0.0;
    }
    for (int t0 = 0; t0 < K; t0 += GM_TILE) {
        const int nt = min(GM_TILE, K - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < nt * GM_C; e += THREADS) tile[e] = cst[(size_t)t0 * GM_C + e];
        __syncthreads();
        for (int j = 0; j < nt; ++j) {
            const double* c = tile + j * GM_C;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const double lp = gm_logp(c, x[r][0], x[r][1], x[r][2]);
                const double e = exp(-fabs(lp - mx[r]));       // one exp per pair: rescale the sum or add the term
                const bool up = lp > mx[r];
                s[r] = up ? s[r] * e + 1.0 : s[r] + e;
                mx[r] = up ? lp : mx[r];
            }
        }
    }
    double lsum[1] = {0.0};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int k = threadIdx.x + r * THREADS;
        if (k < np) {
            const double lse = mx[r] + log(s[r]);
            sp[k][0] = x[r][0]; sp[k][1] = x[r][1]; sp[k][2] = x[r][2]; sp[k][3] = lse;
            lsum[0] += lse;
        }
    }
    block_reduce_store<1>(lsum, lbp + blockIdx.x);     // its __syncthreads also publishes sp
    // phase 2: thread t owns components t, t + THREADS, ...; the chunk's points in order
    for (int j = threadIdx.x; j < K; j += THREADS) {
        double c[GM_C];
#pragma unroll
        for (int t = 0; t < GM_C; ++t) c[t] = cst[(size_t)j * GM_C + t];
        double S[GM_S] = {0.0, 0.0, 0.0, 0.0, 0.0};
        for (int k = 0; k < np; ++k) {
            const double d0 = sp[k][0] - c[0], d1 = sp[k][1] - c[1], d2 = sp[k][2] - c[2];
            const double q = d0 * d0 + d1 * d1 + d2 * d2;
            const double r = exp(c[4] - c[3] * q - sp[k][3]);
            S[0] += r; S[1] += r * d0; S[2] += r * d1; S[3] += r * d2; S[4] += r * q;
        }
        double* o = part + ((size_t)j * nch + blockIdx.x) * GM_S;
#pragma unroll
        for (int t = 0; t < GM_S; ++t) o[t] = S[t];
    }
}

// component j = blockIdx.x: its chunk partials joined in a fixed order (thread t takes chunks t, t + THREADS, ..., then the block
// tree) into sums[j]
__global__ void __launch_bounds__(THREADS)
gm_merge_kernel(const double* __restrict__ part, long long nch, double* __restrict__ sums) {
    const long long j = blockIdx.x;
    double v[GM_S] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (long long ch = threadIdx.x; ch < nch; ch += THREADS) {
        const double* p = part + ((size_t)j * nch + ch) * GM_S;
#pragma unroll
        for (int t = 0; t < GM_S; ++t) v[t] += p[t];
    }
    block_reduce_store<GM_S>(v, sums + (size_t)j * GM_S);
}

// ---- the L2 distance between two mixtures ---------------------------------------------------------------------------------------
// For source i (one per thread) and the target chunk blockIdx.y: S0 = sum_j w_j e_ij and S1 = sum_j w_j e_ij (mu_s,i - mu_t,j),
// e_ij = exp(-|mu_s,i - mu_t,j|^2 * inv2s2), the targets {mu (3), w = phi / z} tiled through shared memory.  part: [chunk][ns][4].
__global__ void __launch_bounds__(L2_SRC)
l2_pair_kernel(const double* __restrict__ src, long long ns, const double* __restrict__ tgt /* [nt][4] */, long long nt, long long tc,
               double inv2s2, double* __restrict__ part) {
    __shared__ double tile[L2_TILE * 4];
    const long long i = (long long)blockIdx.x * L2_SRC + threadIdx.x;
    const long long ii = min(i, ns - 1);
    const double x0 = src[3 * ii], x1 = src[3 * ii + 1], x2 = src[3 * ii + 2];
    const long long j0 = (long long)blockIdx.y * tc, j1 = min(nt, j0 + tc);
    double S[4] = {0.0, 0.0, 0.0, 0.0};
    for (long long t0 = j0; t0 < j1; t0 += L2_TILE) {
        const int cnt = (int)min((long long)L2_TILE, j1 - t0);
        __syncthreads();
        for (int e = threadIdx.x; e < cnt * 4; e += L2_SRC) tile[e] = tgt[(size_t)t0 * 4 + e];
        __syncthreads();
        for (int j = 0; j < cnt; ++j) {
            const double* p = tile + 4 * j;
            const double d0 = x0 - p[0], d1 = x1 - p[1], d2 = x2 - p[2];
            const double we = p[3] * exp(-(d0 * d0 + d1 * d1 + d2 * d2) * inv2s2);
            S[0] += we; S[1] += we * d0; S[2] += we * d1; S[3] += we * d2;
        }
    }
    if (i < ns) {
        double* o = part + ((size_t)blockIdx.y * ns + i) * 4;
        o[0] = S[0]; o[1] = S[1]; o[2] = S[2]; o[3] = S[3];
    }
}

// per source: the chunk partials joined in chunk order; g_i = phi_s,i S1 / (2 sigma^2) (dim columns), and the block partial of
// sum_i phi_s,i S0 to fpart[blockIdx.x]
__global__ void __launch_bounds__(THREADS)
l2_merge_kernel(const double* __restrict__ part, long long ns, int nchunk, const double* __restrict__ phi_s, int dim, double inv2s2,
                double* __restrict__ g, double* __restrict__ fpart) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[1] = {0.0};
    if (i < ns) {
        double S[4] = {0.0, 0.0, 0.0, 0.0};
        for (int c = 0; c < nchunk; ++c) {
            const double* p = part + ((size_t)c * ns + i) * 4;
            S[0] += p[0]; S[1] += p[1]; S[2] += p[2]; S[3] += p[3];
        }
        const double ph = phi_s[i];
#pragma unroll
        for (int a = 0; a < 3; ++a)
            if (a < dim) g[(size_t)i * dim + a] = ph * S[1 + a] * inv2s2;
        v[0] = ph * S[0];
    }
    block_reduce_store<1>(v, fpart + blockIdx.x);
}

// ---- _math.tps_kernel_2d / _3d (cc/math_utils.cc:21-30), float32 -----------------------------------------------------------------
// every float operation rounded on its own (no FMA contraction); 2-D: r^2 log r with the log taken in FP64 of the float32 r and
// rounded once (the same on every host), 0 where r^2 <= 1e-9; 3-D: -r
__global__ void __launch_bounds__(THREADS)
tps_kernel_kernel(const float* __restrict__ x, long long nx, const float* __restrict__ y, long long ny, int dim, float* __restrict__ out) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;
    const long long i = blockIdx.x;
    if (j < ny) {
        float d2 = 0.f;
        for (int a = 0; a < dim; ++a) { const float d = __fsub_rn(x[i * dim + a], y[j * dim + a]); d2 = __fadd_rn(d2, __fmul_rn(d, d)); }
        const float r = __fsqrt_rn(d2);
        float v;
        if (dim == 2) v = d2 > 1.0e-9f ? __fmul_rn(d2, (float)log((double)r)) : 0.0f;
        else v = -r;
        out[i * ny + j] = v;
    }
}

}  // namespace cpd
