// ocsvm.cuh -- the one-class SVM fit behind probreg's SVR features (features.OneClassSVM: sklearn's OneClassSVM(kernel="rbf").fit)
// on sm_90a.  libsvm's SMO with second-order working-set selection (Fan, Chen & Lin, JMLR 2005), without shrinking, on the
// caller's raw coordinates in the caller's order: the same path as sklearn, so the same support vectors and weights.  FP64
// except the kernel values, which are rounded to float32 as libsvm's Qfloat column cache does; no atomics; every reduction in a
// fixed order (the selections are lexicographic maxima, which no order changes), so two runs on one device are bit-identical.
// Host orchestration: host_ocsvm.inl.
//
// One SMO iteration is two launches over OCS_THREADS-thread CTAs, each owning a contiguous slice of the points:
//   ocs_column_kernel  merges the per-CTA candidates for i (argmax of -G over a < 1, ties to the larger index), forms the kernel
//                      column Q_i (stored as float) and writes the CTA's candidate for j (argmax of (Gmax + G_t)^2 / quad over
//                      a > 0 with Gmax + G_t > 0) together with that point's G and a, and the CTA's max of G over a > 0;
//   ocs_update_kernel  merges the j candidates, takes the stop test and libsvm's clipped two-variable step (every CTA the same
//                      scalar arithmetic, CTA 0 stores it), forms Q_j, updates its slice of G and writes its candidate for the next i.
// A CTA reads only its own slice of G and a and takes G_i, G_j, a_i, a_j from the merged candidates, so no CTA reads what another
// CTA of the same launch writes.  Once the stop test has held, the state is final; later launches of the batch see `done` and return,
// so n_iter counts the updates exactly.
#pragma once
#include "kernels.cuh"

namespace cpd {

constexpr int OCS_THREADS = 512;          // threads per CTA of the SMO passes
constexpr int OCS_CTAS = 264;             // CTAs the passes aim at (2 per SM of a 132-SM H100); every CTA merges them all
constexpr double OCS_TAU = 1e-12;         // libsvm's TAU: a quad <= 0 becomes this

// Rounded double arithmetic that the compiler may not contract into an FMA: libsvm's values come from separately rounded
// products and sums.  (The CPU test build compiles with -ffp-contract=off.)
#ifdef CPD_HOST_EMU
__device__ __forceinline__ double ocs_mul(double a, double b) { return a * b; }
__device__ __forceinline__ double ocs_add(double a, double b) { return a + b; }
__device__ __forceinline__ double ocs_sub(double a, double b) { return a - b; }
#else
__device__ __forceinline__ double ocs_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ocs_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ocs_sub(double a, double b) { return __dsub_rn(a, b); }
#endif

struct alignas(32) OcsPt {
    double x, y, z, w;
};

// libsvm's kernel_rbf as its Qfloat: exp(-gamma (|x_i|^2 + |x_k|^2 - 2 x_i.x_k)) rounded to float32, returned as a double.
// p = {x, y, z (0 for 2-D), |x|^2}; the zero third coordinate adds exactly 0 to a 2-D dot product.
__device__ __forceinline__ double ocs_q(const OcsPt& p, const OcsPt& q, double gamma) {
    double dot = ocs_mul(p.x, q.x);
    dot = ocs_add(dot, ocs_mul(p.y, q.y));
    dot = ocs_add(dot, ocs_mul(p.z, q.z));
    const double d = ocs_sub(ocs_add(p.w, q.w), ocs_mul(2.0, dot));
    return (double)(float)exp(ocs_mul(-gamma, d));
}

// a candidate of a selection: the larger v wins, ties to the larger index k (libsvm's >= / <= scans in increasing index);
// g, a: that point's G and alpha
struct OcsCand {
    double v, g, a;
    long long k;
};
struct OcsState {
    long long i;           // this iteration's i (-1: every a is at 1)
    double gmax, gi, ai;   // -G_i, G_i and a_i
    long long a_iter;      // the iteration whose ocs_column_kernel ran last
    long long n_iter;      // updates made
    int done;              // the stop test has held
};

__device__ __forceinline__ void ocs_take(OcsCand& c, const OcsCand& o) {
    if (o.v > c.v || (o.v == c.v && o.k > c.k)) c = o;
}

// the block's best candidate and max of m, returned to every thread
__device__ __forceinline__ void ocs_block_reduce(OcsCand& c, double& m) {
    __shared__ OcsCand sc[OCS_THREADS / 32];
    __shared__ double sm[OCS_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        OcsCand x;
        x.v = __shfl_xor_sync(0xffffffffu, c.v, o);
        x.g = __shfl_xor_sync(0xffffffffu, c.g, o);
        x.a = __shfl_xor_sync(0xffffffffu, c.a, o);
        x.k = __shfl_xor_sync(0xffffffffu, c.k, o);
        ocs_take(c, x);
        m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { sc[wid] = c; sm[wid] = m; }
    __syncthreads();
    c = sc[0];
    m = sm[0];
    for (int w = 1; w < OCS_THREADS / 32; ++w) { ocs_take(c, sc[w]); m = fmax(m, sm[w]); }
    __syncthreads();                                   // the shared arrays may be written again
}

__device__ __forceinline__ OcsCand ocs_none() { return OcsCand{-INFINITY, 0.0, 0.0, -1}; }

// the merged candidates of the previous pass (one per CTA), to every thread
__device__ __forceinline__ void ocs_merge(const OcsCand* __restrict__ part, const double* __restrict__ mpart, int nparts, OcsCand& c,
                                          double& m) {
    c = ocs_none();
    m = -INFINITY;
    for (int b = threadIdx.x; b < nparts; b += OCS_THREADS) {
        ocs_take(c, part[b]);
        if (mpart) m = fmax(m, mpart[b]);
    }
    ocs_block_reduce(c, m);
}

// the CTA's slice of the points
__device__ __forceinline__ void ocs_slice(long long n, long long& lo, long long& hi) {
    const long long per = (n + gridDim.x - 1) / gridDim.x;
    lo = min(n, (long long)blockIdx.x * per);
    hi = min(n, lo + per);
}

// x (n x dim, caller's order) -> {x, y, z, |x|^2}, the squares summed over the dimensions in order
__global__ void __launch_bounds__(THREADS) ocs_prepare_kernel(const double* __restrict__ x, long long n, int dim, OcsPt* __restrict__ pts) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= n) return;
    const double* p = x + (size_t)k * dim;
    const double z = dim == 3 ? p[2] : 0.0;
    double s = ocs_mul(p[0], p[0]);
    s = ocs_add(s, ocs_mul(p[1], p[1]));
    s = ocs_add(s, ocs_mul(z, z));
    pts[k] = OcsPt{p[0], p[1], z, s};
}

// the start's G_k = sum_{i < k0} a_i Q_ik, over i in increasing order (libsvm's Solve); the k0 start points tiled through shared memory
__global__ void __launch_bounds__(THREADS) ocs_g0_kernel(const OcsPt* __restrict__ pts, const double* __restrict__ alpha, long long n,
                                                         long long k0, double gamma, double* __restrict__ G) {
    __shared__ OcsPt tp[THREADS];
    __shared__ double ta[THREADS];
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    const OcsPt pk = pts[min(k, n - 1)];
    double g = 0.0;
    for (long long t0 = 0; t0 < k0; t0 += THREADS) {
        const int cnt = (int)min((long long)THREADS, k0 - t0);
        __syncthreads();
        if (threadIdx.x < cnt) { tp[threadIdx.x] = pts[t0 + threadIdx.x]; ta[threadIdx.x] = alpha[t0 + threadIdx.x]; }
        __syncthreads();
        for (int t = 0; t < cnt; ++t) g = ocs_add(g, ocs_mul(ta[t], ocs_q(tp[t], pk, gamma)));
    }
    if (k < n) G[k] = g;
}

// the first i candidates: the CTA's argmax of -G over a < 1
__global__ void __launch_bounds__(OCS_THREADS) ocs_pick_kernel(const double* __restrict__ alpha, const double* __restrict__ G, long long n,
                                                               OcsCand* __restrict__ ipart) {
    long long lo, hi;
    ocs_slice(n, lo, hi);
    OcsCand c = ocs_none();
    double m = -INFINITY;
    for (long long k = lo + threadIdx.x; k < hi; k += OCS_THREADS)
        if (alpha[k] < 1.0) ocs_take(c, OcsCand{-G[k], 0.0, 0.0, k});
    ocs_block_reduce(c, m);
    if (threadIdx.x == 0) ipart[blockIdx.x] = c;
}

// first pass of iteration `it` (see the top of the file)
__global__ void __launch_bounds__(OCS_THREADS)
ocs_column_kernel(const OcsPt* __restrict__ pts, long long n, double gamma, const double* __restrict__ alpha, const double* __restrict__ G,
                  const OcsCand* __restrict__ ipart, float* __restrict__ qcol, OcsCand* __restrict__ jpart, double* __restrict__ mpart,
                  OcsState* __restrict__ st, long long it) {
    if (st->done) return;
    OcsCand ci;
    double unused;
    ocs_merge(ipart, nullptr, gridDim.x, ci, unused);
    const long long i = ci.k;
    const double gmax = ci.v;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        st->i = i;
        st->gmax = gmax;
        st->gi = i >= 0 ? G[i] : 0.0;
        st->ai = i >= 0 ? alpha[i] : 0.0;
        st->a_iter = it;
    }
    long long lo, hi;
    ocs_slice(n, lo, hi);
    OcsCand cj = ocs_none();
    double gmax2 = -INFINITY;
    const OcsPt pi = pts[max(i, 0LL)];
    for (long long k = lo + threadIdx.x; k < hi; k += OCS_THREADS) {
        const double gk = G[k], ak = alpha[k];
        double q = 0.0;
        if (i >= 0) {
            q = ocs_q(pi, pts[k], gamma);
            qcol[k] = (float)q;
        }
        if (ak > 0.0) {
            gmax2 = fmax(gmax2, gk);
            const double gd = gmax + gk;
            if (gd > 0.0) {                            // false for every k when i = -1 (gmax = -inf)
                double quad = ocs_sub(2.0, ocs_mul(2.0, q));
                if (quad <= 0.0) quad = OCS_TAU;
                ocs_take(cj, OcsCand{ocs_mul(gd, gd) / quad, gk, ak, k});   // libsvm minimises the negation
            }
        }
    }
    ocs_block_reduce(cj, gmax2);
    if (threadIdx.x == 0) { jpart[blockIdx.x] = cj; mpart[blockIdx.x] = gmax2; }
}

// second pass of iteration `it` (see the top of the file)
__global__ void __launch_bounds__(OCS_THREADS)
ocs_update_kernel(const OcsPt* __restrict__ pts, long long n, double gamma, double tol, double* __restrict__ alpha, double* __restrict__ G,
                  const float* __restrict__ qcol, const OcsCand* __restrict__ jpart, const double* __restrict__ mpart,
                  OcsCand* __restrict__ ipart, OcsState* __restrict__ st, long long it) {
    if (st->a_iter != it) return;                      // the column pass returned: the fit had already stopped
    OcsCand cj;
    double gmax2;
    ocs_merge(jpart, mpart, gridDim.x, cj, gmax2);
    const long long i = st->i, j = cj.k;
    const double gmax = st->gmax;
    if (gmax + gmax2 < tol || j < 0) {
        if (blockIdx.x == 0 && threadIdx.x == 0) st->done = 1;
        return;
    }
    // libsvm's update for y_i = y_j = +1 and C = 1
    const double gi = st->gi, ai0 = st->ai, gj = cj.g, aj0 = cj.a;
    double quad = ocs_sub(2.0, ocs_mul(2.0, (double)qcol[j]));
    if (quad <= 0.0) quad = OCS_TAU;
    const double delta = ocs_sub(gi, gj) / quad, sum = ocs_add(ai0, aj0);
    double ai = ocs_sub(ai0, delta), aj = ocs_add(aj0, delta);
    if (sum > 1.0) {
        if (ai > 1.0) { ai = 1.0; aj = ocs_sub(sum, 1.0); }
    } else if (aj < 0.0) {
        aj = 0.0; ai = sum;
    }
    if (sum > 1.0) {
        if (aj > 1.0) { aj = 1.0; ai = ocs_sub(sum, 1.0); }
    } else if (ai < 0.0) {
        ai = 0.0; aj = sum;
    }
    const double dai = ocs_sub(ai, ai0), daj = ocs_sub(aj, aj0);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        alpha[i] = ai;
        alpha[j] = aj;
        st->n_iter += 1;
    }
    long long lo, hi;
    ocs_slice(n, lo, hi);
    OcsCand c = ocs_none();
    double unused = -INFINITY;
    const OcsPt pj = pts[j];
    for (long long k = lo + threadIdx.x; k < hi; k += OCS_THREADS) {
        const double qi = (double)qcol[k], qj = ocs_q(pj, pts[k], gamma);
        const double g = ocs_add(G[k], ocs_add(ocs_mul(qi, dai), ocs_mul(qj, daj)));
        G[k] = g;
        const double ak = k == i ? ai : k == j ? aj : alpha[k];
        if (ak < 1.0) ocs_take(c, OcsCand{-g, 0.0, 0.0, k});
    }
    ocs_block_reduce(c, unused);
    if (threadIdx.x == 0) ipart[blockIdx.x] = c;
}

// libsvm's calculate_rho, per CTA: {sum of G over the free a (thread-strided, then the warp and CTA trees), the free count,
// min G over a = 0, max G over a = 1}; the host joins the CTAs in order
__global__ void __launch_bounds__(OCS_THREADS) ocs_rho_kernel(const double* __restrict__ alpha, const double* __restrict__ G, long long n,
                                                              double* __restrict__ part) {
    __shared__ double sh[4][OCS_THREADS / 32];
    long long lo, hi;
    ocs_slice(n, lo, hi);
    double s = 0.0, cnt = 0.0, ub = INFINITY, lb = -INFINITY;
    for (long long k = lo + threadIdx.x; k < hi; k += OCS_THREADS) {
        const double a = alpha[k], g = G[k];
        if (a >= 1.0) lb = fmax(lb, g);
        else if (a <= 0.0) ub = fmin(ub, g);
        else { s += g; cnt += 1.0; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        ub = fmin(ub, __shfl_xor_sync(0xffffffffu, ub, o));
        lb = fmax(lb, __shfl_xor_sync(0xffffffffu, lb, o));
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { sh[0][wid] = s; sh[1][wid] = cnt; sh[2][wid] = ub; sh[3][wid] = lb; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < OCS_THREADS / 32; ++w) {
            s += sh[0][w]; cnt += sh[1][w]; ub = fmin(ub, sh[2][w]); lb = fmax(lb, sh[3][w]);
        }
        double* o = part + (size_t)blockIdx.x * 4;
        o[0] = s; o[1] = cnt; o[2] = ub; o[3] = lb;
    }
}

}  // namespace cpd
