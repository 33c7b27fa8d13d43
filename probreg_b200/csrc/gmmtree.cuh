// gmmtree.cuh -- GMMTree (Eckart et al., ECCV 2018; probreg/cc/gmmtree.cc) on sm_90a: the hierarchical GMM build and the
// tree-descent registration E-step, FP64 throughout, every reduction in a fixed order (no atomics), so two runs on one device
// are bit-identical.  Host orchestration: host_gmmtree.inl.
//
// Tree layout (gmmtree.cc:42-44): 8 children per node, level l holds 8^(l+1) nodes from index level(l) = 8 (8^l - 1) / 7, and
// child(j) = 8 (j + 1), so child(-1) = 0.  A node is (pi, mu, Sigma); d_gt_nodes keeps 13 doubles per node {pi, mu[3], Sigma[9]}
// and gt_prep_kernel derives what the pdf needs into 16 doubles per node (GT_PREP).
//
// Moments go to the nodes by a sort-based segmented reduction, the same for the build and the registration E-step: the points are
// sorted by a key (the parent + 1 in the build, the chosen node in the registration), the sorted array is cut into fixed chunks of
// GT_CHUNK entries, one CTA per chunk reduces each key's run inside its chunk (gt_seg_partial_kernel), and the partials of one key
// are joined chunk by chunk (gt_build_mstep_kernel / gt_reg_merge_kernel).  A key u whose run touches chunks c0..c1 writes its
// partials to slots u + c0 .. u + c1: the runs are disjoint and sorted, so no two (key, chunk) pairs share a slot.
#pragma once
#include "kernels.cuh"

namespace cpd {

constexpr int GT_PREP = 16;          // {mu[3], Sigma^-1 [00 01 02 11 12 22], c, pi, det ok, complexity, pad[3]}
constexpr int GT_NODE = 13;          // {pi, mu[3], Sigma[9]}
constexpr int GT_MOM = 10;           // {gamma, gamma z[3], gamma z z^T [xx xy xz yy yz zz]}
constexpr int GT_CHUNK = 2048;       // sorted entries per CTA of the segmented reduction
constexpr int GT_LL_TILE = 64;       // nodes per shared-memory tile of the log-likelihood
constexpr double GT_EPS = 1.0e-15;   // gmmtree.cc:9
constexpr double GT_TWO_PI_1_5 = 15.749609945722419;    // (2 pi)^1.5

__host__ __device__ __forceinline__ long long gt_level_start(int l) {   // level(l) = 8 (8^l - 1) / 7
    long long p = 1;
    for (int i = 0; i < l; ++i) p *= 8;
    return 8 * (p - 1) / 7;
}

// gaussianPdf (gmmtree.cc:11-18) on a prepared node: 0 when det Sigma < 1e-15, else c exp(-d^T Sigma^-1 d / 2)
__device__ __forceinline__ double gt_pdf(const double* __restrict__ p, double x0, double x1, double x2) {
    if (p[11] == 0.0) return 0.0;
    const double d0 = x0 - p[0], d1 = x1 - p[1], d2 = x2 - p[2];
    const double q = d0 * (p[3] * d0 + p[4] * d1 + p[5] * d2) + d1 * (p[4] * d0 + p[6] * d1 + p[7] * d2) +
                     d2 * (p[5] * d0 + p[7] * d1 + p[8] * d2);
    return p[9] * exp(-0.5 * q);
}

// gamma over the 8 children from j0 (gmmtree.cc:141-152): pi_j pdf_j, normalised when the sum is > 1e-15, else all 0; returns the
// first index of the maximum (Eigen's maxCoeff), so an all-zero gamma picks child 0
__device__ __forceinline__ int gt_children(const double* __restrict__ prep, long long j0, double x0, double x1, double x2, double (&g)[8],
                                       double& gbest) {
    double den = 0.0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const double* p = prep + (size_t)(j0 + c) * GT_PREP;
        g[c] = p[10] * gt_pdf(p, x0, x1, x2);
        den += g[c];
    }
    const bool ok = den > GT_EPS;
    int best = 0;
    double gb = 0.0;                      // g[best], kept in a register (a dynamic index would put g in local memory)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        g[c] = ok ? g[c] / den : 0.0;
        if (c == 0 || g[c] > gb) { best = c; gb = g[c]; }
    }
    gbest = gb;
    return best;
}

// smallest / sum of the eigenvalues of a symmetric 3x3 matrix (complexity, gmmtree.cc:35-40), closed form (trigonometric)
__device__ __forceinline__ double gt_complexity(const double* __restrict__ s) {
    const double a00 = s[0], a01 = s[1], a02 = s[2], a11 = s[4], a12 = s[5], a22 = s[8];
    const double p1 = a01 * a01 + a02 * a02 + a12 * a12;
    const double tr = a00 + a11 + a22, q = tr / 3.0;
    double lmin;
    if (p1 == 0.0) {
        lmin = fmin(a00, fmin(a11, a22));
    } else {
        const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
        const double p2 = b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * p1;
        const double p = sqrt(p2 / 6.0);
        const double det_b = b00 * (b11 * b22 - a12 * a12) - a01 * (a01 * b22 - a12 * a02) + a02 * (a01 * a12 - b11 * a02);
        const double r = fmin(1.0, fmax(-1.0, det_b / (2.0 * p * p * p)));
        const double phi = acos(r) / 3.0;
        lmin = q + 2.0 * p * cos(phi + 2.0943951023931955);   // + 2 pi / 3: the smallest root
    }
    return lmin / tr;
}

// ---- preparation, initialisation, M-step ------------------------------------------------------------------------------------------
// per node of [j0, j0 + count): mu, Sigma^-1 by cofactors, c = 1 / (sqrt(det) (2 pi)^1.5) (0 when det < 1e-15), pi, the det flag
// and the complexity
__global__ void __launch_bounds__(THREADS)
gt_prep_kernel(const double* __restrict__ nodes, long long j0, long long count, double* __restrict__ prep) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= count) return;
    const double* nd = nodes + (size_t)(j0 + k) * GT_NODE;
    double* p = prep + (size_t)(j0 + k) * GT_PREP;
    const double* s = nd + 4;
    const double c00 = s[4] * s[8] - s[5] * s[7], c01 = s[5] * s[6] - s[3] * s[8], c02 = s[3] * s[7] - s[4] * s[6];
    const double det = s[0] * c00 + s[1] * c01 + s[2] * c02;
    const bool ok = det >= GT_EPS;
    const double id = 1.0 / det;
    p[0] = nd[1]; p[1] = nd[2]; p[2] = nd[3];
    p[3] = ok ? c00 * id : 0.0;
    p[4] = ok ? (s[2] * s[7] - s[1] * s[8]) * id : 0.0;
    p[5] = ok ? (s[1] * s[5] - s[2] * s[4]) * id : 0.0;
    p[6] = ok ? (s[0] * s[8] - s[2] * s[6]) * id : 0.0;
    p[7] = ok ? (s[2] * s[3] - s[0] * s[5]) * id : 0.0;
    p[8] = ok ? (s[0] * s[4] - s[1] * s[3]) * id : 0.0;
    p[9] = ok ? 1.0 / (sqrt(det) * GT_TWO_PI_1_5) : 0.0;
    p[10] = nd[0];
    p[11] = ok ? 1.0 : 0.0;
    p[12] = gt_complexity(s);
    p[13] = p[14] = p[15] = 0.0;
}

// block partials of {sum y (3)} (mean == nullptr) or of the centred scatter {sum (y - mean)(y - mean)^T (6)}
__global__ void __launch_bounds__(THREADS)
gt_moments_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ mean, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (!mean) {
        double v[3] = {0.0, 0.0, 0.0};
        if (i < n) { v[0] = pts[3 * i]; v[1] = pts[3 * i + 1]; v[2] = pts[3 * i + 2]; }
        block_reduce_store<3>(v, part + (size_t)blockIdx.x * 3);
    } else {
        const double inv_n = 1.0 / (double)n;
        double v[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        if (i < n) {
            const double a = pts[3 * i] - mean[0] * inv_n, b = pts[3 * i + 1] - mean[1] * inv_n, c = pts[3 * i + 2] - mean[2] * inv_n;
            v[0] = a * a; v[1] = a * b; v[2] = a * c; v[3] = b * b; v[4] = b * c; v[5] = c * c;
        }
        block_reduce_store<6>(v, part + (size_t)blockIdx.x * 6);
    }
}

// initializeNodes (gmmtree.cc:46-56) for leaf k: pi = 1/8, mu = y_seed, Sigma = sum_i (y_i - mu)(y_i - mu)^T / N, formed without
// cancellation as (S + N (ybar - mu)(ybar - mu)^T) / N.  sums: {sum y (3), S (6)}; inv: caller index -> internal index.
__global__ void __launch_bounds__(THREADS)
gt_leaf_init_kernel(const double* __restrict__ pts, const int* __restrict__ inv, const long long* __restrict__ seeds, long long nleaf,
                    long long lf, long long n, const double* __restrict__ sums, double* __restrict__ nodes) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= nleaf) return;
    const double* y = pts + 3 * (size_t)inv[seeds[k]];
    const double dn = (double)n;
    const double d[3] = {sums[0] / dn - y[0], sums[1] / dn - y[1], sums[2] / dn - y[2]};
    const int si[9] = {0, 1, 2, 1, 3, 4, 2, 4, 5};
    double* nd = nodes + (size_t)(lf + k) * GT_NODE;
    nd[0] = 1.0 / 8.0;
    for (int a = 0; a < 3; ++a) nd[1 + a] = y[a];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) nd[4 + 3 * a + b] = (sums[3 + si[3 * a + b]] + dn * d[a] * d[b]) / dn;
}

// initializeNodes (gmmtree.cc:57-72): every parent moment-matched from its 8 children, bottom up; one CTA
__global__ void __launch_bounds__(THREADS) gt_parent_init_kernel(double* __restrict__ nodes, int levels) {
    for (int l = levels - 2; l >= 0; --l) {
        const long long pl = gt_level_start(l), cl = gt_level_start(l + 1), cnt = cl - pl;
        for (long long j = threadIdx.x; j < cnt; j += THREADS) {
            double mu[3] = {0.0, 0.0, 0.0}, sg[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
            for (int c = 0; c < 8; ++c) {
                const double* ch = nodes + (size_t)(cl + 8 * j + c) * GT_NODE;
                for (int a = 0; a < 3; ++a) mu[a] += ch[1 + a];
                for (int a = 0; a < 3; ++a)
                    for (int b = 0; b < 3; ++b) sg[3 * a + b] += ch[4 + 3 * a + b] + ch[1 + a] * ch[1 + b];
            }
            double* nd = nodes + (size_t)(pl + j) * GT_NODE;
            nd[0] = 1.0 / 8.0;
            for (int a = 0; a < 3; ++a) nd[1 + a] = mu[a] / 8.0;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b) nd[4 + 3 * a + b] = sg[3 * a + b] / 8.0 - nd[1 + a] * nd[1 + b];
        }
        __syncthreads();
    }
}

// ---- the build E-step -------------------------------------------------------------------------------------------------------------
// gmmTreeEstep (gmmtree.cc:125-163) for the point at sorted position k, whose key is parent + 1: the 8 gammas (to g8, sorted
// order) and the argmax node (to cur, sorted order)
__global__ void __launch_bounds__(THREADS)
gt_build_estep_kernel(const double* __restrict__ spts, const unsigned* __restrict__ keys, long long n, const double* __restrict__ prep,
                      double* __restrict__ g8, int* __restrict__ cur) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= n) return;
    const long long j0 = 8LL * keys[k];
    double g[8], gb;
    const int best = gt_children(prep, j0, spts[3 * k], spts[3 * k + 1], spts[3 * k + 2], g, gb);
#pragma unroll
    for (int c = 0; c < 8; ++c) g8[8 * k + c] = g[c];
    cur[k] = (int)(j0 + best);
}

// start[u] / end[u]: the run of key u in the sorted keys (lower bounds of u and u + 1), u < nkeys
__global__ void __launch_bounds__(THREADS)
gt_bounds_kernel(const unsigned* __restrict__ keys, long long n, long long nkeys, int* __restrict__ start, int* __restrict__ end) {
    const long long u = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (u >= nkeys) return;
    for (int e = 0; e < 2; ++e) {
        long long lo = 0, hi = n;
        const unsigned key = (unsigned)(u + e);
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (keys[mid] < key) lo = mid + 1; else hi = mid;
        }
        (e ? end : start)[u] = (int)lo;
    }
}

// One CTA per chunk of GT_CHUNK sorted entries: for every key run inside the chunk and each of the NCH weights per entry, the
// fixed-order block sum of {w, w z, w z z^T}.  Entry k reads point i = idx ? idx[k] : k: pts[i] and weight g[i * NCH + c].
template <int NCH>
__global__ void __launch_bounds__(THREADS)
gt_seg_partial_kernel(const unsigned* __restrict__ keys, const int* __restrict__ idx, const double* __restrict__ pts,
                      const double* __restrict__ g, long long n, const int* __restrict__ start, const int* __restrict__ end,
                      double* __restrict__ part) {
    const long long c0 = (long long)blockIdx.x * GT_CHUNK, c1 = min(n, c0 + GT_CHUNK);
    const unsigned ka = keys[c0], kb = keys[c1 - 1];
    for (unsigned u = ka; u <= kb; ++u) {
        const long long a = max(c0, (long long)start[u]), b = min(c1, (long long)end[u]);
        if (a >= b) continue;                 // the same for every thread of the CTA
        for (int c = 0; c < NCH; ++c) {
            double v[GT_MOM];
#pragma unroll
            for (int t = 0; t < GT_MOM; ++t) v[t] = 0.0;
            for (long long k = a + threadIdx.x; k < b; k += THREADS) {
                const long long i = idx ? idx[k] : k;
                const double w = g[(size_t)i * NCH + c];
                const double z0 = pts[3 * i], z1 = pts[3 * i + 1], z2 = pts[3 * i + 2];
                const double w0 = w * z0, w1 = w * z1, w2 = w * z2;
                v[0] += w; v[1] += w0; v[2] += w1; v[3] += w2;
                v[4] += w0 * z0; v[5] += w0 * z1; v[6] += w0 * z2; v[7] += w1 * z1; v[8] += w1 * z2; v[9] += w2 * z2;
            }
            block_reduce_store<GT_MOM>(v, part + ((size_t)(u + blockIdx.x) * NCH + c) * GT_MOM);
            __syncthreads();                  // block_reduce_store's shared array is used again
        }
    }
}

// the moments of key u, child c: its chunk partials joined in chunk order (0 for an empty run)
template <int NCH>
__device__ __forceinline__ void gt_join(const double* __restrict__ part, const int* __restrict__ start, const int* __restrict__ end,
                                        long long u, int c, double (&s)[GT_MOM]) {
#pragma unroll
    for (int t = 0; t < GT_MOM; ++t) s[t] = 0.0;
    if (end[u] <= start[u]) return;
    for (long long ch = start[u] / GT_CHUNK; ch <= (end[u] - 1) / GT_CHUNK; ++ch) {
        const double* p = part + ((size_t)(u + ch) * NCH + c) * GT_MOM;
#pragma unroll
        for (int t = 0; t < GT_MOM; ++t) s[t] += p[t];
    }
}

// gmmTreeMstep / mlEstimator (gmmtree.cc:81-96, 166-173) for the nodes [j0, j0 + count) of one level; node j is child j % 8 of key
// j / 8 (= parent + 1).  n_points: all points, not the parent's.
__global__ void __launch_bounds__(THREADS)
gt_build_mstep_kernel(const double* __restrict__ part, const int* __restrict__ start, const int* __restrict__ end, long long j0,
                      long long count, long long n_points, double lambda_d, double* __restrict__ nodes) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= count) return;
    const long long j = j0 + k;
    double s[GT_MOM];
    gt_join<8>(part, start, end, j / 8, (int)(j % 8), s);
    double* nd = nodes + (size_t)j * GT_NODE;
    nd[0] = s[0] / (double)n_points;
    if (s[0] < lambda_d) {
        nd[0] = 0.0;
        for (int a = 0; a < 3; ++a) nd[1 + a] = 0.0;
        for (int a = 0; a < 9; ++a) nd[4 + a] = (a % 4 == 0) ? 1.0 : 0.0;
    } else {
        const int si[9] = {4, 5, 6, 5, 7, 8, 6, 8, 9};
        for (int a = 0; a < 3; ++a) nd[1 + a] = s[1 + a] / s[0];
        for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 3; ++b) nd[4 + 3 * a + b] = s[si[3 * a + b]] / s[0] - nd[1 + a] * nd[1 + b];
    }
}

// logLikelihood (gmmtree.cc:20-33) over the nodes [j0, j0 + count): per point log(max(sum_j pi_j pdf_j, 1e-15)), skipping nodes
// with pi < 1e-15, the nodes in index order through shared memory; block partials to part[blockIdx.x]
__global__ void __launch_bounds__(THREADS)
gt_loglik_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ prep, long long j0, long long count,
                 double* __restrict__ part) {
    __shared__ double tile[GT_LL_TILE * GT_PREP];
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double x0 = 0.0, x1 = 0.0, x2 = 0.0;
    if (i < n) { x0 = pts[3 * i]; x1 = pts[3 * i + 1]; x2 = pts[3 * i + 2]; }
    double tmp = 0.0;
    for (long long t0 = 0; t0 < count; t0 += GT_LL_TILE) {
        const int nt = (int)min((long long)GT_LL_TILE, count - t0);
        for (int e = threadIdx.x; e < nt * GT_PREP; e += THREADS) tile[e] = prep[(size_t)(j0 + t0) * GT_PREP + e];
        __syncthreads();
        for (int j = 0; j < nt; ++j) {
            const double* p = tile + j * GT_PREP;
            if (p[10] < GT_EPS) continue;
            tmp += p[10] * gt_pdf(p, x0, x1, x2);
        }
        __syncthreads();
    }
    double v[1] = {i < n ? log(fmax(tmp, GT_EPS)) : 0.0};
    block_reduce_store<1>(v, part + blockIdx.x);
}

// next level's sort input: key = argmax node + 1 (the parent + 1 of the next level), value = internal point index
__global__ void __launch_bounds__(THREADS)
gt_next_keys_kernel(const int* __restrict__ cur, const int* __restrict__ idx, long long n, unsigned* __restrict__ keys,
                    int* __restrict__ vals) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) { keys[k] = (unsigned)(cur[k] + 1); vals[k] = idx[k]; }
}
__global__ void __launch_bounds__(THREADS)
gt_gather_kernel(const double* __restrict__ pts, const int* __restrict__ idx, long long n, double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) {
        const long long i = idx[k];
        out[3 * k] = pts[3 * i]; out[3 * k + 1] = pts[3 * i + 1]; out[3 * k + 2] = pts[3 * i + 2];
    }
}
// caller's coordinates of the handle's cloud (internal order): in + origin; and the identity permutation
__global__ void __launch_bounds__(THREADS)
gt_uncentre_kernel(const double* __restrict__ in, long long n, double o0, double o1, double o2, double* __restrict__ out,
                   int* __restrict__ iota) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) {
        out[3 * k] = in[3 * k] + o0; out[3 * k + 1] = in[3 * k + 1] + o1; out[3 * k + 2] = in[3 * k + 2] + o2;
        iota[k] = (int)k;
    }
}
// inv[perm[k]] = k
__global__ void __launch_bounds__(THREADS) gt_inverse_perm_kernel(const int* __restrict__ perm, long long n, int* __restrict__ inv) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) inv[perm[k]] = (int)k;
}
// the final argmax of sorted entry k to the caller's order of the source
__global__ void __launch_bounds__(THREADS)
gt_assign_kernel(const int* __restrict__ cur, const int* __restrict__ idx, const int* __restrict__ perm, long long n,
                 int* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) out[perm[idx[k]]] = cur[k];
}

// ---- the registration E-step ------------------------------------------------------------------------------------------------------
// gmmTreeRegEstep (gmmtree.cc:175-215) for target point k: z = R (xc_k + origin) + t in FP64, descend from the root taking the
// argmax child, stop after the first node whose complexity is <= lambda_c; out: z, gamma of the chosen child, key = its node,
// val = k
__global__ void __launch_bounds__(THREADS)
gt_reg_descend_kernel(const double* __restrict__ xc, long long n, double o0, double o1, double o2, const double* __restrict__ rt,
                      const double* __restrict__ prep, int levels, double lambda_c, double* __restrict__ z, double* __restrict__ gsel,
                      unsigned* __restrict__ keys, int* __restrict__ vals) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k >= n) return;
    const double x0 = xc[3 * k] + o0, x1 = xc[3 * k + 1] + o1, x2 = xc[3 * k + 2] + o2;
    const double z0 = rt[0] * x0 + rt[1] * x1 + rt[2] * x2 + rt[9];
    const double z1 = rt[3] * x0 + rt[4] * x1 + rt[5] * x2 + rt[10];
    const double z2 = rt[6] * x0 + rt[7] * x1 + rt[8] * x2 + rt[11];
    long long search = -1;
    double gs = 0.0;
    for (int l = 0; l < levels; ++l) {
        const long long j0 = 8 * (search + 1);
        double g[8];
        search = j0 + gt_children(prep, j0, z0, z1, z2, g, gs);
        if (prep[(size_t)search * GT_PREP + 12] <= lambda_c) break;
    }
    z[3 * k] = z0; z[3 * k + 1] = z1; z[3 * k + 2] = z2;
    gsel[k] = gs;
    keys[k] = (unsigned)search;
    vals[k] = (int)k;
}

// the moments of every node (its chunk partials joined in chunk order), 13 per node: m0, m1[3], m2[3][3]
__global__ void __launch_bounds__(THREADS)
gt_reg_merge_kernel(const double* __restrict__ part, const int* __restrict__ start, const int* __restrict__ end, long long n_total,
                    double* __restrict__ out) {
    const long long j = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (j >= n_total) return;
    double s[GT_MOM];
    gt_join<1>(part, start, end, j, 0, s);
    const int si[9] = {4, 5, 6, 5, 7, 8, 6, 8, 9};
    double* o = out + (size_t)j * 13;
    for (int t = 0; t < 4; ++t) o[t] = s[t];
    for (int a = 0; a < 9; ++a) o[4 + a] = s[si[a]];
}

}  // namespace cpd
