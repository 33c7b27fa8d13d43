// lattice.cuh -- the permutohedral lattice of probreg's FilterReg (probreg/gaussian_filtering.py, third_party/permutohedral) on
// sm_90a, reproducing bit for bit what the reference's x86-64 build computes (its SSE lattice build and its compute() dispatch).
// Host orchestration: host_filterreg.inl.
//
// Build (Permutohedral::init, SSE path):
//   lat_elevate_kernel   one thread per point, plus one for the zero feature vector when the point count is not a multiple of 4 (the
//                        reference elevates points in blocks of 4 and hashes the padding lanes, whose vertices then enter the
//                        lattice): elevation, rounding to nearest-even (_mm_cvtps_epi32), rank, barycentric weights and the d+1
//                        keys, every float operation separately rounded in the reference's order.  A key (d shorts, wrapped to
//                        16 bits as the reference's (short) conversion wraps) is packed into 64 bits; the item is point*(d+1)+r.
//   radix sort           stable, so inside a vertex's run the items stay in (point, remainder) order: the reference's splat order.
//   lat_count / lat_scan_blocks / lat_number_kernel
//                        vertex ids from the run heads; the vertex's first sorted entry and key; each (point, remainder)'s vertex.
//   lat_neighbors_kernel the blur neighbours by binary search in the sorted unique keys.
// The hash table's numbering of the vertices changes no output, so the sorted numbering replaces it.
//
// Filter (Permutohedral::compute, which dispatches on the value size: seqCompute for 1-2 channels, sseCompute for 3 or more): all
// value sets of one call run together, each channel with its set's formulas (bit c of `sse`).
//   lat_splat_kernel     one warp per vertex streams the vertex's run: the lanes form the products w*v in parallel, then the sum is
//                        taken serially in run order, as the reference's point loop adds them.
//   lat_blur_kernel      one Jacobi pass per axis: new = old + 0.5*(n1 + n2); the scalar formula adds in double and rounds once.
//   lat_slice_kernel     per output point: scalar (w*v)*alpha, SSE (w*alpha)*v, summed over the d+1 vertices from 0.
#pragma once
#include "kernels.cuh"

namespace cpd {

constexpr int LAT_SCAN = 1024;            // entries per CTA of the vertex numbering
constexpr int LAT_MAX_CH = 8;             // channels one filter call carries (E-step: m0, m1, m2, nx)

// separately rounded arithmetic (no FMA contraction) and the reference's conversions
#ifdef CPD_HOST_EMU
__device__ __forceinline__ double lat_dadd(double a, double b) { return a + b; }
__device__ __forceinline__ double lat_dmul(double a, double b) { return a * b; }
__device__ __forceinline__ double lat_ddiv(double a, double b) { return a / b; }
__device__ __forceinline__ float lat_rint(float v) { return (float)(int)nearbyintf(v); }          // default mode: nearest-even
__device__ __forceinline__ short lat_short(float v) { return (short)(int)v; }
__device__ __forceinline__ float lat_d2f(double v) { return (float)v; }
#else
__device__ __forceinline__ double lat_dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double lat_dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double lat_ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float lat_rint(float v) { return __int2float_rn(__float2int_rn(v)); }
__device__ __forceinline__ short lat_short(float v) { return (short)__float2int_rz(v); }
__device__ __forceinline__ float lat_d2f(double v) { return __double2float_rn(v); }
#endif

__device__ __forceinline__ unsigned long long lat_pack(const short* k, int d) {
    unsigned long long r = 0;
    for (int i = 0; i < d; ++i) r |= (unsigned long long)(unsigned short)k[i] << (16 * i);
    return r;
}

// E-step features: [t_source / sigma ; target / sigma] rounded once to float (numpy's division, then pybind11's float32 copy)
__global__ void lat_features_kernel(const double* __restrict__ src, long long m, const double* __restrict__ tgt, long long n, int d,
                                    double sigma, float* __restrict__ feat) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (m + n) * d) return;
    const double x = k < m * d ? src[k] : tgt[k - m * d];
    feat[k] = lat_d2f(lat_ddiv(x, sigma));
}

// E-step values of every point, `ch` channels: sources 0; targets 1 | y | (y0^2 + y1^2) + y2^2 (FP64, rounded once) | normal
__global__ void lat_estep_values_kernel(const double* __restrict__ tgt, const double* __restrict__ nrm, long long m, long long n, int d,
                                        int with_m2, int ch, float* __restrict__ vals) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m + n) return;
    float* o = vals + i * ch;
    if (i < m) {
        for (int c = 0; c < ch; ++c) o[c] = 0.0f;
        return;
    }
    const double* y = tgt + (i - m) * d;
    int c = 0;
    o[c++] = 1.0f;
    for (int a = 0; a < d; ++a) o[c++] = lat_d2f(y[a]);
    if (with_m2) {
        double s = lat_dmul(y[0], y[0]);
        for (int a = 1; a < d; ++a) s = lat_dadd(s, lat_dmul(y[a], y[a]));
        o[c++] = lat_d2f(s);
    }
    if (nrm)
        for (int a = 0; a < d; ++a) o[c++] = lat_d2f(nrm[(i - m) * d + a]);
}

// Permutohedral::init (permutohedral.cpp:140-277) for point p of `np` (the last is the zero padding lane when np > n)
template <int D>
__global__ void lat_elevate_kernel(const float* __restrict__ feat, long long n, long long np, int with_blur,
                                   unsigned long long* __restrict__ keys, int* __restrict__ items, float* __restrict__ bary) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= np) return;
    const float invdp1 = 1.0f / (D + 1), dp1 = (float)(D + 1);
    const float inv_std = with_blur ? (float)(sqrt(2.0 / 3.0) * (D + 1)) : (float)(sqrt(1.0 / 6.0) * (D + 1));
    float f[D], el[D + 1], rem0[D + 1], rank[D + 1], b[D + 2];
    for (int j = 0; j < D; ++j) f[j] = p < n ? feat[p * D + j] : 0.0f;
    float sm = 0.0f;
    for (int j = D; j > 0; --j) {
        const float sf = lat_d2f(lat_dmul(1.0 / sqrt((double)((j + 1) * j)), (double)inv_std));
        const float cf = __fmul_rn(f[j - 1], sf);
        el[j] = __fsub_rn(sm, __fmul_rn((float)j, cf));
        sm = __fadd_rn(sm, cf);
    }
    el[0] = sm;
    float sum = 0.0f;
    for (int i = 0; i <= D; ++i) {
        const float v = lat_rint(__fmul_rn(invdp1, el[i]));
        rem0[i] = __fmul_rn(v, dp1);
        sum = __fadd_rn(sum, v);
        rank[i] = 0.0f;
    }
    for (int i = 0; i < D; ++i) {
        const float di = __fsub_rn(el[i], rem0[i]);
        for (int j = i + 1; j <= D; ++j) {
            const float c = di < __fsub_rn(el[j], rem0[j]) ? 1.0f : 0.0f;
            rank[i] = __fadd_rn(rank[i], c);
            rank[j] = __fadd_rn(rank[j], __fsub_rn(1.0f, c));
        }
    }
    for (int i = 0; i <= D; ++i) {
        rank[i] = __fadd_rn(rank[i], sum);
        const float add = rank[i] < 0.0f ? dp1 : 0.0f, sub = rank[i] >= dp1 ? dp1 : 0.0f;
        const float as = __fsub_rn(add, sub);
        rank[i] = __fadd_rn(rank[i], as);
        rem0[i] = __fadd_rn(rem0[i], as);
    }
    for (int i = 0; i < D + 2; ++i) b[i] = 0.0f;
    for (int i = 0; i <= D; ++i) {
        const float v = __fmul_rn(__fsub_rn(el[i], rem0[i]), invdp1);
        const int q = D - (int)rank[i];
        b[q] = __fadd_rn(b[q], v);
        b[q + 1] = __fsub_rn(b[q + 1], v);
    }
    b[0] = __fadd_rn(b[0], __fadd_rn(1.0f, b[D + 1]));
    for (int r = 0; r <= D; ++r) {
        short key[D];
        for (int i = 0; i < D; ++i) {
            const int ri = (int)rank[i];
            const int canon = ri <= D - r ? r : r - (D + 1);
            key[i] = lat_short(__fadd_rn(rem0[i], (float)canon));
        }
        const long long e = p * (D + 1) + r;
        keys[e] = lat_pack(key, D);
        items[e] = (int)e;
        bary[e] = b[r];
    }
}

// per CTA of LAT_SCAN sorted entries: the number of run heads
__global__ void lat_count_kernel(const unsigned long long* __restrict__ skeys, long long ne, int* __restrict__ cnt) {
    __shared__ int s[32];
    const long long i = (long long)blockIdx.x * LAT_SCAN + threadIdx.x;
    int h = (i < ne && (i == 0 || skeys[i] != skeys[i - 1])) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = h;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < LAT_SCAN / 32; ++w) t += s[w];
        cnt[blockIdx.x] = t;
    }
}

// exclusive scan of the CTA counts in place; cnt[nb] = the lattice size
__global__ void lat_scan_blocks_kernel(int* cnt, int nb) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    int run = 0;
    for (int b = 0; b < nb; ++b) {
        const int c = cnt[b];
        cnt[b] = run;
        run += c;
    }
    cnt[nb] = run;
}

// vertex ids: each head starts vertex v (first entry start[v], key ukey[v]); each real (point, remainder) learns its vertex
__global__ void lat_number_kernel(const unsigned long long* __restrict__ skeys, const int* __restrict__ sitems, long long ne,
                                  long long n_real_items, const int* __restrict__ cnt, int* __restrict__ start,
                                  unsigned long long* __restrict__ ukey, int* __restrict__ off) {
    __shared__ int s[LAT_SCAN];
    const long long i = (long long)blockIdx.x * LAT_SCAN + threadIdx.x;
    const int h = (i < ne && (i == 0 || skeys[i] != skeys[i - 1])) ? 1 : 0;
    s[threadIdx.x] = h;
    __syncthreads();
    for (int o = 1; o < LAT_SCAN; o <<= 1) {
        const int a = threadIdx.x >= (unsigned)o ? s[threadIdx.x - o] : 0;
        __syncthreads();
        s[threadIdx.x] += a;
        __syncthreads();
    }
    if (i >= ne) return;
    const int v = cnt[blockIdx.x] + s[threadIdx.x] - 1;
    if (h) {
        start[v] = (int)i;
        ukey[v] = skeys[i];
    }
    const int it = sitems[i];
    if (it < n_real_items) off[it] = v;
}

__device__ __forceinline__ int lat_find(const unsigned long long* ukey, int nv, unsigned long long k) {
    int lo = 0, hi = nv;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ukey[mid] < k) lo = mid + 1; else hi = mid;
    }
    return (lo < nv && ukey[lo] == k) ? lo : -1;
}

// blur neighbours (permutohedral.cpp:300-324) of vertex v along axis j, the pair (n1, n2) stored +1 (0: absent, the zero row)
template <int D>
__global__ void lat_neighbors_kernel(const unsigned long long* __restrict__ ukey, int nv, int* __restrict__ nbr) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)nv * (D + 1)) return;
    const int j = (int)(t / nv), v = (int)(t % nv);
    const unsigned long long k = ukey[v];
    short n1[D], n2[D];
    for (int i = 0; i < D; ++i) {
        const short ki = (short)(unsigned short)(k >> (16 * i));
        n1[i] = (short)(ki - 1);
        n2[i] = (short)(ki + 1);
        if (i == j) {
            n1[i] = (short)(ki + D);
            n2[i] = (short)(ki - D);
        }
    }
    nbr[2 * t] = lat_find(ukey, nv, lat_pack(n1, D)) + 1;
    nbr[2 * t + 1] = lat_find(ukey, nv, lat_pack(n2, D)) + 1;
}

// splat (permutohedral.cpp:491-499 / 553-562): one warp per vertex, the products in parallel, the sum serially in run order.
// vals row 0 stays zero (the reference shifts the vertices by one so that a missing neighbour reads 0).
__global__ void lat_splat_kernel(const int* __restrict__ sitems, const int* __restrict__ start, int nv, long long ne, int d,
                                 long long n, const float* __restrict__ bary, const float* __restrict__ in, int ch,
                                 float* __restrict__ vals) {
    const int lane = threadIdx.x & 31;
    const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long v = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < nv; v += nwarps) {
        const long long s0 = start[v], s1 = v + 1 < nv ? start[v + 1] : ne;
        float acc[LAT_MAX_CH];
        for (int c = 0; c < LAT_MAX_CH; ++c) acc[c] = 0.0f;
        for (long long base = s0; base < s1; base += 32) {
            const long long s = base + lane;
            float pr[LAT_MAX_CH];
            int ok = 0;
            if (s < s1) {
                const int it = sitems[s];
                const long long p = it / (d + 1);
                if (p < n) {
                    ok = 1;
                    const float w = bary[it];
                    for (int c = 0; c < LAT_MAX_CH; ++c) pr[c] = c < ch ? __fmul_rn(w, in[p * ch + c]) : 0.0f;
                }
            }
            if (!ok)
                for (int c = 0; c < LAT_MAX_CH; ++c) pr[c] = 0.0f;
            // all LAT_MAX_CH shuffles are issued unconditionally: they do not depend on the sum, so they run ahead of the serial
            // adds (guarding them by the live channel count measured 1.4x slower on the H100)
            const int cnt = (int)(s1 - base < 32 ? s1 - base : 32);
            for (int k = 0; k < cnt; ++k) {
                const int okk = __shfl_sync(0xffffffffu, ok, k);
                for (int c = 0; c < LAT_MAX_CH; ++c) {
                    const float x = __shfl_sync(0xffffffffu, pr[c], k);
                    if (okk && c < ch) acc[c] = __fadd_rn(acc[c], x);
                }
            }
        }
        if (lane < ch) {
            float a = acc[0];
            for (int c = 1; c < LAT_MAX_CH; ++c) if (c == lane) a = acc[c];
            vals[(v + 1) * ch + lane] = a;
        }
    }
}

// one Jacobi pass of the blur along axis j (permutohedral.cpp:501-517 / 564-581)
__global__ void lat_blur_kernel(const float* __restrict__ vals, const int* __restrict__ nbr, int nv, int j, int ch, unsigned sse,
                                float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)nv * ch) return;
    const long long v = t / ch;
    const int c = (int)(t % ch);
    const long long q = 2 * ((long long)j * nv + v);
    const float old = vals[(v + 1) * ch + c];
    const float s = __fadd_rn(vals[(long long)nbr[q] * ch + c], vals[(long long)nbr[q + 1] * ch + c]);
    out[(v + 1) * ch + c] = (sse >> c) & 1u ? __fadd_rn(old, __fmul_rn(0.5f, s))
                                            : lat_d2f(lat_dadd((double)old, lat_dmul(0.5, (double)s)));
}

// slice (permutohedral.cpp:521-531 / 586-596) at the first `ns` points
__global__ void lat_slice_kernel(const float* __restrict__ vals, const int* __restrict__ off, const float* __restrict__ bary,
                                 long long ns, int d, int ch, unsigned sse, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ns) return;
    const float alpha = 1.0f / (1.0f + (d == 2 ? 0.25f : 0.125f));
    float acc[LAT_MAX_CH];
    for (int c = 0; c < ch; ++c) acc[c] = 0.0f;
    for (int j = 0; j <= d; ++j) {
        const long long o = off[i * (d + 1) + j] + 1;
        const float w = bary[i * (d + 1) + j], wa = __fmul_rn(w, alpha);
        for (int c = 0; c < ch; ++c) {
            const float v = vals[o * ch + c];
            acc[c] = __fadd_rn(acc[c], (sse >> c) & 1u ? __fmul_rn(wa, v) : __fmul_rn(__fmul_rn(w, v), alpha));
        }
    }
    for (int c = 0; c < ch; ++c) out[i * ch + c] = acc[c];
}

// ---- FilterReg loop (cpd_filterreg_step): the move and the M-step moments, FP64 --------------------------------------------
constexpr int FR_MOM = 49;                // moments of one step, see include/cpd_b200.h
constexpr int FR_K1 = 12, FR_KH = 9, FR_KP = 28;

// x' = ((R_a0 x + R_a1 y) + R_a2 z) + t_a, every product and sum rounded on its own; tf = {R (d x d row-major), t}
__global__ void fr_move_kernel(const double* __restrict__ src, long long m, int d, const double* __restrict__ tf, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    for (int a = 0; a < d; ++a) {
        double acc = lat_dmul(tf[a * d], src[i * d]);
        for (int b = 1; b < d; ++b) acc = lat_dadd(acc, lat_dmul(tf[a * d + b], src[i * d + b]));
        out[i * d + a] = lat_dadd(acc, tf[d * d + a]);
    }
}

// one source's terms of filterreg.py:163-196: survivors have m0 != 0; y = m1 / m0, wt = sqrt(m0 / (m0 + c) / sigma2)
struct FrPoint {
    bool live;
    double m0, wt, x[3], y[3], m1[3], m2, nrm[3];
};
__device__ __forceinline__ FrPoint fr_point(const float* __restrict__ est, const double* __restrict__ x, long long i, int d, int ch,
                                            int upd, int has_n, double c, double sigma2) {
    FrPoint p;
    const float* r = est + i * ch;
    p.m0 = (double)r[0];
    p.live = p.m0 != 0.0;
    for (int a = 0; a < 3; ++a) p.x[a] = p.y[a] = p.m1[a] = p.nrm[a] = 0.0;
    p.m2 = upd ? (double)r[1 + d] : 0.0;
    p.wt = 0.0;
    if (!p.live) return p;
    p.wt = sqrt(p.m0 / (p.m0 + c) / sigma2);
    for (int a = 0; a < d; ++a) {
        p.x[a] = x[i * d + a];
        p.m1[a] = (double)r[1 + a];
        p.y[a] = p.m1[a] / p.m0;
        if (has_n) p.nrm[a] = (double)r[1 + d + upd + a] / p.m0;
    }
    return p;
}

// per CTA: {count, sum wt, sum wt x (3), sum wt y (3), sum wt^2, q = sum wt |x - y|, sigma2 numerator, sum m0 / (m0 + c)}
__global__ void __launch_bounds__(THREADS) fr_moments1_kernel(const float* __restrict__ est, const double* __restrict__ x, long long m,
                                                              int d, int ch, int upd, int has_n, double c, double sigma2,
                                                              double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[FR_K1];
    for (int k = 0; k < FR_K1; ++k) v[k] = 0.0;
    if (i < m) {
        const FrPoint p = fr_point(est, x, i, d, ch, upd, has_n, c, sigma2);
        if (p.live) {
            v[0] = 1.0;
            v[1] = p.wt;
            double dd = 0.0, xx = 0.0, xm = 0.0;
            for (int a = 0; a < 3; ++a) {
                v[2 + a] = p.wt * p.x[a];
                v[5 + a] = p.wt * p.y[a];
                dd += (p.x[a] - p.y[a]) * (p.x[a] - p.y[a]);
                xx += p.x[a] * p.x[a];
                xm += p.x[a] * p.m1[a];
            }
            v[8] = p.wt * p.wt;
            v[9] = p.wt * sqrt(dd);
            v[10] = (p.m0 * xx - 2.0 * xm + p.m2) / (p.m0 + c);
            v[11] = p.m0 / (p.m0 + c);
        }
    }
    block_reduce_store<FR_K1>(v, part + (size_t)blockIdx.x * FR_K1);
}

// per CTA: H = sum wt^2 (x - mc)(y - tc)^T (3 x 3 row-major), the centres from the first moments (mom)
__global__ void __launch_bounds__(THREADS) fr_moments_h_kernel(const float* __restrict__ est, const double* __restrict__ x, long long m,
                                                               int d, int ch, int upd, int has_n, double c, double sigma2,
                                                               const double* __restrict__ mom, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[FR_KH];
    for (int k = 0; k < FR_KH; ++k) v[k] = 0.0;
    if (i < m) {
        const FrPoint p = fr_point(est, x, i, d, ch, upd, has_n, c, sigma2);
        if (p.live) {
            const double w2 = p.wt * p.wt;
            for (int a = 0; a < 3; ++a)
                for (int b = 0; b < 3; ++b)
                    v[3 * a + b] = w2 * (p.x[a] - mom[2 + a] / mom[1]) * (p.y[b] - mom[5 + b] / mom[1]);
        }
    }
    block_reduce_store<FR_KH>(v, part + (size_t)blockIdx.x * FR_KH);
}

// per CTA (point to plane, cc/point_to_plane.cc:13-27): J = [x cross n, n], r = n . (y - x); J^T J weighted by wt (upper triangle,
// 21), J^T r weighted by wt (6), sum wt^2 r^2
__global__ void __launch_bounds__(THREADS) fr_moments_pl_kernel(const float* __restrict__ est, const double* __restrict__ x, long long m,
                                                                int ch, int upd, double c, double sigma2, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[FR_KP];
    for (int k = 0; k < FR_KP; ++k) v[k] = 0.0;
    if (i < m) {
        const FrPoint p = fr_point(est, x, i, 3, ch, upd, 1, c, sigma2);
        if (p.live) {
            const double* q = p.x;
            const double* nn = p.nrm;
            const double j[6] = {q[1] * nn[2] - q[2] * nn[1], q[2] * nn[0] - q[0] * nn[2], q[0] * nn[1] - q[1] * nn[0], nn[0], nn[1], nn[2]};
            const double r = nn[0] * (p.y[0] - q[0]) + nn[1] * (p.y[1] - q[1]) + nn[2] * (p.y[2] - q[2]);
            int k = 0;
            for (int a = 0; a < 6; ++a)
                for (int b = a; b < 6; ++b) v[k++] = p.wt * j[a] * j[b];
            for (int a = 0; a < 6; ++a) v[21 + a] = p.wt * r * j[a];
            v[27] = p.wt * p.wt * r * r;
        }
    }
    block_reduce_store<FR_KP>(v, part + (size_t)blockIdx.x * FR_KP);
}

}  // namespace cpd
