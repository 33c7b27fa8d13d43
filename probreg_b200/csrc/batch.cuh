// batch.cuh -- sm_90a device code of cpd_batch_register (host side: host_batch.inl): many independent rigid / affine CPD
// registrations in one launch, one CTA per pair for the whole registration.
//
// Why: clouds of a few hundred to a few thousand points leave the large-pair path (kernels.cuh) with almost nothing to do per
// launch; a registration then costs its set-up and one host round trip per iteration.  Here a pair's whole EM loop -- transform,
// E-step, moments, M-step and the tol test -- runs inside one CTA, and the B pairs of a batch share the GPU.
//
// The arithmetic is that of DESIGN.md section 2, pair for pair:
//   * the transform in FP64, one rounding to FP32 in the sigma-scaled frame centred on the target centroid (as pack_kernel);
//   * pass 1 per target: the integer-offset log-sum-exp (o, S, SU) with pass1_t's FMA chain, two-level FP32 sums (groups of GRP
//     from zero, SUB-point sub-chunks) and FP64 beyond;
//   * finalize-1 per target: dead columns, the outlier constant c, rn = 2^-o / den rounded once to FP32 and used by pass 2;
//   * pass 2 per source: p1 and the residual sd = sum_n P (a - b) with the SAME exponent (pass1_t on the record {b, -o}), the
//     same two-level sums;
//   * finalize-2's source-side sums into the RM_* layout, then mstep_solve_residual on the pair's DevState in shared memory.
// Both clouds are Morton-ordered inside their pair (DESIGN 2.4(i)) before this kernel runs (batch_frame_kernel + one CUB sort).
//
// Where it departs from the large-pair kernels, and why:
//   * Offsets.  A CTA of the large-pair pass 1 seeds each warp's offsets from the nearest source stage and rebases lazily when a
//     sub-chunk overflows.  Here one thread owns a target for a whole sweep over the pair's sources, so it takes the exact
//     minimum of u first (a sweep of pass1_u) and sets o = floor(min u) once: the rebasing slow path can never fire, and the
//     offset depends on the pair alone.  The extra sweep costs less than the pair sums it precedes.
//   * Finalize-1 and finalize-2 run per thread on one split's sums.  The per-column arithmetic of finalize 1 (finalize_column,
//     outlier_constant), the transform (frame_transform / frame_apply) and sigma2_0 (sigma2_closed_form) are the helpers the
//     large-pair path calls itself; only the merge of splits and the grid-wide layout of finalize1/2_kernel are not shared.
// Every sum runs in an order fixed by the pair's own sizes and points: a pair's result does not depend on its CTA index, on the
// other pairs or on the batch size.
//
// Resources of batch_em_kernel (ptxas -v, sm_90a, CUDA 12.9, the Makefile's flags): 223 registers, 0 bytes of spill stores and
// loads, an 832-byte stack frame in local memory (the M-step's 3 x 3 arrays, as moments_kernel<1> has one), 18 944 bytes of static
// shared memory; one CTA of 256 threads (8 warps) per SM.  Capped at 128 registers for two CTAs per SM, the kernel spills (60 bytes
// with mstep_solve_residual inlined; 24 bytes in the kernel and 24 in the callee with it behind a call), so it asks for one; whether
// two spilling CTAs per SM would be faster has not been measured.
#pragma once
#include "kernels.cuh"

namespace cpd {

constexpr int BT_TILE1 = 512;   // sources per shared-memory tile of pass 1 (16 B records: 8 KB); a multiple of SUB
constexpr int BT_TILE2 = 512;   // targets per tile of pass 2 (32 B records: 16 KB); a multiple of SUB
constexpr int BT_PAD = GRP;     // each pair's FP32 records are padded to whole groups with records whose terms are exactly 0
static_assert(BT_TILE1 % SUB == 0 && BT_TILE2 % SUB == 0 && SUB % GRP == 0 && GRP > 0, "batch tiles hold whole sub-chunks");

// one pair of the batch (host_batch.inl fills it)
struct BatchPair {
    long long src;     // first row of the pair's sources in the concatenated clouds (sources first, then targets)
    long long tgt;     // first row of its targets
    long long srcp;    // first record of its padded FP32 sources (srcP) and of its FP64 pass-2 sums (4 per record)
    long long tgtp;    // first record of its padded target records (tgtQ: 2 float4 each)
    int m, n;
};

__device__ __forceinline__ long long bt_pad(long long k) { return (k + BT_PAD - 1) / BT_PAD * BT_PAD; }

// block-wide min and max of three coordinates each (exact, so the order does not matter); result in lo[3], hi[3] of every thread
__device__ __forceinline__ void bt_block_minmax(double (&lo)[3], double (&hi)[3]) {
    __shared__ double sh[6][THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fmin(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmax(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if (lane == 0) { sh[a][wid] = lo[a]; sh[3 + a][wid] = hi[a]; }
    }
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = sh[a][0]; hi[a] = sh[3 + a][0];
        for (int w = 1; w < THREADS / 32; ++w) { lo[a] = fmin(lo[a], sh[a][w]); hi[a] = fmax(hi[a], sh[3 + a][w]); }
    }
    __syncthreads();
}

// One CTA per (pair, cloud): blockIdx.y = 0 the pair's sources, 1 its targets, slot = blockIdx.y * npairs + pair.  The cloud's
// centroid (FP64, fixed-order block reduction) goes to frame[4 slot ..], and every point gets the sort key
// slot << 30 | its Morton code in the cloud's own bounding box (the quantisation of morton_frame_kernel) and its row as the value.
// One stable radix sort over all keys then orders each cloud inside its pair and keeps the pairs where they were.
__global__ void __launch_bounds__(THREADS)
batch_frame_kernel(const double* __restrict__ raw /* rows x 3 */, const BatchPair* __restrict__ pairs, int npairs,
                   double* __restrict__ frame, unsigned long long* __restrict__ keys, int* __restrict__ idx) {
    __shared__ double sums[4];
    const int p = blockIdx.x, cloud = blockIdx.y;
    const BatchPair bp = pairs[p];
    const long long r0 = cloud ? bp.tgt : bp.src, cnt = cloud ? bp.n : bp.m;
    double v[3] = {0.0, 0.0, 0.0}, lo[3] = {1.0e300, 1.0e300, 1.0e300}, hi[3] = {-1.0e300, -1.0e300, -1.0e300};
    for (long long i = threadIdx.x; i < cnt; i += THREADS)
        for (int a = 0; a < 3; ++a) {
            const double x = raw[3 * (r0 + i) + a];
            v[a] += x; lo[a] = fmin(lo[a], x); hi[a] = fmax(hi[a], x);
        }
    block_reduce_store<3>(v, sums);
    bt_block_minmax(lo, hi);                  // its first __syncthreads also publishes sums[]
    const long long slot = (long long)cloud * npairs + p;
    if (threadIdx.x < 3) frame[4 * slot + threadIdx.x] = sums[threadIdx.x] / (double)cnt;
    const double range = fmax(hi[0] - lo[0], fmax(hi[1] - lo[1], hi[2] - lo[2]));
    const double inv_range = range > 0.0 ? 1.0 / range : 0.0;
    for (long long i = threadIdx.x; i < cnt; i += THREADS) {
        const double* q = raw + 3 * (r0 + i);
        const unsigned a = (unsigned)fmin(fmax((q[0] - lo[0]) * inv_range * 1023.0, 0.0), 1023.0),
                       b = (unsigned)fmin(fmax((q[1] - lo[1]) * inv_range * 1023.0, 0.0), 1023.0),
                       c = (unsigned)fmin(fmax((q[2] - lo[2]) * inv_range * 1023.0, 0.0), 1023.0);
        keys[r0 + i] = ((unsigned long long)slot << 30) | (spread3(a) | (spread3(b) << 1) | (spread3(c) << 2));
        idx[r0 + i] = (int)(r0 + i);
    }
}

// out[k] = raw[perm[k]] - the centroid of k's cloud: the sorted rows of a cloud stay in the rows the cloud had
__global__ void __launch_bounds__(THREADS)
batch_gather_kernel(const double* __restrict__ raw, const int* __restrict__ perm, const BatchPair* __restrict__ pairs, int npairs,
                    const double* __restrict__ frame, double* __restrict__ out) {
    const int p = blockIdx.x, cloud = blockIdx.y;
    const BatchPair bp = pairs[p];
    const long long r0 = cloud ? bp.tgt : bp.src, cnt = cloud ? bp.n : bp.m;
    const double* c = frame + 4 * ((long long)cloud * npairs + p);
    for (long long k = threadIdx.x; k < cnt; k += THREADS) {
        const long long j = perm[r0 + k];
        for (int a = 0; a < 3; ++a) out[3 * (r0 + k) + a] = raw[3 * j + a] - c[a];
    }
}

// finalize 1 of one target from its single (o, S, SU): finalize1_kernel's column arithmetic (finalize_column) without the merge of
// splits.  Returns the pass-2 record in rec0, rec1 and the target-side moments {SU rn, pt1}.
__device__ __forceinline__ void batch_finalize1(const DevState& st, float o, double S, double SU, float bx, float by, float bz,
                                                float4& rec0, float4& rec1, double& srr, double& pt1) {
    const double log2S = S > 0.0 ? log2(S) - (double)o : -INFINITY;
    const double c = outlier_constant(st.sigma2, st.w, st.dim, st.m, st.n_global);
    float no, rnf;
    finalize_column(log2S, c, c > 0.0 ? log2(c) : -INFINITY, 0.0, o, SU, pt1, no, rnf, srr);
    rec0 = make_float4(bx, by, bz, no);
    rec1 = make_float4(rnf, 0.f, 0.f, 0.f);
}

// The whole registration of pair order[blockIdx.x] (longest first: the host sorts by m n).  states[p] arrives with the
// transformation to start from, tf_kind, update_scale, w, dim, m and n_global; the kernel adds the centroids, sigma2_0 and q_0
// (cpd_sigma2_init's closed form, cpd.py:148), runs at most maxiter EM iterations with cpd_em_run's stop rule and leaves the last
// MstepResult in states[p] and the iterations run in iters[p].  A pair whose sigma2_0 is not a positive number runs nothing and
// gets err = 1.  Scratch per pair: srcP (padded sources), tgtQ (padded target records), part (p1 and sd per source).
__global__ void __launch_bounds__(THREADS, 1)
batch_em_kernel(const BatchPair* __restrict__ pairs, const int* __restrict__ order, int npairs, const double* __restrict__ pts,
                const double* __restrict__ frame, DevState* __restrict__ states, int maxiter, double tol, float4* __restrict__ srcP,
                float4* __restrict__ tgtQ, double* __restrict__ part, int* __restrict__ iters) {
    __shared__ DevState sst;
    __shared__ double smom[MOM_PAD];
    __shared__ __align__(16) float4 tile[2 * BT_TILE2];
    __shared__ int s_done;
    static_assert(2 * BT_TILE2 >= BT_TILE1, "one tile buffer serves both passes");
    static_assert(sizeof(DevState) % 8 == 0, "DevState is copied as 8-byte words");
    const int p = order[blockIdx.x], tid = threadIdx.x;
    const BatchPair bp = pairs[p];
    const int m = bp.m, n = bp.n;
    const int mp = (int)bt_pad(m), np = (int)bt_pad(n);
    const double* __restrict__ yc = pts + 3 * bp.src;
    const double* __restrict__ xc = pts + 3 * bp.tgt;
    float4* __restrict__ sP = srcP + bp.srcp;
    float4* __restrict__ tQ = tgtQ + 2 * bp.tgtp;
    double* __restrict__ pp = part + 4 * bp.srcp;
    for (int e = tid; e < (int)(sizeof(DevState) / 8); e += THREADS)
        reinterpret_cast<double*>(&sst)[e] = reinterpret_cast<const double*>(&states[p])[e];
    // prologue: sigma2_0 from the clouds' sums in the target frame (cpd_sigma2_init), q_0 = 1 + N D / 2 log sigma2_0
    {
        double v[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int j = tid; j < n; j += THREADS) {
            const double a = xc[3 * j], b = xc[3 * j + 1], c = xc[3 * j + 2];
            v[0] += a * a + b * b + c * c; v[1] += a; v[2] += b; v[3] += c;
        }
        for (int i = tid; i < m; i += THREADS) {
            const double a = yc[3 * i], b = yc[3 * i + 1], c = yc[3 * i + 2];
            v[4] += a * a + b * b + c * c; v[5] += a; v[6] += b; v[7] += c;
        }
        block_reduce_store<8>(v, smom);
        __syncthreads();
        if (tid == 0) {
            const double* sx = smom;
            const double* sy = smom + 4;
            const double* cy = frame + 4 * (long long)p;
            const double* cx = frame + 4 * ((long long)npairs + p);
            for (int a = 0; a < 3; ++a) { sst.cx[a] = cx[a]; sst.cy[a] = cy[a]; }
            const double N = (double)n;
            const double s2 = sigma2_closed_form(sx, sy, sst.cx, sst.cy, (double)m, N, sst.dim);
            sst.sigma2 = s2;
            sst.q = 1.0 + N * sst.dim * 0.5 * log(s2);
            sst.n_p = 0.0;
            sst.err = (s2 > 0.0 && isfinite(s2)) ? 0 : 1;
            s_done = sst.err || maxiter <= 0;
        }
        __syncthreads();
    }
    int it = 0;
    while (!s_done) {
        // transform + centre + scale the sources, one rounding to FP32 (pack_kernel's arithmetic)
        const double sk = sqrt(LOG2E / (2.0 * sst.sigma2));
        {
            double l[9], tp[3];
            frame_transform(sst, l, tp);
            for (int i = tid; i < mp; i += THREADS) {
                float4 o;
                if (i < m) {
                    double px, py, pz;
                    frame_apply(l, tp, yc[3 * i], yc[3 * i + 1], yc[3 * i + 2], px, py, pz);
                    o = make_float4((float)(sk * px), (float)(sk * py), (float)(sk * pz), 0.0f);
                } else {
                    o = make_float4(FAR_COORD, FAR_COORD, FAR_COORD, 0.0f);     // u = 3e36: every term exactly 0
                }
                sP[i] = o;
            }
        }
        __syncthreads();
        // pass 1 + finalize 1, one target per thread
        double vt[RM_TGT] = {0.0, 0.0};
        for (int j0 = 0; j0 < n; j0 += THREADS) {
            const int j = j0 + tid;
            const int jj = j < n ? j : n - 1;
            const float bx = (float)(sk * xc[3 * jj]), by = (float)(sk * xc[3 * jj + 1]), bz = (float)(sk * xc[3 * jj + 2]);
            float cm = 3.0e38f;
            for (int s0 = 0; s0 < mp; s0 += BT_TILE1) {
                const int len = min(BT_TILE1, mp - s0);
                __syncthreads();
                for (int k = tid; k < len; k += THREADS) tile[k] = sP[s0 + k];
                __syncthreads();
#pragma unroll 8
                for (int k = 0; k < len; ++k) cm = fminf(cm, pass1_u<false>(bx, by, bz, tile[k]));
            }
            const float o = fminf(O_INIT, floorf(cm)), no = -o;
            double S = 0.0, SU = 0.0;
            for (int s0 = 0; s0 < mp; s0 += BT_TILE1) {
                const int len = min(BT_TILE1, mp - s0);
                __syncthreads();
                for (int k = tid; k < len; k += THREADS) tile[k] = sP[s0 + k];
                __syncthreads();
                for (int sc = 0; sc < len; sc += SUB) {
                    const int end = min(sc + SUB, len);
                    float Sc = 0.0f, Uc = 0.0f;
#pragma unroll 1
                    for (int g0 = sc; g0 < end; g0 += GRP) {
                        float gs = 0.0f, gu = 0.0f;
#pragma unroll
                        for (int q = 0; q < GRP; ++q) {
                            const float t = pass1_t<false>(bx, by, bz, no, tile[g0 + q]);
                            const float e = ex2(-t);
                            gs = q == 0 ? e : __fadd_rn(gs, e);
                            gu = q == 0 ? __fmul_rn(e, t) : __fmaf_rn(e, t, gu);
                        }
                        Sc = __fadd_rn(Sc, gs); Uc = __fadd_rn(Uc, gu);
                    }
                    S += (double)Sc;
                    SU += (double)Uc - (double)no * (double)Sc;         // sum e*u = sum e*t' + o * sum e
                }
            }
            if (j < n) {
                float4 r0, r1;
                double srr, pt1;
                batch_finalize1(sst, o, S, SU, bx, by, bz, r0, r1, srr, pt1);
                tQ[2 * j] = r0; tQ[2 * j + 1] = r1;
                vt[0] += srr; vt[1] += pt1;
            }
        }
        for (int j = n + tid; j < np; j += THREADS) {      // dead padding records: 2^-(u - o) == 0, rn = 0
            tQ[2 * j] = make_float4(0.f, 0.f, 0.f, INFINITY);
            tQ[2 * j + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        block_reduce_store<RM_TGT>(vt, smom + RM_SRR);
        __syncthreads();
        // pass 2, one source per thread: p1 and sd = sum_n P (a - b)
        for (int i0 = 0; i0 < m; i0 += THREADS) {
            const int i = i0 + tid;
            const float4 a = sP[i < m ? i : m - 1];
            double A1 = 0.0, AX = 0.0, AY = 0.0, AZ = 0.0;
            for (int t0 = 0; t0 < np; t0 += BT_TILE2) {
                const int len = min(BT_TILE2, np - t0);
                __syncthreads();
                for (int k = tid; k < 2 * len; k += THREADS) tile[k] = tQ[2 * t0 + k];
                __syncthreads();
                for (int sc = 0; sc < len; sc += SUB) {
                    const int end = min(sc + SUB, len);
                    float s1 = 0.0f, sx = 0.0f, sy = 0.0f, sz = 0.0f;
#pragma unroll 1
                    for (int g0 = sc; g0 < end; g0 += GRP) {
                        float g1 = 0.0f, gx = 0.0f, gy = 0.0f, gz = 0.0f;
#pragma unroll
                        for (int q = 0; q < GRP; ++q) {
                            const float4 b = tile[2 * (g0 + q)];
                            const float rn = tile[2 * (g0 + q) + 1].x;
                            const float dx = __fsub_rn(a.x, b.x), dy = __fsub_rn(a.y, b.y), dz = __fsub_rn(a.z, b.z);
                            const float t = pass1_t<false>(a.x, a.y, a.z, b.w, b);       // t' = u - o_n: pass 1's exponent
                            const float pr = __fmul_rn(ex2(-t), rn);
                            g1 = q == 0 ? pr : __fadd_rn(g1, pr);
                            gx = q == 0 ? __fmul_rn(pr, dx) : __fmaf_rn(pr, dx, gx);
                            gy = q == 0 ? __fmul_rn(pr, dy) : __fmaf_rn(pr, dy, gy);
                            gz = q == 0 ? __fmul_rn(pr, dz) : __fmaf_rn(pr, dz, gz);
                        }
                        s1 = __fadd_rn(s1, g1); sx = __fadd_rn(sx, gx); sy = __fadd_rn(sy, gy); sz = __fadd_rn(sz, gz);
                    }
                    A1 += (double)s1; AX += (double)sx; AY += (double)sy; AZ += (double)sz;
                }
            }
            if (i < m) {
                pp[4 * i] = A1; pp[4 * i + 1] = AX; pp[4 * i + 2] = AY; pp[4 * i + 3] = AZ;
            }
        }
        __syncthreads();
        // finalize 2: the source-side moments (finalize2_kernel's sums), each thread over its sources, then the block in a fixed order
        {
            double v[RM_SRC];
#pragma unroll
            for (int k = 0; k < RM_SRC; ++k) v[k] = 0.0;
            const double inv_sk = 1.0 / sk;
            for (int i = tid; i < m; i += THREADS) {
                const double a1 = pp[4 * i];
                const double vv[3] = {-pp[4 * i + 1] * inv_sk, -pp[4 * i + 2] * inv_sk, -pp[4 * i + 3] * inv_sk};
                const double y[3] = {yc[3 * i], yc[3 * i + 1], yc[3 * i + 2]};
                v[RM_NP] += a1;
#pragma unroll
                for (int d = 0; d < 3; ++d) {
                    v[RM_SY + d] += a1 * y[d];
                    v[RM_V1 + d] += vv[d];
#pragma unroll
                    for (int e = 0; e < 3; ++e) v[RM_VY + 3 * d + e] += vv[d] * y[e];
                }
                v[RM_C + 0] += a1 * y[0] * y[0]; v[RM_C + 1] += a1 * y[0] * y[1]; v[RM_C + 2] += a1 * y[0] * y[2];
                v[RM_C + 3] += a1 * y[1] * y[1]; v[RM_C + 4] += a1 * y[1] * y[2]; v[RM_C + 5] += a1 * y[2] * y[2];
            }
            block_reduce_store<RM_SRC>(v, smom);
        }
        __syncthreads();
        // M-step on the shared state, then cpd_em_run's stop rule (cpd.py:117)
        if (tid == 0) {
            const double q_prev = sst.q;
            mstep_solve_residual(&sst, smom);
            s_done = fabs(sst.q - q_prev) < tol || it + 1 >= maxiter;
        }
        ++it;
        __syncthreads();
    }
    if (tid == 0) iters[p] = it;
    for (int e = tid; e < (int)(sizeof(DevState) / 8); e += THREADS)
        reinterpret_cast<double*>(&states[p])[e] = reinterpret_cast<const double*>(&sst)[e];
}

}  // namespace cpd
