// gram_i8.cuh -- the Gram-matrix product  out[c][i] = sum_j G_ij X[c][j]  with EXACT accumulation on the tensor cores:
// both operands are cut into 8-bit digits and multiplied with Hopper's warpgroup MMA (wgmma.mma_async m64n64k32, unsigned x
// signed 8-bit, 32-bit integer accumulators in registers).  Integer MMAs do not round, so the only errors are the two
// quantisations (2^-24 absolute on G, 2^-23 of the column maximum on X), at the level of the float32 G the reference itself uses
// (cc/math_utils.cc:17-19).  Role: the products of the low-rank range finder (probreg/cpd.py:296-297 with
// G = rbf_kernel(Y, Y, beta) of transformation.py:91-102) and, as the LR_IMQ instantiation, of low-rank BCPD (the inverse multiquadric,
// lowrank.cuh); G is never stored -- it is generated tile by tile on the CUDA cores.
//
// Fixed point ("Ozaki splitting" with integer digits):
//     g_ij = round(2^23 G_ij) in [0, 2^23]         = a0 2^16 + a1 2^8 + a2,     a_s in [0, 255]        (unsigned digits, a0 <= 128)
//     x_cj = round(2^22 X[c][j] / max_j |X[c][j]|) = b0 2^16 + b1 2^8 + b2,     b_t in [-128, 127]     (balanced digits, |b0| <= 64)
//     g x  = sum_{s,t} a_s b_t 2^(8 (4 - s - t)):   the products of level l = s + t share one accumulator,
//            levels 0, 1, 2 are kept (6 MMAs per 32 points), levels 3 and 4 (< 2^-22 of the largest term) are dropped.
// An accumulator receives at most 3 products of magnitude < 2^15 per point: exact in int32 for chunks of up to 16384 points.
// The epilogue joins the three levels in FP64 (exact) and applies the column scale; chunk partials are added in a fixed order.
//
// CTA = GI_WG consumer warpgroups of 64 rows each + one producer warp, persistent over work units {row tile, j-chunk}; the
// columns of X are taken in passes of GI_N = 64 (3 levels x 32 accumulator registers per thread).
//     producer warp   one lane streams each 32-point stage -- the three digit planes of X (the B operands, 3 x 2 KB) and the
//                     stage's 32 j-points (512 B) -- into a ring of GI_STAGES shared-memory slots with bulk copies (TMA,
//                     cp.async.bulk) completing on the slot's `full` mbarrier
//     warpgroups      generate their 64 x 32 tile of G straight into the wgmma A-operand register fragment (no shared-memory
//                     round trip for A), issue the six MMAs, wait for them and release the slot (`empty` mbarrier, one arrival
//                     per warp).  While one warpgroup waits on its MMAs the others generate: the CUDA-core work and the
//                     tensor-core work of the SM overlap across warpgroups.
// Shared-memory B layout: K-major, 32-byte rows, 32-byte swizzle: row r at byte 32 r (8-row groups 256 B apart = the descriptor's
// stride byte offset), the 16-byte half h of a row at position h ^ ((r >> 2) & 1).  gi_split_kernel stores the digit planes of X in
// global memory AS these stage images, so a stage is one bulk copy.
#pragma once
#ifndef CPD_HOST_EMU
#include "kernels.cuh"

namespace cpd {

constexpr int GI_WG = 2;                               // consumer warpgroups per CTA
constexpr int GI_ROWS = 64 * GI_WG;                    // rows of G per work unit
constexpr int GI_KS = 32;                              // j-points per stage = one m64n64k32 K-step (32 bytes per row)
constexpr int GI_N = 64;                               // columns of X per pass (the MMA's N)
constexpr int GI_STAGES = 8;
constexpr int GI_PLANE = GI_N * GI_KS;                 // bytes of one digit plane of a stage (2 KB)
constexpr int GI_PTS_BYTES = GI_KS * 16;               // the stage's 32 j-points (float4)
constexpr int GI_THREADS = GI_WG * 128 + 32;
constexpr int GI_SMEM = GI_STAGES * (3 * GI_PLANE + GI_PTS_BYTES) + 256 /* alignment slack */ + 256 /* barriers */;
constexpr int GI_MAX_CHUNK = 16384;

// ---- PTX wrappers ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void gi_mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// shared-memory matrix descriptor of a K-major operand with 32-byte swizzle: start >> 4 in [0,14), leading byte offset >> 4 in
// [16,30) (unused for a swizzled K-major operand whose K extent is one swizzle row; 1 by convention), stride byte offset >> 4 in
// [32,46) (8 rows x 32 B = 256), layout type in [62,64): 3 = 32-byte swizzle
__device__ __forceinline__ uint64_t gi_smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3ffffu) >> 4) | (1ull << 16) | ((uint64_t)(256 >> 4) << 32) | (3ull << 62);
}
__device__ __forceinline__ uint32_t gi_row_half_offset(int r, int h) { return (uint32_t)(r * 32 + ((h ^ ((r >> 2) & 1)) << 4)); }
__device__ __forceinline__ void gi_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void gi_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void gi_wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 64] (+)= A[64 x 32] (u8, this thread's register fragment) * B[32 x 64] (s8, K-major in shared memory)
__device__ __forceinline__ void gi_mma(int (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, int accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p;\n"
        "}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]),
          "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
          "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]),
          "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
        : "memory");
}

// ---- operand preparation -----------------------------------------------------------------------------------------------------------
// colmax[c] = max_j |X[c][j]|   (one CTA per column)
__global__ void __launch_bounds__(THREADS)
gi_colmax_kernel(const double* __restrict__ X, long long m, long long ld, double* __restrict__ colmax) {
    __shared__ double sh[THREADS / 32];
    const int c = blockIdx.x;
    double v = 0.0;
    for (long long j = threadIdx.x; j < m; j += THREADS) v = fmax(v, fabs(X[(long long)c * ld + j]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < THREADS / 32; ++w) v = fmax(v, sh[w]);
        colmax[c] = v;
    }
}
// digit planes of the columns [c0, c0 + nc) as stage images: image[jb] (jb = point block of 32) = 3 planes x GI_PLANE bytes, plane p
// holds digit p of column c (row c, 32 bytes, the two 16-byte halves swizzled like the MMA reads them).  One thread = one column x
// 16 points = one 16-byte store per plane; rows c >= nc and points j >= m are zero.
__global__ void __launch_bounds__(THREADS)
gi_split_kernel(const double* __restrict__ X, long long m, long long ld, int nc, int n16, long long ldx, const double* __restrict__ colmax,
                unsigned char* __restrict__ images) {
    const long long jh = (long long)blockIdx.x * THREADS + threadIdx.x;          // 16-point group
    const int c = blockIdx.y;
    if (jh * 16 < ldx && c < n16) {
        uint32_t w[3][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
        const double mx = c < nc ? colmax[c] : 0.0;
        if (mx > 0.0) {
            const double inv = 4194304.0 / mx;
#pragma unroll
            for (int k = 0; k < 16; ++k) {
                const long long j = jh * 16 + k;
                if (j < m) {
                    const int xi = (int)rint(X[(long long)c * ld + j] * inv);                 // |xi| <= 2^22
                    const int b2 = ((xi + 128) & 255) - 128;
                    const int r1 = (xi - b2) >> 8;
                    const int b1 = ((r1 + 128) & 255) - 128;
                    const int b0 = (r1 - b1) >> 8;
                    w[0][k >> 2] |= (uint32_t)(b0 & 255) << (8 * (k & 3));
                    w[1][k >> 2] |= (uint32_t)(b1 & 255) << (8 * (k & 3));
                    w[2][k >> 2] |= (uint32_t)(b2 & 255) << (8 * (k & 3));
                }
            }
        }
        unsigned char* img = images + (jh >> 1) * (3 * GI_PLANE) + gi_row_half_offset(c, (int)(jh & 1));
#pragma unroll
        for (int p = 0; p < 3; ++p) *reinterpret_cast<uint4*>(img + p * GI_PLANE) = make_uint4(w[p][0], w[p][1], w[p][2], w[p][3]);
    }
}
// out[c][i_begin + ii] = sum over the j-chunks of part[q][c][ii] (FP64, chunk order)
__global__ void __launch_bounds__(THREADS)
gi_reduce_kernel(const double* __restrict__ part, int nq, int n16, long long ldp, int nc, long long rows, long long i_begin, long long ld,
                 double* __restrict__ out) {
    const long long ii = (long long)blockIdx.x * THREADS + threadIdx.x;
    const int c = blockIdx.y;
    if (ii < rows && c < nc) {
        double s = 0.0;
        for (int q = 0; q < nq; ++q) s += part[((long long)q * n16 + c) * ldp + ii];
        out[(long long)c * ld + i_begin + ii] = s;
    }
}
// first-use self-check: the largest |a - b| and |b| over rows [0, rows) of `cols` columns  ->  res[0], res[1] (one CTA)
__global__ void __launch_bounds__(THREADS)
gi_compare_kernel(const double* __restrict__ a, const double* __restrict__ b, long long ld, long long i_begin, long long rows, int cols,
                  double* __restrict__ res) {
    __shared__ double sd[THREADS], sv[THREADS];
    double d = 0.0, v = 0.0;
    for (int c = 0; c < cols; ++c)
        for (long long i = threadIdx.x; i < rows; i += THREADS) {
            const double x = a[(long long)c * ld + i_begin + i], y = b[(long long)c * ld + i_begin + i];
            d = fmax(d, fabs(x - y)); v = fmax(v, fabs(y));
            if (!(x == x)) d = 1e300;                      // NaN in the tensor-core result
        }
    sd[threadIdx.x] = d; sv[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < THREADS; ++t) { d = fmax(d, sd[t]); v = fmax(v, sv[t]); }
        res[0] = d; res[1] = v;
    }
}

// ---- the product -----------------------------------------------------------------------------------------------------------------
// one column pass: images = the stage images of gi_split_kernel (jpad / 32 of them); pts: float4 {a, 0} per point in the scaled frame
// of lr_pack_kernel, padded to jpad with far-away records (G == 0); rows [i_begin, i_end) of G;
// part[q][c][ii] (FP64) = colmax[c] 2^-45 sum_{j in chunk q} g_ij x_cj  for c < GI_N, ii < ldp (a multiple of GI_ROWS)
// KIND: the tile values of lr_kernel_value (lowrank.cuh); for LR_IMQ the epilogue scale also carries gscale = c^(-1/2).
template <int KIND>
__global__ void __launch_bounds__(GI_THREADS, 1)
gi_gram_kernel(const unsigned char* __restrict__ images, const float4* __restrict__ pts, long long jpad, int chunk, long long i_begin,
               long long i_end, const double* __restrict__ colmax, double* __restrict__ part, long long ldp, double gscale) {
    // 256-byte alignment anchors the 32-byte swizzle pattern of every B plane the way the MMA unit reads it
    extern __shared__ __align__(256) unsigned char gi_smem_raw[];
    unsigned char* planes = gi_smem_raw;                                      // [GI_STAGES][3][GI_PLANE]
    const float4* spts = reinterpret_cast<const float4*>(planes + GI_STAGES * 3 * GI_PLANE);     // [GI_STAGES][GI_KS]
    uint64_t* bars = reinterpret_cast<uint64_t*>(planes + GI_STAGES * (3 * GI_PLANE + GI_PTS_BYTES));
    uint64_t* full = bars;                     // [GI_STAGES]: the slot's bytes have landed
    uint64_t* empty = bars + GI_STAGES;        // [GI_STAGES]: every warp of every warpgroup is done with the slot

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long rows = i_end - i_begin;
    const int ntiles = (int)((rows + GI_ROWS - 1) / GI_ROWS);
    const int nq = (int)((jpad + chunk - 1) / chunk);
    const long long nunits = (long long)ntiles * nq;

    if (threadIdx.x == 0) {
        for (int s = 0; s < GI_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * GI_WG); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 4 * GI_WG) {
        // ===== producer: one bulk copy of the stage image (three digit planes of X) + one of the stage's j-points =====
        if (lane == 0) {
            uint32_t stage = 0, phase = 0;
            for (long long u = blockIdx.x; u < nunits; u += gridDim.x) {
                const int q = (int)(u / ntiles);
                const long long j0 = (long long)q * chunk;
                const int nst = (int)((min((long long)chunk, jpad - j0)) / GI_KS);
                const unsigned char* src = images + (j0 / GI_KS) * (3 * GI_PLANE);
                for (int kb = 0; kb < nst; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], (uint32_t)(3 * GI_PLANE + GI_PTS_BYTES));
                    tma_load_1d(planes + stage * 3 * GI_PLANE, src + (long long)kb * (3 * GI_PLANE), (uint32_t)(3 * GI_PLANE), &full[stage]);
                    tma_load_1d((void*)(spts + stage * GI_KS), pts + j0 + (long long)kb * GI_KS, (uint32_t)GI_PTS_BYTES, &full[stage]);
                    if (++stage == GI_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===== warpgroups: G tile -> A fragment, six MMAs per stage, epilogue per work unit =====
    // A fragment of m64k32 (8-bit): warp w of the warpgroup holds rows 16 w + lane / 4 (registers 0, 2) and + 8 (registers 1, 3);
    // register 0 / 1 carry k = 4 (lane % 4) .. + 3, registers 2 / 3 the same k + 16, lowest k in the lowest byte.
    // Accumulator fragment of m64n64: register 4 i + h (+ 2 for row + 8) is column 8 i + 2 (lane % 4) + h.
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);             // row of the tile; the other row is r0 + 8
    const int kq = (lane & 3) * 4;
    uint32_t stage = 0, phase = 0;
    for (long long u = blockIdx.x; u < nunits; u += gridDim.x) {
        const int q = (int)(u / ntiles), t = (int)(u % ntiles);
        const long long j0 = (long long)q * chunk;
        const int nst = (int)((min((long long)chunk, jpad - j0)) / GI_KS);
        float ax[2], ay[2], az[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            long long i = i_begin + (long long)t * GI_ROWS + r0 + 8 * h;
            if (i >= i_end) i = i_end - 1;                              // rows past the end: computed, never read back
            const float4 a = pts[i];
            ax[h] = a.x; ay[h] = a.y; az[h] = a.z;
        }
        int acc0[32] = {}, acc1[32] = {}, acc2[32] = {};
        for (int kb = 0; kb < nst; ++kb) {
            mbar_wait(&full[stage], phase);
            const float4* bj = spts + stage * GI_KS;
            // g = round(2^23 G) sits in the mantissa of 2^23 + 2^23 G (one FMA; a float -> integer conversion would go through the
            // quarter-rate pipe that MUFU.EX2 already loads): bytes 2, 1, 0 of the float ARE the digits a0 < 128, a1, a2.
            // gq[h][s]: row r0 + 8 h, point kq + s (s < 4) or 16 + kq + s - 4
            uint32_t gq[2][8];
#pragma unroll
            for (int s = 0; s < 8; ++s) {
                const float4 b = bj[(s < 4 ? 0 : 16) + kq + (s & 3)];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float dx = __fsub_rn(ax[h], b.x), dy = __fsub_rn(ay[h], b.y), dz = __fsub_rn(az[h], b.z);
                    const float uu = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
                    const float e = lr_kernel_value<KIND>(uu);  // the same float32 G as the other kernels; G = 1 gives the digits (128, 0, 0)
                    gq[h][s] = __float_as_uint(__fmaf_rn(e, 8388608.0f, 8388608.0f));
                }
            }
            uint32_t a[3][4];
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                const uint32_t sel = p == 0 ? 0x0062u : (p == 1 ? 0x0051u : 0x0040u);     // byte (2 - p) of both inputs
#pragma unroll
                for (int reg = 0; reg < 4; ++reg) {
                    const uint32_t* g = &gq[reg & 1][(reg >> 1) * 4];
                    a[p][reg] = __byte_perm(__byte_perm(g[0], g[1], sel), __byte_perm(g[2], g[3], sel), 0x5410u);
                }
            }
            const uint32_t sb = smem_u32(planes + stage * 3 * GI_PLANE);
            const uint64_t b0 = gi_smem_desc(sb), b1 = gi_smem_desc(sb + GI_PLANE), b2 = gi_smem_desc(sb + 2 * GI_PLANE);
            const int more = kb != 0;
            gi_wgmma_fence();
            gi_mma(acc0, a[0], b0, more);
            gi_mma(acc1, a[0], b1, more);
            gi_mma(acc1, a[1], b0, 1);
            gi_mma(acc2, a[0], b2, more);
            gi_mma(acc2, a[1], b1, 1);
            gi_mma(acc2, a[2], b0, 1);
            gi_wgmma_commit();
            gi_wgmma_wait_all();
            __syncwarp();
            if (lane == 0) gi_mbar_arrive(&empty[stage]);
            if (++stage == GI_STAGES) { stage = 0; phase ^= 1; }
        }
        // ===== epilogue: join the three levels in FP64 (exact), scale, store the chunk partial =====
        const long long ii = (long long)t * GI_ROWS + r0;
        double* dst = part + (long long)q * GI_N * ldp + ii;
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int c = 8 * i + 2 * (lane & 3) + h;
                double sc = colmax[c] * (1.0 / 536870912.0);                                       // 2^16 2^-45
                if constexpr (KIND == LR_IMQ) sc *= gscale;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int k = 4 * i + 2 * rr + h;
                    const double s = (double)acc0[k] * 65536.0 + (double)acc1[k] * 256.0 + (double)acc2[k];     // exact: < 2^48
                    dst[(long long)c * ldp + 8 * rr] = s * sc;
                }
            }
    }
}

}  // namespace cpd
#endif  // CPD_HOST_EMU
