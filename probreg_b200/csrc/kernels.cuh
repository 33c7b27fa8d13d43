// kernels.cuh -- sm_90a (H100) device code of the CPD EM hot path.
//
// What is computed (reference: probreg/cpd.py:71-88, restated in oracle/cpd_oracle.py):
//   K_mn = exp(-|yhat_m - x_n|^2 / (2 sigma^2)),  den_n = sum_m K_mn (+ eps32 if 0) + c,
//   P = K / den,  pt1_n = sum_m P_mn,  p1_m = sum_n P_mn,  px_m = sum_n P_mn x_n.
// How: two tiled passes over the M x N pair space that never store P.
//   pass 1  (i = targets in registers, j = sources streamed through shared memory by TMA bulk
//            copies): per target an integer offset o and FP64 sums S, SU with
//              sum_m 2^(-u_mn) = S 2^(-o),   sum_m 2^(-u_mn) u_mn = SU 2^(-o)
//            -- a lazily rebased log-sum-exp that also yields the weighted squared residual.
//   pass 2  (i = sources in registers, j = targets streamed): K = 2^(o_n - u) recomputed with the
//            SAME integer offset (so MUFU.EX2 sees the same fractional argument as in pass 1 and
//            its approximation error cancels in K / sum K), P = K * rn_n, and per source
//            p1_m = sum_n P and the RESIDUAL sum  sd_m = sum_n P (a_m - b_n)  -- not sum_n P b_n.
// u_mn = |a_m - b_n|^2 where a, b are the two clouds centred on a common origin and scaled by
// sqrt(log2(e) / (2 sigma^2)), so that exp(-d^2/2sigma^2) == 2^(-u): one MUFU.EX2 per pair and
// no multiply by 1/(2 sigma^2).  Pair arithmetic is FP32 on direct differences (never the
// |a|^2+|b|^2-2ab expansion, which cancels catastrophically once sigma << extent); every
// accumulation that crosses a 64-point sub-chunk is FP64.
//
// Why residual sums: the reference's M-step forms sigma2 = (tr_xp1x - s tr_atr)/(Np D), a
// difference of two sums that agree to extent^2/(3 sigma^2) -- 40x on the bunny after ten
// iterations, >1e4x near convergence.  FP64 P (the reference) survives that; FP32-accurate P does
// not (measured: 5e-6 relative on sigma2).  Accumulating P*(a-b) and P*u instead gives the same
// M-step as an UPDATE of the previous transform (mstep_solve_residual) in which every large term
// is formed in FP64 from p1 alone and the FP32-accurate sums only enter through small quantities.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cpd {

// tunables (tools/tune.sh builds variants with -D...; the defaults are not tuned for the H100)
#ifndef CPD_RI1
#define CPD_RI1 4
#endif
#ifndef CPD_RI2
#define CPD_RI2 4
#endif
#ifndef CPD_MINB1
#define CPD_MINB1 2
#endif
#ifndef CPD_MINB2
#define CPD_MINB2 2
#endif
#ifndef CPD_UNROLL1
#define CPD_UNROLL1 4
#endif
#ifndef CPD_UNROLL2
#define CPD_UNROLL2 4
#endif
#ifndef CPD_SUB
#define CPD_SUB 64
#endif
#ifndef CPD_GRP
#define CPD_GRP 8
#endif
constexpr int UNROLL1 = CPD_UNROLL1, UNROLL2 = CPD_UNROLL2;
constexpr int THREADS = 256;           // threads per CTA in both passes
constexpr int RI1 = CPD_RI1, RI2 = CPD_RI2;            // i-points held in registers per thread (pass 1 / pass 2)
constexpr int ITILE1 = THREADS * RI1, ITILE2 = THREADS * RI2;   // i-points per CTA
constexpr int NPAIR1 = RI1 / 2, NPAIR2 = RI2 / 2;      // i-points are processed in pairs (fsub2 / ffma2 below)
#ifndef CPD_P1_STAGE
#define CPD_P1_STAGE 512
#endif
#ifndef CPD_P2_STAGE
#define CPD_P2_STAGE 512
#endif
constexpr int P1_STAGE = CPD_P1_STAGE;   // sources per TMA stage in pass 1 (32 B records -> 16 KB); a multiple of 256
constexpr int P2_STAGE = CPD_P2_STAGE;   // targets per TMA stage in pass 2 (48 B records -> 24 KB); a multiple of 256
static_assert(P1_STAGE % 256 == 0 && P2_STAGE % 256 == 0 && P1_STAGE >= 256 && P2_STAGE >= 256, "stage sizes are multiples of 256");
constexpr int P1_REC = 32, P2_REC = 48;    // bytes per streamed j-record (coordinates duplicated for the pair loops)
#ifndef CPD_NSTAGE
#define CPD_NSTAGE 3
#endif
constexpr int NSTAGE = CPD_NSTAGE;     // TMA pipeline depth
constexpr int P1_STAGE_BYTES = P1_STAGE * P1_REC, P2_STAGE_BYTES = P2_STAGE * P2_REC;
constexpr int SUB = CPD_SUB;           // j-points between offset checks / FP64 flushes
constexpr int GRP = CPD_GRP;           // j-points summed from zero before joining the sub-chunk sum (0: off)
constexpr int PASS1_SMEM = NSTAGE * P1_STAGE_BYTES + 64, PASS2_SMEM = NSTAGE * P2_STAGE_BYTES + 64;

// dynamic shared memory of the running CTA (the CPU test build of tests/emu substitutes its own buffer)
#ifdef CPD_HOST_EMU
#define CPD_DYN_SMEM(name) unsigned char* const name = emu::g_dyn_smem
#else
#define CPD_DYN_SMEM(name) extern __shared__ __align__(128) unsigned char name[]
#endif

constexpr float O_INIT = 1048576.0f;   // 2^20: "no source seen yet" offset; u above it is dead anyway
constexpr float TWO100 = 1.2676506002282294e30f;
constexpr float FAR_COORD = 1.0e18f;   // padding sources: u = 3e36, 2^(o-u) == 0

constexpr double LOG2E = 1.4426950408889634074;
constexpr double DEAD_LOG2 = -1075.0;  // float64 exp(x) == 0  <=>  x*log2(e) < -1075 (half the least denormal)
constexpr double EPS32 = 1.1920928955078125e-07;

// Moments of the fused EM loop (residual form, all-reduced across ranks):
//   source side, per block of finalize2:  Np, Sy = sum p1 y~, C = sum p1 y~ y~^T (6), V1 = sum v, VY = sum v y~^T (9)
//   target side, per block of finalize1:  Srr = sum_n sum_m P_mn u_mn (scaled units), Npt = sum pt1
// with v_m = sum_n P_mn (x_n - T(y_m)) the weighted residual of source m and y~ = y - cy.
enum { RM_NP = 0, RM_SY = 1, RM_C = 4, RM_V1 = 10, RM_VY = 13, RM_SRC = 22, RM_SRR = 22, RM_NPT = 23, RM_TGT = 2,
       RM_COUNT = 24, MOM_PAD = 32 };
// Moments of the API-faithful M-step (cpd_mstep: a caller-supplied EstepResult;
// the reference's sums extended with the pt1-side sums the reference uses)
enum { MOM_NP = 0, MOM_SX = 1, MOM_SY = 4, MOM_B = 7, MOM_C = 16, MOM_NPT = 22, MOM_SXT = 23, MOM_TXX = 26,
       MOM_COUNT = 27, MOM_SRC = 22, MOM_TGT = 5 };

// per-split, per-target result of pass 1
struct P1Part {
    double S;    // sum_m 2^(o - u)
    double SU;   // sum_m 2^(o - u) u
    float o;     // integer-valued offset
    float pad;
};

// Device-resident EM state.  The first 16 doubles mirror cpd_params.
struct DevState {
    double lin[9];
    double t[3];
    double scale;
    double sigma2;
    double q;
    double n_p;
    double cx[3];        // frame origin of the targets (and of the distance frame)
    double cy[3];        // centroid the sources are centred on for the moments
    double w;
    double es_sigma2;    // inputs of a stand-alone cpd_estep call
    double es_w;
    long long m;
    long long n_global;
    int tf_kind;
    int update_scale;
    int dim;
    int err;             // set by a kernel that gave up waiting for a peer (P2P exchange); checked by the host
};

// One-shot all-reduce of the 32 moment doubles over NVLink peer memory: every rank owns
// a mailbox that its peers write into; slots are double-buffered by exchange parity, flags carry the
// exchange sequence number (monotonic, never reset), sums are formed in rank order => bit-identical on all ranks.
constexpr int P2P_MAX = 16;
struct P2PMailbox {
    double slots[2][P2P_MAX][MOM_PAD];
    unsigned long long flags[2][P2P_MAX];
};
struct P2PInfo {
    P2PMailbox* box[P2P_MAX];     // box[r]: rank r's mailbox mapped into this process (box[rank] is local memory)
    int world, rank;
    unsigned long long seq;       // exchanges completed
    unsigned long long timeout_ns;   // how long a rank waits for its peers' moments (wall clock, %globaltimer); see cpd_p2p_attach
};

// ---------------------------------------------------------------------------------------------
// small PTX helpers
// ---------------------------------------------------------------------------------------------
#ifdef CPD_HOST_EMU
}  // namespace cpd
#include "emu_device.h"   // tests/emu: host stand-ins for the inline-PTX helpers below (CPU test build only)
namespace cpd {
#else
__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// FP32 pairs: two i-points travel together through the pair loops (one 64-bit register pair, one 8-byte shared-memory load
// per j-coordinate for both).  Hopper has no packed FP32 instructions, so each helper is two scalar IEEE operations with the
// rounding of the corresponding f32x2 instruction (the _rn intrinsics also keep the compiler from contracting them).
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ float2 unpack2(u64 v) { float2 r; asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v)); return r; }
__device__ __forceinline__ u64 fsub2(u64 a, u64 b) {
    const float2 x = unpack2(a), y = unpack2(b);
    return pack2(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y));
}
__device__ __forceinline__ u64 fadd2(u64 a, u64 b) {
    const float2 x = unpack2(a), y = unpack2(b);
    return pack2(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ u64 fmul2(u64 a, u64 b) {
    const float2 x = unpack2(a), y = unpack2(b);
    return pack2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ u64 ffma2(u64 a, u64 b, u64 c) {
    const float2 x = unpack2(a), y = unpack2(b), z = unpack2(c);
    return pack2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
#endif  // CPD_HOST_EMU
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Fixed-order block reduction of K doubles per thread; the block's K sums go to out[0..K).
template <int K>
__device__ __forceinline__ void block_reduce_store(double (&v)[K], double* out) {
    __shared__ double sh[K][THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double s = warp_sum(v[k]);
        if (lane == 0) sh[k][wid] = s;
    }
    __syncthreads();
    if (threadIdx.x < K) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < THREADS / 32; ++w) s += sh[threadIdx.x][w];
        out[threadIdx.x] = s;
    }
}

// ---------------------------------------------------------------------------------------------
// pack: transform + centre + scale both clouds into the FP32 working frame
//   a_m = sk * (lin_eff * (y_m - cy) + t')   with t' = lin_eff*cy + t - cx     (sources)
//   b_n = sk * (x_n - cx)                                                      (targets)
//   sk = sqrt(log2(e) / (2 sigma^2)).  One FP64 evaluation, one rounding to FP32.
// Reference: Transformation.transform (transformation.py:49-50 / 77-78) fused with the
// 1/(2 sigma^2) scaling of cpd.py:76.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS)
pack_kernel(const DevState* __restrict__ st, const double* __restrict__ sigma2_ptr,
            const double* __restrict__ yc /* m x 3 centred sources */, const double* __restrict__ ts /* explicit transformed sources or null */,
            const double* __restrict__ xc /* n x 3 centred targets */, long long m, long long mpad, long long n,
            float4* __restrict__ srcP /* i-points of pass 2 */, float4* __restrict__ srcJ /* j-records of pass 1: {x,x,y,y},{z,z,0,0} */,
            float4* __restrict__ tgtP /* i-points of pass 1 */) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    const double sk = sqrt(LOG2E / (2.0 * *sigma2_ptr));
    if (i < mpad) {
        float4 o;
        if (i < m) {
            double px, py, pz;
            if (ts != nullptr) {
                px = ts[3 * i + 0] - st->cx[0];
                py = ts[3 * i + 1] - st->cx[1];
                pz = ts[3 * i + 2] - st->cx[2];
            } else {
                const double s = (st->tf_kind == 0) ? st->scale : 1.0;
                double l[9], tp[3];
#pragma unroll
                for (int k = 0; k < 9; ++k) l[k] = s * st->lin[k];
#pragma unroll
                for (int a = 0; a < 3; ++a)
                    tp[a] = l[3 * a] * st->cy[0] + l[3 * a + 1] * st->cy[1] + l[3 * a + 2] * st->cy[2] + st->t[a] - st->cx[a];
                const double y0 = yc[3 * i], y1 = yc[3 * i + 1], y2 = yc[3 * i + 2];
                px = l[0] * y0 + l[1] * y1 + l[2] * y2 + tp[0];
                py = l[3] * y0 + l[4] * y1 + l[5] * y2 + tp[1];
                pz = l[6] * y0 + l[7] * y1 + l[8] * y2 + tp[2];
            }
            o = make_float4((float)(sk * px), (float)(sk * py), (float)(sk * pz), 0.0f);
        } else {
            o = make_float4(FAR_COORD, FAR_COORD, FAR_COORD, 0.0f);
        }
        srcP[i] = o;
        srcJ[2 * i] = make_float4(o.x, o.x, o.y, o.y);
        srcJ[2 * i + 1] = make_float4(o.z, o.z, 0.0f, 0.0f);
    }
    if (i < n) {
        tgtP[i] = make_float4((float)(sk * xc[3 * i]), (float)(sk * xc[3 * i + 1]), (float)(sk * xc[3 * i + 2]), 0.0f);
    }
}

// Per-source weights of a weighted E-step (BCPD): la_m = -log2(weight_m) - min(...) >= 0 goes into the spare lanes of the
// records pack_kernel wrote: srcP[m].w (pass 2 i-points) and srcJ[2m+1].zw (pass 1 j-records).  Padding keeps 0.
__global__ void __launch_bounds__(THREADS)
weight_patch_kernel(const float* __restrict__ la, long long m, float4* __restrict__ srcP, float4* __restrict__ srcJ) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const float v = la[i];
        srcP[i].w = v;
        float4 r = srcJ[2 * i + 1];
        r.z = v; r.w = v;
        srcJ[2 * i + 1] = r;
    }
}

// ---------------------------------------------------------------------------------------------
// pass 1: per target n and split:  (o, S, SU) with  sum_m 2^(-u) = S 2^(-o),  sum_m 2^(-u) u = SU 2^(-o)
// One CTA per work item {target tile, source-stage range, partial slot}; the host chooses the number of stage
// ranges per tile that minimises the makespan over the resident CTA slots (build_work in cpd_b200.cu).
// Per two pairs: 8 packed FP32 instructions + 2 MUFU in the common path.
//
// Lazy log-sum-exp: each target carries an integer-valued offset o (only ever lowered), seeded per warp from
// the nearest source stage.  A sub-chunk of 64 sources is summed in FP32 with the current o -- groups of 8 from
// zero, the 8 group sums joined (pass1_sum): Sc = sum e, Uc = sum e*t' with t' = u - o, e = 2^-t' -- and folded
// into the FP64 running sums (S += Sc, SU += Uc + o*Sc).  If any lane's sub-chunk sum reaches 2^100 (a source much
// nearer than any seen before: 2^(o-u) overflowed or nearly did) the warp re-does that sub-chunk: one sweep for
// the sub-chunk minimum of u, o := min(o, floor(umin)), S and SU rescaled by the exact power of two, sub-chunk
// summed again.  The largest term of a target is >= 2^-1 right after its offset was set and <= 2^100 always,
// so every term that matters stays a normal FP32 number.
// ---------------------------------------------------------------------------------------------
// ---------------------------------------------------------------------------------------------
// Exact culling of far (warp, stage) blocks.  ex2.approx.ftz returns exactly 0 below 2^-126, so a block of
// pairs whose every t' = u - o exceeds ~127 contributes exactly nothing to any sum: skipping it is bit-identical
// to evaluating it.  With Z-ordered clouds both a warp's i-points and a 512-record j-stage are spatially
// compact, so  dist^2(bbox_warp, bbox_stage) - max(o)  >= CULL_GAP  proves that cheaply.  It only ever
// triggers once sigma << extent (late iterations: 13 sigma is the reach of a point), which is when the dense
// sweep wastes most of its work; the host enables it only then (cpd_em_step).
// ---------------------------------------------------------------------------------------------
constexpr float CULL_GAP = 130.0f;
// per block of `blk` consecutive points: {min xyz, 0}, {max xyz, 0}
__global__ void __launch_bounds__(THREADS)
stage_bbox_kernel(const float4* __restrict__ pts, int n, int blk, float4* __restrict__ box) {
    __shared__ float sh[6][THREADS / 32];
    const int b = blockIdx.x;
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    for (int i = b * blk + threadIdx.x; i < min(n, (b + 1) * blk); i += THREADS) {
        const float4 p = pts[i];
        lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
        hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
        if (lane == 0) { sh[a][wid] = lo[a]; sh[3 + a][wid] = hi[a]; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float l[3], h[3];
        for (int a = 0; a < 3; ++a) {
            l[a] = sh[a][0]; h[a] = sh[3 + a][0];
            for (int w = 1; w < THREADS / 32; ++w) { l[a] = fminf(l[a], sh[a][w]); h[a] = fmaxf(h[a], sh[3 + a][w]); }
        }
        box[2 * b] = make_float4(l[0], l[1], l[2], 0.f);
        box[2 * b + 1] = make_float4(h[0], h[1], h[2], 0.f);
    }
}
// per pass-2 stage: the largest offset o_n of its live targets (records hold -o; dead / padding hold +inf)
__global__ void __launch_bounds__(THREADS)
stage_omax_kernel(const float4* __restrict__ tgtQ, float* __restrict__ omax) {
    __shared__ float sh[THREADS / 32];
    const int b = blockIdx.x;
    float m = 3.0e38f;
    for (int i = threadIdx.x; i < P2_STAGE; i += THREADS) m = fminf(m, tgtQ[3 * ((size_t)b * P2_STAGE + i) + 1].z);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < THREADS / 32; ++w) m = fminf(m, sh[w]);
        omax[b] = -m;                                   // -inf when the whole stage is dead
    }
}
// the same two quantities per 64-record sub-chunk (one warp each): the second, finer level of the culling test
__global__ void __launch_bounds__(THREADS)
sub_bbox_kernel(const float4* __restrict__ pts, int n, int nsub, float4* __restrict__ box) {
    const int b = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= nsub) return;
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
    for (int i = b * SUB + lane; i < min(n, (b + 1) * SUB); i += 32) {
        const float4 p = pts[i];
        lo[0] = fminf(lo[0], p.x); lo[1] = fminf(lo[1], p.y); lo[2] = fminf(lo[2], p.z);
        hi[0] = fmaxf(hi[0], p.x); hi[1] = fmaxf(hi[1], p.y); hi[2] = fmaxf(hi[2], p.z);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if (lane == 0) {
        box[2 * b] = make_float4(lo[0], lo[1], lo[2], 0.f);
        box[2 * b + 1] = make_float4(hi[0], hi[1], hi[2], 0.f);
    }
}
__global__ void __launch_bounds__(THREADS)
sub_omax_kernel(const float4* __restrict__ tgtQ, int nsub, float* __restrict__ omax) {
    const int b = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= nsub) return;
    float m = 3.0e38f;
    for (int i = lane; i < SUB; i += 32) m = fminf(m, tgtQ[3 * ((size_t)b * SUB + i) + 1].z);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) omax[b] = -m;
}
// bounding box of this warp's packed i-points -> wbox[0..6) (shared, one row per warp)
template <int NP>
__device__ __forceinline__ void warp_bbox(const u64 (&ax)[NP], const u64 (&ay)[NP], const u64 (&az)[NP], float* __restrict__ wbox) {
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        const float2 x = unpack2(ax[p]), y = unpack2(ay[p]), z = unpack2(az[p]);
        lo[0] = fminf(lo[0], fminf(x.x, x.y)); hi[0] = fmaxf(hi[0], fmaxf(x.x, x.y));
        lo[1] = fminf(lo[1], fminf(y.x, y.y)); hi[1] = fmaxf(hi[1], fmaxf(y.x, y.y));
        lo[2] = fminf(lo[2], fminf(z.x, z.y)); hi[2] = fmaxf(hi[2], fmaxf(z.x, z.y));
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
            hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int a = 0; a < 3; ++a) { wbox[a] = lo[a]; wbox[3 + a] = hi[a]; }
    }
    __syncwarp();
}
__device__ __forceinline__ float box_gap2(const float* __restrict__ wbox, const float4 blo, const float4 bhi) {
    const float gx = fmaxf(0.f, fmaxf(blo.x - wbox[3], wbox[0] - bhi.x));
    const float gy = fmaxf(0.f, fmaxf(blo.y - wbox[4], wbox[1] - bhi.y));
    const float gz = fmaxf(0.f, fmaxf(blo.z - wbox[5], wbox[2] - bhi.z));
    return fmaf(gz, gz, fmaf(gy, gy, gx * gx)) * 0.9999f;      // a whisker below the true lower bound of u
}

// Sum one sub-chunk of pass 1 into Sc (sum e) and Uc (sum e*t'), both starting from zero.  With GRP > 0 the
// terms are first summed in groups of GRP from zero and the group sums joined: a two-level FP32 summation.
// Why: adding thousands of tiny terms one by one to a partial sum that already holds a dominant term drops
// them (absorption), a SYSTEMATIC loss that does not average out -- measured -1.2e-6 on sigma2 with a flat
// 64-term sum, -2e-6 with 128.
// WGT: every source carries a weight 2^-la (la >= 0) in the spare half of its z-record; t' = u - o + la, added LAST so that
// pass 2 (which adds the same la after the same FMA chain) sees bit-identical exponents (the BCPD E-step, bcpd.py:53-66).
template <bool WGT>
__device__ __forceinline__ void pass1_sum(const ulonglong2* __restrict__ q, const u64 (&ax)[NPAIR1], const u64 (&ay)[NPAIR1],
                                          const u64 (&az)[NPAIR1], const u64 (&no)[NPAIR1], u64 (&Sc)[NPAIR1], u64 (&Uc)[NPAIR1]) {
    if (GRP > 0) {
#pragma unroll 1
        for (int g0 = 0; g0 < SUB; g0 += (GRP > 0 ? GRP : SUB)) {
            u64 gs[NPAIR1], gu[NPAIR1];
#pragma unroll
            for (int jj = 0; jj < (GRP > 0 ? GRP : 1); ++jj) {
                const ulonglong2 bxy = q[2 * (g0 + jj)];
                const u64 bz = q[2 * (g0 + jj) + 1].x;
                u64 la = 0ull;
                if (WGT) la = q[2 * (g0 + jj) + 1].y;
#pragma unroll
                for (int p = 0; p < NPAIR1; ++p) {
                    const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bz);
                    u64 t = ffma2(dx, dx, no[p]);
                    t = ffma2(dy, dy, t);
                    t = ffma2(dz, dz, t);
                    if (WGT) t = fadd2(t, la);
                    const float2 tt = unpack2(t);
                    const u64 e = pack2(ex2(-tt.x), ex2(-tt.y));
                    gs[p] = jj == 0 ? e : fadd2(gs[p], e);
                    gu[p] = jj == 0 ? fmul2(e, t) : ffma2(e, t, gu[p]);
                }
            }
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) { Sc[p] = fadd2(Sc[p], gs[p]); Uc[p] = fadd2(Uc[p], gu[p]); }
        }
    } else {
#pragma unroll UNROLL1
        for (int jj = 0; jj < SUB; ++jj) {
            const ulonglong2 bxy = q[2 * jj];
            const u64 bz = q[2 * jj + 1].x;
            u64 la = 0ull;
            if (WGT) la = q[2 * jj + 1].y;
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) {
                const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bz);
                u64 t = ffma2(dx, dx, no[p]);
                t = ffma2(dy, dy, t);
                t = ffma2(dz, dz, t);
                if (WGT) t = fadd2(t, la);
                const float2 tt = unpack2(t);
                const u64 e = pack2(ex2(-tt.x), ex2(-tt.y));
                Sc[p] = fadd2(Sc[p], e);
                Uc[p] = ffma2(e, t, Uc[p]);
            }
        }
    }
}

template <bool CULL, bool WGT>
__global__ void __launch_bounds__(THREADS, CPD_MINB1)
pass1_kernel(const float4* __restrict__ ipts, int ni, const float4* __restrict__ jrec, const int4* __restrict__ work,
             P1Part* __restrict__ part, const float4* __restrict__ sbox /* bounding boxes of the source stages */,
             int nstages_total, const float4* __restrict__ ssub /* ... and of their 64-record sub-chunks (CULL only) */) {
    __shared__ float wbox[THREADS / 32][8];
    CPD_DYN_SMEM(smraw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smraw + NSTAGE * P1_STAGE_BYTES);
    const int tid = threadIdx.x;
    const int4 wk = work[blockIdx.x];               // {i-tile, first sub-chunk, end sub-chunk, partial slot}: see build_work()
    constexpr int SPS = P1_STAGE / SUB;             // an item may begin and end inside a stage: whole stages are loaded,
    const int itile = wk.x, split = wk.w;           // the sub-chunks outside the item are skipped
    const int st0 = wk.y / SPS, nst = (wk.z + SPS - 1) / SPS - st0;
    const int sc_first = wk.y - st0 * SPS, sc_last = wk.z - (st0 + nst - 1) * SPS;
    const unsigned char* jbytes = reinterpret_cast<const unsigned char*>(jrec);
    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 0; s < NSTAGE && s < nst; ++s) {
            mbar_expect_tx(&full[s], P1_STAGE_BYTES);
            tma_load_1d(smraw + s * P1_STAGE_BYTES, jbytes + (size_t)(st0 + s) * P1_STAGE_BYTES, P1_STAGE_BYTES, &full[s]);
        }
    }
    // A warp whose i-points are all padding (the tail of the last tile) has nothing to add: it leaves before the stage loop, whose
    // barriers then count the remaining warps only (warp 0, the TMA issuer, always has i-points); build_work() gives such a tile
    // correspondingly longer items.
    if (itile * ITILE1 + (tid >> 5) * (32 * RI1) >= ni) return;
    // two packed pairs of targets per thread: pair p = targets (2p, 2p+1) of this thread
    u64 ax[NPAIR1], ay[NPAIR1], az[NPAIR1], no[NPAIR1];    // no = (-o, -o'): negated integer offsets
    double S[RI1], SU[RI1];
#pragma unroll
    for (int p = 0; p < NPAIR1; ++p) {
        // a warp owns 32*RI1 CONSECUTIVE (Z-ordered) targets: compact for the culling test, still coalesced per 32
        int n0 = itile * ITILE1 + (tid >> 5) * (32 * RI1) + (2 * p) * 32 + (tid & 31), n1 = n0 + 32;
        n0 = n0 < ni ? n0 : ni - 1;
        n1 = n1 < ni ? n1 : ni - 1;
        const float4 p0 = ipts[n0], p1 = ipts[n1];
        ax[p] = pack2(p0.x, p1.x); ay[p] = pack2(p0.y, p1.y); az[p] = pack2(p0.z, p1.z);
        no[p] = pack2(-O_INIT, -O_INIT);
    }
    // Seed the offsets from the source stage whose bounding box is nearest to this warp's targets (any source
    // gives a valid upper bound of the final offset; a near one gives a tight bound).  With tight seeds the
    // offset slow path below becomes rare even when sigma << extent, and the culling test bites from the first
    // stage on.  Cost: one scan of the stage boxes + one 128-source sweep per warp.
    float* const mybox = wbox[tid >> 5];
    warp_bbox<NPAIR1>(ax, ay, az, mybox);
    {
        const int lane = tid & 31;
        float best = 3.0e38f;
        int bi = 0;
        for (int sidx = lane; sidx < nstages_total; sidx += 32) {
            const float g2 = box_gap2(mybox, sbox[2 * sidx], sbox[2 * sidx + 1]);
            if (g2 < best) { best = g2; bi = sidx; }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        const ulonglong2* near = reinterpret_cast<const ulonglong2*>(jbytes + (size_t)bi * P1_STAGE_BYTES);
        float cm[RI1];
#pragma unroll
        for (int r = 0; r < RI1; ++r) cm[r] = 3.0e38f;
#pragma unroll 4
        for (int jj = 0; jj < 128; ++jj) {
            const ulonglong2 bxy = near[2 * jj];
            const u64 bz = near[2 * jj + 1].x;
            u64 la = 0ull;
            if (WGT) la = near[2 * jj + 1].y;
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) {
                const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bz);
                u64 uu = ffma2(dz, dz, ffma2(dy, dy, fmul2(dx, dx)));
                if (WGT) uu = fadd2(uu, la);
                const float2 u = unpack2(uu);
                cm[2 * p] = fminf(cm[2 * p], u.x);
                cm[2 * p + 1] = fminf(cm[2 * p + 1], u.y);
            }
        }
#pragma unroll
        for (int p = 0; p < NPAIR1; ++p)
            no[p] = pack2(-fminf(O_INIT, floorf(cm[2 * p])), -fminf(O_INIT, floorf(cm[2 * p + 1])));
    }
    float omax_w = O_INIT;            // warp-uniform upper bound of this warp's offsets (culling test)
    if (CULL) {
        float om = -3.0e38f;
#pragma unroll
        for (int p = 0; p < NPAIR1; ++p) { const float2 nv = unpack2(no[p]); om = fmaxf(om, fmaxf(-nv.x, -nv.y)); }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) om = fmaxf(om, __shfl_xor_sync(0xffffffffu, om, o));
        omax_w = om;
    }
#pragma unroll
    for (int r = 0; r < RI1; ++r) { S[r] = 0.0; SU[r] = 0.0; }
    for (int it = 0; it < nst; ++it) {
        const int s = it % NSTAGE;
        mbar_wait(&full[s], (uint32_t)((it / NSTAGE) & 1));
        const ulonglong2* sp = reinterpret_cast<const ulonglong2*>(smraw + s * P1_STAGE_BYTES);
        bool skip = false;
        if (CULL) {      // every pair of (this warp, this stage) has t' = u - o >= CULL_GAP: exactly zero terms
            const float4 blo = sbox[2 * (st0 + it)], bhi = sbox[2 * (st0 + it) + 1];
            skip = box_gap2(mybox, blo, bhi) - omax_w >= CULL_GAP;
        }
#pragma unroll 1
        for (int sc = (it == 0 ? sc_first : 0); sc < (skip ? 0 : (it == nst - 1 ? sc_last : SPS)); ++sc) {
            if (CULL) {
                const int sb = (st0 + it) * (P1_STAGE / SUB) + sc;
                if (box_gap2(mybox, ssub[2 * sb], ssub[2 * sb + 1]) - omax_w >= CULL_GAP) continue;
            }
            const ulonglong2* q = sp + sc * (2 * SUB);
            u64 Sc[NPAIR1], Uc[NPAIR1];          // Sc = sum e,  Uc = sum e * t'  with t' = u - o, e = 2^-t'
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) { Sc[p] = 0ull; Uc[p] = 0ull; }
            pass1_sum<WGT>(q, ax, ay, az, no, Sc, Uc);
            bool bad = false;
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) {
                const float2 v = unpack2(Sc[p]);
                bad |= !(v.x < TWO100) | !(v.y < TWO100);
            }
            if (__any_sync(0xffffffffu, bad)) {
                float cm[RI1];
#pragma unroll
                for (int r = 0; r < RI1; ++r) cm[r] = 3.0e38f;
#pragma unroll UNROLL1
                for (int jj = 0; jj < SUB; ++jj) {
                    const ulonglong2 bxy = q[2 * jj];
                    const u64 bz = q[2 * jj + 1].x;
                    u64 la = 0ull;
                    if (WGT) la = q[2 * jj + 1].y;
#pragma unroll
                    for (int p = 0; p < NPAIR1; ++p) {
                        const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bz);
                        u64 uu = ffma2(dz, dz, ffma2(dy, dy, fmul2(dx, dx)));
                        if (WGT) uu = fadd2(uu, la);
                        const float2 u = unpack2(uu);
                        cm[2 * p] = fminf(cm[2 * p], u.x);
                        cm[2 * p + 1] = fminf(cm[2 * p + 1], u.y);
                    }
                }
#pragma unroll
                for (int p = 0; p < NPAIR1; ++p) {
                    const float2 nv = unpack2(no[p]);
                    const float o0 = -nv.x, o1 = -nv.y;
                    const float on0 = fminf(o0, floorf(cm[2 * p])), on1 = fminf(o1, floorf(cm[2 * p + 1]));
                    const int sh0 = (int)fmaxf(on0 - o0, -4000.0f), sh1 = (int)fmaxf(on1 - o1, -4000.0f);
                    S[2 * p] = ldexp(S[2 * p], sh0); SU[2 * p] = ldexp(SU[2 * p], sh0);
                    S[2 * p + 1] = ldexp(S[2 * p + 1], sh1); SU[2 * p + 1] = ldexp(SU[2 * p + 1], sh1);
                    no[p] = pack2(-on0, -on1);
                    Sc[p] = 0ull; Uc[p] = 0ull;
                }
                if (CULL) {      // the offsets just dropped: tighten the warp's bound for the culling test
                    float om = -3.0e38f;
#pragma unroll
                    for (int p = 0; p < NPAIR1; ++p) { const float2 nv = unpack2(no[p]); om = fmaxf(om, fmaxf(-nv.x, -nv.y)); }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) om = fmaxf(om, __shfl_xor_sync(0xffffffffu, om, o));
                    omax_w = om;
                }
                pass1_sum<WGT>(q, ax, ay, az, no, Sc, Uc);
            }
#pragma unroll
            for (int p = 0; p < NPAIR1; ++p) {
                const float2 sv = unpack2(Sc[p]), uv = unpack2(Uc[p]), nv = unpack2(no[p]);
                S[2 * p] += (double)sv.x;
                S[2 * p + 1] += (double)sv.y;
                SU[2 * p] += (double)uv.x - (double)nv.x * (double)sv.x;         // sum e*u = sum e*t' + o * sum e
                SU[2 * p + 1] += (double)uv.y - (double)nv.y * (double)sv.y;
            }
        }
        __syncthreads();
        if (tid == 0 && it + NSTAGE < nst) {
            mbar_expect_tx(&full[s], P1_STAGE_BYTES);
            tma_load_1d(smraw + s * P1_STAGE_BYTES, jbytes + (size_t)(st0 + it + NSTAGE) * P1_STAGE_BYTES, P1_STAGE_BYTES, &full[s]);
        }
    }
#pragma unroll
    for (int p = 0; p < NPAIR1; ++p) {
        const float2 nv = unpack2(no[p]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = itile * ITILE1 + (tid >> 5) * (32 * RI1) + (2 * p + h) * 32 + (tid & 31);
            if (n < ni) {
                P1Part out;
                out.S = S[2 * p + h]; out.SU = SU[2 * p + h]; out.o = h ? -nv.y : -nv.x; out.pad = 0.0f;
                part[(size_t)split * ni + n] = out;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// finalize 1: merge the per-split sums, apply the reference's column semantics, emit pt1 and the
// pass-2 target records.
//   omin   = smallest offset of any split that saw something; S, SU rebased to it (exact)
//   log2S  = log2 sum_m K_mn = log2(S) - omin                                  (FP64)
//   dead   = log2S < -1075  -> the float64 column sum of the reference is exactly 0 (cpd.py:81:
//            den = eps32 + c, every K_mn == 0, so P == 0 and pt1 == 0)
//   L      = log2(den) = log2(2^log2S + c)          c = (2 pi s2)^(D/2) w/(1-w) M/N  (cpd.py:78-79)
//   pt1    = 2^(log2S - L)                          (cpd.py:85; == 1 when w == 0)
//   rn     = 2^(-omin) / den = 2^-(L + omin)        P_mn = 2^(omin - u_mn) * rn in pass 2
//   record = {bx,bx,by,by},{bz,bz,-omin,-omin},{rn,rn,0,0}   (48 B, duplicated for the pair inner loop)
//            dead / padding: -omin = +inf (so 2^-(u - omin) == 0), rn = 0
// and the target-side moments: Srr = sum_n SU_n rn_n (= sum_mn P_mn u_mn), Npt = sum pt1.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS)
finalize1_kernel(const DevState* __restrict__ st, const double* __restrict__ sigma2_ptr, const double* __restrict__ w_ptr,
                 const P1Part* __restrict__ part, const int* __restrict__ tile_slots, int n, const float4* __restrict__ tgtP,
                 float4* __restrict__ tgtQ, long long npad, double* __restrict__ pt1, double* __restrict__ mom_part,
                 const double* __restrict__ log2c_ptr /* null: c from w (cpd.py:79); else log2 of the constant added to sum_m K (BCPD) */) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    double v[RM_TGT] = {0.0, 0.0};
    if (i < n) {
        const int nsplit = tile_slots[i / ITILE1];          // how many CTAs contributed a partial for this tile
        float omin = 3.0e38f;
        for (int s = 0; s < nsplit; ++s) {
            const P1Part p = part[(size_t)s * n + i];
            if (p.S > 0.0) omin = fminf(omin, p.o);
        }
        double log2S = -INFINITY, SU = 0.0;
        if (omin < 3.0e38f) {
            double S = 0.0;
            for (int s = 0; s < nsplit; ++s) {
                const P1Part p = part[(size_t)s * n + i];
                if (p.S > 0.0) {
                    const int sh = (int)fmaxf(omin - p.o, -4000.0f);       // integer-valued, <= 0
                    S += ldexp(p.S, sh);
                    SU += ldexp(p.SU, sh);
                }
            }
            log2S = log2(S) - (double)omin;
        }
        const double sigma2 = *sigma2_ptr, w = *w_ptr;
        double c = 0.0;
        if (w > 0.0) {
            const double tps = 2.0 * 3.14159265358979323846 * sigma2;
            c = (st->dim == 3 ? tps * sqrt(tps) : tps) * (w / (1.0 - w) * (double)st->m / (double)st->n_global);
        }
        double lc = c > 0.0 ? log2(c) : -INFINITY, dead_shift = 0.0;
        if (log2c_ptr != nullptr) { lc = log2c_ptr[0]; dead_shift = log2c_ptr[1]; c = (lc > -INFINITY) ? 1.0 : 0.0; }
        const bool dead = !(log2S + dead_shift >= DEAD_LOG2);
        double L = 0.0, p1n = 0.0;
        if (!dead) {
            if (c > 0.0) {
                const double hi = fmax(log2S, lc), lo = fmin(log2S, lc);
                L = hi + log2(1.0 + exp2(lo - hi));
                p1n = exp2(log2S - L);
            } else {
                L = log2S; p1n = 1.0;
            }
        }
        pt1[i] = p1n;
        const float4 b = tgtP[i];
        float no = INFINITY, rnf = 0.0f;
        if (!dead) {
            const double rn = exp2(-(L + (double)omin));
            no = -omin;
            rnf = (float)rn;
            v[0] = SU * (double)rnf;       // the same (rounded) rn that pass 2 multiplies by
        }
        v[1] = p1n;
        tgtQ[3 * (size_t)i] = make_float4(b.x, b.x, b.y, b.y);
        tgtQ[3 * (size_t)i + 1] = make_float4(b.z, b.z, no, no);
        tgtQ[3 * (size_t)i + 2] = make_float4(rnf, rnf, 0.f, 0.f);
    } else if (i < npad) {
        tgtQ[3 * (size_t)i] = make_float4(0.f, 0.f, 0.f, 0.f);
        tgtQ[3 * (size_t)i + 1] = make_float4(0.f, 0.f, INFINITY, INFINITY);
        tgtQ[3 * (size_t)i + 2] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    block_reduce_store<RM_TGT>(v, mom_part + (size_t)blockIdx.x * RM_TGT);
}

// ---------------------------------------------------------------------------------------------
// pass 2: per source m and split of the targets:  p1_m = sum_n P_mn,  sd_m = sum_n P_mn (a_m - b_n)
// with P_mn = 2^(o_n - u_mn) * rn_n.  Per two pairs: 11 packed FP32 instructions + 2 MUFU.
// ---------------------------------------------------------------------------------------------
template <bool CULL, bool WGT>
__global__ void __launch_bounds__(THREADS, CPD_MINB2)
pass2_kernel(const float4* __restrict__ ipts, int ni, const float4* __restrict__ jrec, const int4* __restrict__ work,
             double* __restrict__ part /* [slot][ni][4] */, const float4* __restrict__ tbox /* per target stage bbox or null */,
             const float* __restrict__ omax_stage, const float4* __restrict__ tsub, const float* __restrict__ omax_sub) {
    __shared__ float wbox[THREADS / 32][8];
    CPD_DYN_SMEM(smraw);
    uint64_t* full = reinterpret_cast<uint64_t*>(smraw + NSTAGE * P2_STAGE_BYTES);
    const int tid = threadIdx.x;
    const int4 wk = work[blockIdx.x];               // {i-tile, first stage, end stage, partial slot}: whole stages (build_work with
    const int itile = wk.x, st0 = wk.y, split = wk.w;   // a stage as the unit; pass 1 cuts at sub-chunks)
    const int nst = wk.z - wk.y;
    const unsigned char* jbytes = reinterpret_cast<const unsigned char*>(jrec);
    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        for (int s = 0; s < NSTAGE && s < nst; ++s) {
            mbar_expect_tx(&full[s], P2_STAGE_BYTES);
            tma_load_1d(smraw + s * P2_STAGE_BYTES, jbytes + (size_t)(st0 + s) * P2_STAGE_BYTES, P2_STAGE_BYTES, &full[s]);
        }
    }
    u64 ax[NPAIR2], ay[NPAIR2], az[NPAIR2], al[NPAIR2];      // al = (la, la') of the two sources: WGT only
    double A1[RI2], AX[RI2], AY[RI2], AZ[RI2];
#pragma unroll
    for (int p = 0; p < NPAIR2; ++p) {
        int m0 = itile * ITILE2 + (tid >> 5) * (32 * RI2) + (2 * p) * 32 + (tid & 31), m1 = m0 + 32;
        m0 = m0 < ni ? m0 : ni - 1;
        m1 = m1 < ni ? m1 : ni - 1;
        const float4 p0 = ipts[m0], p1 = ipts[m1];
        ax[p] = pack2(p0.x, p1.x); ay[p] = pack2(p0.y, p1.y); az[p] = pack2(p0.z, p1.z);
        if (WGT) al[p] = pack2(p0.w, p1.w);
    }
    float* const mybox = wbox[tid >> 5];
    if (CULL) warp_bbox<NPAIR2>(ax, ay, az, mybox);
#pragma unroll
    for (int r = 0; r < RI2; ++r) { A1[r] = 0.0; AX[r] = 0.0; AY[r] = 0.0; AZ[r] = 0.0; }
    for (int it = 0; it < nst; ++it) {
        const int s = it % NSTAGE;
        mbar_wait(&full[s], (uint32_t)((it / NSTAGE) & 1));
        const ulonglong2* sp = reinterpret_cast<const ulonglong2*>(smraw + s * P2_STAGE_BYTES);
        bool skip = false;
        if (CULL) {
            const float4 blo = tbox[2 * (st0 + it)], bhi = tbox[2 * (st0 + it) + 1];
            skip = box_gap2(mybox, blo, bhi) - omax_stage[st0 + it] >= CULL_GAP;
        }
#pragma unroll 1
        for (int sc = 0; sc < (skip ? 0 : P2_STAGE / SUB); ++sc) {
            if (CULL) {
                const int sb = (st0 + it) * (P2_STAGE / SUB) + sc;
                if (box_gap2(mybox, tsub[2 * sb], tsub[2 * sb + 1]) - omax_sub[sb] >= CULL_GAP) continue;
            }
            const ulonglong2* q = sp + sc * (3 * SUB);
            u64 s1[NPAIR2], sx[NPAIR2], sy[NPAIR2], sz[NPAIR2];
#pragma unroll
            for (int p = 0; p < NPAIR2; ++p) { s1[p] = 0ull; sx[p] = 0ull; sy[p] = 0ull; sz[p] = 0ull; }
            if (GRP > 0) {
#pragma unroll 1
                for (int g0 = 0; g0 < SUB; g0 += (GRP > 0 ? GRP : SUB)) {
                    u64 g1[NPAIR2], gx[NPAIR2], gy[NPAIR2], gz[NPAIR2];
#pragma unroll
                    for (int jj = 0; jj < (GRP > 0 ? GRP : 1); ++jj) {
                        const ulonglong2 bxy = q[3 * (g0 + jj)];
                        const ulonglong2 bzo = q[3 * (g0 + jj) + 1];
                        const u64 rn = q[3 * (g0 + jj) + 2].x;
#pragma unroll
                        for (int p = 0; p < NPAIR2; ++p) {
                            const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bzo.x);
                            u64 t = ffma2(dx, dx, bzo.y);         // t' = u - o_n: the same FMA chain and offset as pass 1
                            t = ffma2(dy, dy, t);
                            t = ffma2(dz, dz, t);
                            if (WGT) t = fadd2(t, al[p]);
                            const float2 tt = unpack2(t);
                            const u64 pr = fmul2(pack2(ex2(-tt.x), ex2(-tt.y)), rn);
                            g1[p] = jj == 0 ? pr : fadd2(g1[p], pr);
                            gx[p] = jj == 0 ? fmul2(pr, dx) : ffma2(pr, dx, gx[p]);
                            gy[p] = jj == 0 ? fmul2(pr, dy) : ffma2(pr, dy, gy[p]);
                            gz[p] = jj == 0 ? fmul2(pr, dz) : ffma2(pr, dz, gz[p]);
                        }
                    }
#pragma unroll
                    for (int p = 0; p < NPAIR2; ++p) {
                        s1[p] = fadd2(s1[p], g1[p]); sx[p] = fadd2(sx[p], gx[p]);
                        sy[p] = fadd2(sy[p], gy[p]); sz[p] = fadd2(sz[p], gz[p]);
                    }
                }
            } else {
#pragma unroll UNROLL2
                for (int jj = 0; jj < SUB; ++jj) {
                    const ulonglong2 bxy = q[3 * jj];
                    const ulonglong2 bzo = q[3 * jj + 1];
                    const u64 rn = q[3 * jj + 2].x;
#pragma unroll
                    for (int p = 0; p < NPAIR2; ++p) {
                        const u64 dx = fsub2(ax[p], bxy.x), dy = fsub2(ay[p], bxy.y), dz = fsub2(az[p], bzo.x);
                        u64 t = ffma2(dx, dx, bzo.y);
                        t = ffma2(dy, dy, t);
                        t = ffma2(dz, dz, t);
                        if (WGT) t = fadd2(t, al[p]);
                        const float2 tt = unpack2(t);
                        const u64 pr = fmul2(pack2(ex2(-tt.x), ex2(-tt.y)), rn);
                        s1[p] = fadd2(s1[p], pr);
                        sx[p] = ffma2(pr, dx, sx[p]);
                        sy[p] = ffma2(pr, dy, sy[p]);
                        sz[p] = ffma2(pr, dz, sz[p]);
                    }
                }
            }
#pragma unroll
            for (int p = 0; p < NPAIR2; ++p) {
                const float2 v1 = unpack2(s1[p]), vx = unpack2(sx[p]), vy = unpack2(sy[p]), vz = unpack2(sz[p]);
                A1[2 * p] += (double)v1.x; AX[2 * p] += (double)vx.x; AY[2 * p] += (double)vy.x; AZ[2 * p] += (double)vz.x;
                A1[2 * p + 1] += (double)v1.y; AX[2 * p + 1] += (double)vx.y; AY[2 * p + 1] += (double)vy.y; AZ[2 * p + 1] += (double)vz.y;
            }
        }
        __syncthreads();
        if (tid == 0 && it + NSTAGE < nst) {
            mbar_expect_tx(&full[s], P2_STAGE_BYTES);
            tma_load_1d(smraw + s * P2_STAGE_BYTES, jbytes + (size_t)(st0 + it + NSTAGE) * P2_STAGE_BYTES, P2_STAGE_BYTES, &full[s]);
        }
    }
#pragma unroll
    for (int r = 0; r < RI2; ++r) {
        const int m = itile * ITILE2 + (tid >> 5) * (32 * RI2) + r * 32 + (tid & 31);
        if (m < ni) {
            double2* dst = reinterpret_cast<double2*>(part + ((size_t)split * ni + m) * 4);
            dst[0] = make_double2(A1[r], AX[r]);
            dst[1] = make_double2(AY[r], AZ[r]);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// finalize 2: per source m  p1_m,  v_m = sum_n P_mn (x_n - z_m) = -sd_m / sk,  px~_m = p1_m z~_m + v_m
// (z~ = transformed source in the targets' frame, recomputed in FP64) and the source-side moments
//   Np, Sy = sum p1 y~, C = sum p1 y~ y~^T, V1 = sum v, VY = sum v y~^T          (y~ = y - cy)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS)
finalize2_kernel(const DevState* __restrict__ st, const double* __restrict__ sigma2_ptr, const double* __restrict__ part,
                 const int* __restrict__ tile_slots, int m, const double* __restrict__ yc, const double* __restrict__ ts, double* __restrict__ p1,
                 double* __restrict__ pxc, double* __restrict__ mom_part) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    double v[RM_SRC];
#pragma unroll
    for (int k = 0; k < RM_SRC; ++k) v[k] = 0.0;
    if (i < m) {
        double a1 = 0.0, a[3] = {0.0, 0.0, 0.0};
        const int nsplit = tile_slots[i / ITILE2];
        for (int s = 0; s < nsplit; ++s) {
            const double2* src = reinterpret_cast<const double2*>(part + ((size_t)s * m + i) * 4);
            const double2 u0 = src[0], u1 = src[1];
            a1 += u0.x; a[0] += u0.y; a[1] += u1.x; a[2] += u1.y;
        }
        const double inv_sk = 1.0 / sqrt(LOG2E / (2.0 * *sigma2_ptr));
        const double vv[3] = {-a[0] * inv_sk, -a[1] * inv_sk, -a[2] * inv_sk};
        const double y[3] = {yc[3 * (size_t)i], yc[3 * (size_t)i + 1], yc[3 * (size_t)i + 2]};
        double z[3];
        if (ts != nullptr) {
#pragma unroll
            for (int d = 0; d < 3; ++d) z[d] = ts[3 * (size_t)i + d] - st->cx[d];
        } else {
            const double sc = (st->tf_kind == 0) ? st->scale : 1.0;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const double l0 = sc * st->lin[3 * d], l1 = sc * st->lin[3 * d + 1], l2 = sc * st->lin[3 * d + 2];
                const double tp = l0 * st->cy[0] + l1 * st->cy[1] + l2 * st->cy[2] + st->t[d] - st->cx[d];
                z[d] = l0 * y[0] + l1 * y[1] + l2 * y[2] + tp;
            }
        }
        p1[i] = a1;
#pragma unroll
        for (int d = 0; d < 3; ++d) pxc[3 * (size_t)i + d] = a1 * z[d] + vv[d];
        v[RM_NP] = a1;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            v[RM_SY + d] = a1 * y[d];
            v[RM_V1 + d] = vv[d];
#pragma unroll
            for (int e = 0; e < 3; ++e) v[RM_VY + 3 * d + e] = vv[d] * y[e];
        }
        v[RM_C + 0] = a1 * y[0] * y[0]; v[RM_C + 1] = a1 * y[0] * y[1]; v[RM_C + 2] = a1 * y[0] * y[2];
        v[RM_C + 3] = a1 * y[1] * y[1]; v[RM_C + 4] = a1 * y[1] * y[2]; v[RM_C + 5] = a1 * y[2] * y[2];
    }
    block_reduce_store<RM_SRC>(v, mom_part + (size_t)blockIdx.x * RM_SRC);
}

// ---------------------------------------------------------------------------------------------
// API-faithful M-step inputs (cpd_mstep: an EstepResult supplied by the caller, FP64-accurate):
// the reference's own moment form.  Source side from p1 / px~ arrays, target side from pt1.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS)
src_moments_api_kernel(int m, const double* __restrict__ yc, const double* __restrict__ p1, const double* __restrict__ pxc,
                       double* __restrict__ mom_part) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    double v[MOM_SRC];
#pragma unroll
    for (int k = 0; k < MOM_SRC; ++k) v[k] = 0.0;
    if (i < m) {
        const double a1 = p1[i];
        const double a[3] = {pxc[3 * (size_t)i], pxc[3 * (size_t)i + 1], pxc[3 * (size_t)i + 2]};
        const double y[3] = {yc[3 * (size_t)i], yc[3 * (size_t)i + 1], yc[3 * (size_t)i + 2]};
        v[MOM_NP] = a1;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            v[MOM_SX + d] = a[d];
            v[MOM_SY + d] = a1 * y[d];
#pragma unroll
            for (int e = 0; e < 3; ++e) v[MOM_B + 3 * d + e] = a[d] * y[e];
        }
        v[MOM_C + 0] = a1 * y[0] * y[0]; v[MOM_C + 1] = a1 * y[0] * y[1]; v[MOM_C + 2] = a1 * y[0] * y[2];
        v[MOM_C + 3] = a1 * y[1] * y[1]; v[MOM_C + 4] = a1 * y[1] * y[2]; v[MOM_C + 5] = a1 * y[2] * y[2];
    }
    block_reduce_store<MOM_SRC>(v, mom_part + (size_t)blockIdx.x * MOM_SRC);
}

__global__ void __launch_bounds__(THREADS)
tgt_moments_api_kernel(const double* __restrict__ pt1, const double* __restrict__ xc, int n, double* __restrict__ mom_part) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    double v[MOM_TGT] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (i < n) {
        const double p = pt1[i], x0 = xc[3 * (size_t)i], x1 = xc[3 * (size_t)i + 1], x2 = xc[3 * (size_t)i + 2];
        v[0] = p; v[1] = p * x0; v[2] = p * x1; v[3] = p * x2; v[4] = p * (x0 * x0 + x1 * x1 + x2 * x2);
    }
    block_reduce_store<MOM_TGT>(v, mom_part + (size_t)blockIdx.x * MOM_TGT);
}

// ---------------------------------------------------------------------------------------------
// M-step solves in FP64 (one thread).  Rigid: probreg/cpd.py:169-192.  Affine: probreg/cpd.py:227-244.
// mstep_solve_api     : the reference's moment form, from a caller-supplied EstepResult (27 moments)
// mstep_solve_residual: the same optimum written as an update of the previous transform (24 moments)
// ---------------------------------------------------------------------------------------------
// One-sided Jacobi SVD of the leading n x n block (n = 2 or 3): a = U diag(s) V^T, s descending.
__device__ inline void jacobi_svd(int n, const double a[3][3], double U[3][3], double s[3], double V[3][3]) {
    double W[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { W[i][j] = (i < n && j < n) ? a[i][j] : 0.0; V[i][j] = (i == j) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < n - 1; ++p)
            for (int q = p + 1; q < n; ++q) {
                double al = 0, be = 0, ga = 0;
                for (int i = 0; i < n; ++i) { al += W[i][p] * W[i][p]; be += W[i][q] * W[i][q]; ga += W[i][p] * W[i][q]; }
                if (ga == 0.0) continue;
                const double lim = 1e-32 * al * be;   // |cos angle|^2 below 1e-32: orthogonal to FP64
                if (ga * ga <= lim) continue;
                off = fmax(off, ga * ga / (al * be));
                const double zeta = (be - al) / (2.0 * ga);
                const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
                for (int i = 0; i < n; ++i) {
                    const double wp = W[i][p], wq = W[i][q];
                    W[i][p] = c * wp - sn * wq; W[i][q] = sn * wp + c * wq;
                    const double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - sn * vq; V[i][q] = sn * vp + c * vq;
                }
            }
        if (off == 0.0) break;
    }
    int ord[3] = {0, 1, 2};
    double nrm[3] = {0, 0, 0};
    for (int j = 0; j < n; ++j) { double t = 0; for (int i = 0; i < n; ++i) t += W[i][j] * W[i][j]; nrm[j] = sqrt(t); }
    for (int i = 0; i < n - 1; ++i)
        for (int j = 0; j < n - 1 - i; ++j)
            if (nrm[ord[j]] < nrm[ord[j + 1]]) { int t = ord[j]; ord[j] = ord[j + 1]; ord[j + 1] = t; }
    double Vs[3][3];
    for (int j = 0; j < 3; ++j)
        for (int i = 0; i < 3; ++i) { U[i][j] = (i == j) ? 1.0 : 0.0; Vs[i][j] = (i == j) ? 1.0 : 0.0; }
    const double tiny = nrm[ord[0]] * 1e-300;
    for (int j = 0; j < n; ++j) {
        const int c = ord[j];
        s[j] = nrm[c];
        for (int i = 0; i < n; ++i) { Vs[i][j] = V[i][c]; U[i][j] = (nrm[c] > tiny) ? W[i][c] / nrm[c] : 0.0; }
    }
    for (int j = n; j < 3; ++j) s[j] = 0.0;
    // complete U for vanishing singular values so that it stays orthogonal
    if (n == 3) {
        if (!(s[2] > tiny) && s[1] > tiny) {
            U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
            U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
            U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
        }
    } else if (n == 2) {
        if (!(s[1] > tiny) && s[0] > tiny) { U[0][1] = -U[1][0]; U[1][1] = U[0][0]; }
    }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) V[i][j] = Vs[i][j];
}

__device__ inline double det_n(int n, const double a[3][3]) {
    if (n == 2) return a[0][0] * a[1][1] - a[0][1] * a[1][0];
    return a[0][0] * (a[1][1] * a[2][2] - a[1][2] * a[2][1]) - a[0][1] * (a[1][0] * a[2][2] - a[1][2] * a[2][0]) +
           a[0][2] * (a[1][0] * a[2][1] - a[1][1] * a[2][0]);
}

// solve  Y^T Z = A^T  (n x n, partial pivoting), return B = Z^T        (cpd.py:235)
__device__ inline void solve_affine(int n, const double Y[3][3], const double A[3][3], double B[3][3]) {
    double Mx[3][6];
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) { Mx[i][j] = Y[j][i]; Mx[i][n + j] = A[j][i]; }
    for (int k = 0; k < n; ++k) {
        int piv = k;
        for (int i = k + 1; i < n; ++i) if (fabs(Mx[i][k]) > fabs(Mx[piv][k])) piv = i;
        if (piv != k) for (int j = 0; j < 2 * n; ++j) { const double t = Mx[k][j]; Mx[k][j] = Mx[piv][j]; Mx[piv][j] = t; }
        for (int i = k + 1; i < n; ++i) {
            const double f = Mx[i][k] / Mx[k][k];
            for (int j = k; j < 2 * n; ++j) Mx[i][j] -= f * Mx[k][j];
        }
    }
    double Z[3][3];
    for (int c = 0; c < n; ++c)
        for (int i = n - 1; i >= 0; --i) {
            double t = Mx[i][n + c];
            for (int j = i + 1; j < n; ++j) t -= Mx[i][j] * Z[j][c];
            Z[i][c] = t / Mx[i][i];
        }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) B[i][j] = (i < n && j < n) ? Z[j][i] : (i == j ? 1.0 : 0.0);
}

__device__ inline void mstep_solve_api(DevState* st, const double* __restrict__ mom) {
    const int n = st->dim;
    const double Np = mom[MOM_NP];
    double mux[3], muy[3], A[3][3], Y[3][3];
    for (int a = 0; a < 3; ++a) { mux[a] = mom[MOM_SX + a] / Np; muy[a] = mom[MOM_SY + a] / Np; }
    const double Cs[3][3] = {{mom[MOM_C + 0], mom[MOM_C + 1], mom[MOM_C + 2]},
                             {mom[MOM_C + 1], mom[MOM_C + 3], mom[MOM_C + 4]},
                             {mom[MOM_C + 2], mom[MOM_C + 4], mom[MOM_C + 5]}};
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            A[a][b] = mom[MOM_B + 3 * a + b] - mom[MOM_SX + a] * mom[MOM_SY + b] / Np;     // cpd.py:175
            Y[a][b] = Cs[a][b] - mom[MOM_SY + a] * mom[MOM_SY + b] / Np;                    // cpd.py:181 / :234
        }
    double tr_yp1y = 0.0;
    for (int a = 0; a < n; ++a) tr_yp1y += Y[a][a];
    double tr_xp1x = mom[MOM_TXX] + mom[MOM_NPT] * (mux[0] * mux[0] + mux[1] * mux[1] + mux[2] * mux[2]) -
                     2.0 * (mux[0] * mom[MOM_SXT] + mux[1] * mom[MOM_SXT + 1] + mux[2] * mom[MOM_SXT + 2]);   // cpd.py:184
    double lin[3][3], scale = 1.0, sigma2, q;
    if (st->tf_kind == 0) {
        double U[3][3], s[3], V[3][3], UVt[3][3];
        jacobi_svd(n, A, U, s, V);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) { double t = 0; for (int k = 0; k < n; ++k) t += U[i][k] * V[j][k]; UVt[i][j] = t; }
        const double dt = det_n(n, UVt);                                                     // cpd.py:177-178
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double t = 0;
                for (int k = 0; k < n; ++k) t += U[i][k] * (k == n - 1 ? dt : 1.0) * V[j][k];
                lin[i][j] = (i < n && j < n) ? t : (i == j ? 1.0 : 0.0);                      // cpd.py:179
            }
        double tr_atr = 0.0;
        for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) tr_atr += A[i][j] * lin[i][j];   // cpd.py:180
        scale = st->update_scale ? tr_atr / tr_yp1y : 1.0;                                   // cpd.py:182
        if (st->update_scale) sigma2 = (tr_xp1x - scale * tr_atr) / (Np * n);                // cpd.py:186
        else sigma2 = (tr_xp1x + tr_yp1y - scale * tr_atr) / (Np * n);                       // cpd.py:188
        sigma2 = fmax(sigma2, EPS32);                                                        // cpd.py:189
        q = (tr_xp1x - 2.0 * scale * tr_atr + scale * scale * tr_yp1y) / (2.0 * sigma2) + n * Np * 0.5 * log(sigma2);
    } else {
        solve_affine(n, Y, A, lin);
        double tr_abt = 0.0;
        for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) tr_abt += A[i][j] * lin[i][j];   // cpd.py:238
        sigma2 = fmax((tr_xp1x - tr_abt) / (Np * n), EPS32);                                 // cpd.py:239-241
        q = (tr_xp1x - 2.0 * tr_abt + tr_abt) / (2.0 * sigma2) + n * Np * 0.5 * log(sigma2);  // cpd.py:242-243
    }
    // t = mu_x - scale * lin * mu_y  with mu_x = cx + mux, mu_y = cy + muy                  cpd.py:183 / :236
    for (int a = 0; a < 3; ++a) {
        double r = 0.0;
        for (int b = 0; b < 3; ++b) r += lin[a][b] * (st->cy[b] + muy[b]);
        st->t[a] = (a < n) ? (st->cx[a] + mux[a]) - scale * r : 0.0;
        for (int b = 0; b < 3; ++b) st->lin[3 * a + b] = lin[a][b];
    }
    st->scale = scale; st->sigma2 = sigma2; st->q = q; st->n_p = Np;
}

// ---------------------------------------------------------------------------------------------
// Residual-form M-step.  With A = previous linear part (s R or B), z~ = A y~ + t' the previous
// transformed source, v_m = sum_n P_mn (x_n - z_m):
//   Ycov = C - Sy Sy^T / Np,  Vcov = VY - V1 Sy^T / Np
//   A_mat = sum_mn P x^ y^T (cpd.py:175 / :233) = A Ycov + Vcov           -- FP64, no FP32 sum enters a large term
//   rigid : R' from the SVD of A_mat, s' = tr(A_mat^T R') / tr(Ycov)        (cpd.py:176-182)
//   affine: B' = A_mat Ycov^-1                                               (cpd.py:234-235)
//   Q = sum_mn P |x_n - T'(y_m)|^2 = Srr + 2 <dA, Vcov> - |V1|^2 / Np + tr(dA Ycov dA^T),  dA = A - A'
//   sigma2' = Q / (Np D)           [== (tr_xp1x - s tr_atr)/(Np D) at the optimal s, cpd.py:186 / :239]
//           = (Q + tr_atr)/(Np D)  when update_scale is False (the reference's formula, cpd.py:188)
//   q = Q / (2 sigma2') + D Np / 2 log sigma2'                                (cpd.py:190-191 / :242-243)
//   t' = mu_x - A' mu_y,  mu_x = cx + A mu~_y + t'_old + V1/Np,  mu_y = cy + Sy/Np
// ---------------------------------------------------------------------------------------------
__device__ inline void mstep_solve_residual(DevState* st, const double* __restrict__ mom) {
    const int n = st->dim;
    const double Np = mom[RM_NP];
    const double sk2 = LOG2E / (2.0 * st->sigma2);
    const double Srr = mom[RM_SRR] / sk2;
    double muy[3], V1[3], Aold[3][3], Y[3][3], Vc[3][3], Am[3][3], told[3];
    const double sc = (st->tf_kind == 0) ? st->scale : 1.0;
    for (int a = 0; a < 3; ++a) {
        muy[a] = mom[RM_SY + a] / Np;
        V1[a] = mom[RM_V1 + a];
        for (int b = 0; b < 3; ++b) Aold[a][b] = sc * st->lin[3 * a + b];
    }
    for (int a = 0; a < 3; ++a)
        told[a] = Aold[a][0] * st->cy[0] + Aold[a][1] * st->cy[1] + Aold[a][2] * st->cy[2] + st->t[a] - st->cx[a];
    const double Cs[3][3] = {{mom[RM_C + 0], mom[RM_C + 1], mom[RM_C + 2]},
                             {mom[RM_C + 1], mom[RM_C + 3], mom[RM_C + 4]},
                             {mom[RM_C + 2], mom[RM_C + 4], mom[RM_C + 5]}};
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            Y[a][b] = Cs[a][b] - mom[RM_SY + a] * mom[RM_SY + b] / Np;
            Vc[a][b] = mom[RM_VY + 3 * a + b] - V1[a] * mom[RM_SY + b] / Np;
        }
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            double t = Vc[a][b];
            for (int k = 0; k < 3; ++k) t += Aold[a][k] * Y[k][b];
            Am[a][b] = (a < n && b < n) ? t : 0.0;
        }
    double tr_yp1y = 0.0;
    for (int a = 0; a < n; ++a) tr_yp1y += Y[a][a];
    double lin[3][3], Anew[3][3], scale = 1.0, tr_atr = 0.0;
    if (st->tf_kind == 0) {
        double U[3][3], s[3], V[3][3], UVt[3][3];
        jacobi_svd(n, Am, U, s, V);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) { double t = 0; for (int k = 0; k < n; ++k) t += U[i][k] * V[j][k]; UVt[i][j] = t; }
        const double dt = det_n(n, UVt);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                double t = 0;
                for (int k = 0; k < n; ++k) t += U[i][k] * (k == n - 1 ? dt : 1.0) * V[j][k];
                lin[i][j] = (i < n && j < n) ? t : (i == j ? 1.0 : 0.0);
            }
        for (int i = 0; i < n; ++i) for (int j = 0; j < n; ++j) tr_atr += Am[i][j] * lin[i][j];
        scale = st->update_scale ? tr_atr / tr_yp1y : 1.0;
    } else {
        solve_affine(n, Y, Am, lin);
    }
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Anew[i][j] = scale * lin[i][j];
    // Q = Srr + 2 <dA, Vcov> - |V1|^2/Np + tr(dA Ycov dA^T)
    double Q = Srr - (V1[0] * V1[0] + V1[1] * V1[1] + V1[2] * V1[2]) / Np;
    for (int a = 0; a < n; ++a)
        for (int b = 0; b < n; ++b) {
            const double dab = Aold[a][b] - Anew[a][b];
            Q += 2.0 * dab * Vc[a][b];
            double t = 0.0;
            for (int k = 0; k < n; ++k) t += (Aold[a][k] - Anew[a][k]) * Y[k][b];
            Q += t * dab;
        }
    double sigma2;
    if (st->tf_kind == 0 && !st->update_scale) sigma2 = (Q + tr_atr) / (Np * n);      // cpd.py:188
    else sigma2 = Q / (Np * n);                                                        // cpd.py:186 / :239
    sigma2 = fmax(sigma2, EPS32);                                                      // cpd.py:189 / :241
    const double q = Q / (2.0 * sigma2) + n * Np * 0.5 * log(sigma2);
    // t' = mu_x - A' mu_y
    for (int a = 0; a < 3; ++a) {
        double mux = st->cx[a] + told[a] + V1[a] / Np, r = 0.0;
        for (int b = 0; b < 3; ++b) { mux += Aold[a][b] * muy[b]; r += Anew[a][b] * (st->cy[b] + muy[b]); }
        st->t[a] = (a < n) ? mux - r : 0.0;
    }
    for (int a = 0; a < 3; ++a) for (int b = 0; b < 3; ++b) st->lin[3 * a + b] = lin[a][b];
    st->scale = scale; st->sigma2 = sigma2; st->q = q; st->n_p = Np;
}

// The M-step of the fused loop on a shared-memory copy of the state: thread 0 alone walking DevState and the moments in global
// memory paid one L2 round trip per field (~50 dependent loads).
// All threads of the calling block must enter; `mom` may be global or shared.
__device__ __forceinline__ void mstep_staged(DevState* st, const double* mom) {
    __shared__ DevState sst;
    __shared__ double smom[MOM_PAD];
    static_assert(sizeof(DevState) % 8 == 0, "DevState is copied as 8-byte words");
    const int nw = (int)(sizeof(DevState) / 8);
    for (int e = threadIdx.x; e < nw; e += blockDim.x) reinterpret_cast<double*>(&sst)[e] = reinterpret_cast<const double*>(st)[e];
    for (int e = threadIdx.x; e < MOM_PAD; e += blockDim.x) smom[e] = mom[e];
    __syncthreads();
    if (threadIdx.x == 0) mstep_solve_residual(&sst, smom);
    __syncthreads();
    if (threadIdx.x < 16) reinterpret_cast<double*>(st)[threadIdx.x] = reinterpret_cast<const double*>(&sst)[threadIdx.x];   // lin, t, scale, sigma2, q, n_p
}

// Fixed-order reduction of per-block moment partials: column k < ka of part_a, then kb columns of
// part_b, into mom[0 .. ka+kb); the rest of mom[0..32) is zeroed.  SOLVE = 1: the same (single)
// block then runs the residual-form M-step.  In multi-rank runs the all-reduce sits in between.
template <int SOLVE>
__global__ void __launch_bounds__(256)
moments_kernel(DevState* st, const double* __restrict__ part_a, int nb_a, int ka, const double* __restrict__ part_b, int nb_b,
               int kb, double* __restrict__ mom) {
    // 32 columns x 8 lanes of blocks; lane w takes blocks w, w+8, ... (fixed order), then the 8 lane sums are
    // combined in a fixed order: bit-reproducible, and 8x shorter dependent chains than one thread per column.
    __shared__ double sh[8][32];
    const int k = threadIdx.x & 31, w = threadIdx.x >> 5;
    double s = 0.0;
    if (k < ka) {
#pragma unroll 8
        for (int b = w; b < nb_a; b += 8) s += part_a[(size_t)b * ka + k];      // unrolled: 8 loads in flight, summed in the same order
    } else if (k < ka + kb) {
#pragma unroll 8
        for (int b = w; b < nb_b; b += 8) s += part_b[(size_t)b * kb + (k - ka)];
    }
    sh[w][k] = s;
    __syncthreads();
    if (w == 0) {
        double t = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sh[i][k];
        mom[k] = t;
    }
    if (SOLVE) {
        __syncthreads();                    // mom[] written by warp 0 is read back by the whole block (same-block global visibility)
        mstep_staged(st, mom);
    }
}
__global__ void mstep_residual_kernel(DevState* st, const double* __restrict__ mom) {
    mstep_staged(st, mom);
}
__global__ void mstep_api_kernel(DevState* st, const double* __restrict__ mom) {
    if (threadIdx.x == 0) mstep_solve_api(st, mom);
}

// ---------------------------------------------------------------------------------------------
// Fused "reduce moments -> all-reduce over NVLink -> M-step" for multi-GPU runs: ONE launch instead of
// (reduce kernel, ncclAllReduce, M-step kernel).  The collective is 32 doubles, i.e. pure latency, so it is
// done as a one-shot exchange through peer-mapped memory inside the kernel that needs the result:
//   1. fixed-order reduction of this rank's block partials (as moments_kernel)
//   2. store the 32 sums into slot [parity][my rank] of EVERY rank's mailbox (st.global over NVLink / local)
//   3. __threadfence_system, then a release store of the sequence number into every mailbox's flag
//   4. acquire-spin on my own mailbox's flags until every rank's sequence number has arrived (bounded)
//   5. sum the slots in rank order (identical arithmetic on every rank), run the FP64 M-step
// ---------------------------------------------------------------------------------------------
#ifndef CPD_HOST_EMU
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_relaxed_sys(const double* p) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
#endif
__global__ void __launch_bounds__(256)
moments_p2p_kernel(DevState* st, const double* __restrict__ part_a, int nb_a, int ka, const double* __restrict__ part_b,
                   int nb_b, int kb, double* __restrict__ mom, P2PInfo* info) {
    __shared__ double sh[8][32];
    __shared__ double loc[32];
    __shared__ int timeout;
    const int k = threadIdx.x & 31, w = threadIdx.x >> 5;
    double s = 0.0;
    if (k < ka) {
#pragma unroll 8
        for (int b = w; b < nb_a; b += 8) s += part_a[(size_t)b * ka + k];      // unrolled: 8 loads in flight, summed in the same order
    } else if (k < ka + kb) {
#pragma unroll 8
        for (int b = w; b < nb_b; b += 8) s += part_b[(size_t)b * kb + (k - ka)];
    }
    sh[w][k] = s;
    if (threadIdx.x == 0) timeout = 0;
    __syncthreads();
    if (w == 0) {
        double t = 0.0;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sh[i][k];
        loc[k] = t;
    }
    __syncthreads();
    const int world = info->world, rank = info->rank;
    const unsigned long long seq = info->seq + 1;
    const int par = (int)(seq & 1ull);
    for (int r = w; r < world; r += 8) info->box[r]->slots[par][rank][k] = loc[k];
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < world) {
        st_release_sys(&info->box[threadIdx.x]->flags[par][rank], seq);
        const unsigned long long* f = &info->box[rank]->flags[par][threadIdx.x];
        // wall-clock bound (a spin count would depend on the clock and on time slicing): ranks are only loosely synchronised by
        // their host loops, so a peer may legitimately be late by as long as its slowest per-iteration callback
        const unsigned long long t0 = globaltimer_ns(), limit = info->timeout_ns;
        while (ld_acquire_sys(f) < seq) {
            __nanosleep(64);
            if (globaltimer_ns() - t0 > limit) { timeout = 1; break; }     // a peer is gone: fail instead of hanging the GPU
        }
    }
    __syncthreads();
    if (w == 0) {
        double t = 0.0;
        for (int r = 0; r < world; ++r) t += ld_relaxed_sys(&info->box[rank]->slots[par][r][k]);
        mom[k] = t;
        if (k == 0) {
            info->seq = seq;
            if (timeout) st->err = 1;                   // incomplete sums: the state is left as it was; the host reports the error
        }
    }
    __syncthreads();
    if (!timeout && st->err == 0) mstep_staged(st, mom);             // (every later step of a failed run is a no-op)
}

// ---------------------------------------------------------------------------------------------
// Spatial (Morton / Z-order) ordering of both clouds inside the library.  Purely an internal permutation:
// every result leaves the library in the caller's order.  Why it exists: consecutive j-points are then
// spatial neighbours, so the 8-point groups / 64-point sub-chunks of the FP32 summations hold terms of
// similar magnitude and the systematic loss of small terms (absorption) vanishes -- on the 1500-point
// fixture the CPU emulation of the kernel arithmetic (tools/emulate_resid.py) goes from -1.7e-7 to +1.6e-8
// relative error on sigma2; it also makes a warp's lanes spatially coherent, so the rare offset slow path of
// pass 1 fires for whole warps at once instead of for one lane at a time.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned spread3(unsigned v) {       // 10 bits -> every third bit
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}
__global__ void __launch_bounds__(THREADS)
morton_kernel(const double* __restrict__ pts, long long n, double lo0, double lo1, double lo2, double inv_range,
              unsigned* __restrict__ codes, int* __restrict__ idx) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < n) {
        const double q0 = (pts[3 * i] - lo0) * inv_range, q1 = (pts[3 * i + 1] - lo1) * inv_range, q2 = (pts[3 * i + 2] - lo2) * inv_range;
        const unsigned a = (unsigned)fmin(fmax(q0 * 1023.0, 0.0), 1023.0), b = (unsigned)fmin(fmax(q1 * 1023.0, 0.0), 1023.0),
                       c = (unsigned)fmin(fmax(q2 * 1023.0, 0.0), 1023.0);
        codes[i] = spread3(a) | (spread3(b) << 1) | (spread3(c) << 2);
        idx[i] = (int)i;
    }
}
// The same two kernels taking their parameters from device memory (`frame`, written by cloud_frame_kernel): set_source / set_target
// enqueue upload -> statistics -> frame -> Morton sort without a host round trip in between.
__global__ void __launch_bounds__(THREADS)
morton_frame_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ frame, unsigned* __restrict__ codes,
                    int* __restrict__ idx) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < n) {
        const double inv_range = frame[3];
        const double q0 = (pts[3 * i] - frame[0]) * inv_range, q1 = (pts[3 * i + 1] - frame[1]) * inv_range,
                     q2 = (pts[3 * i + 2] - frame[2]) * inv_range;
        const unsigned a = (unsigned)fmin(fmax(q0 * 1023.0, 0.0), 1023.0), b = (unsigned)fmin(fmax(q1 * 1023.0, 0.0), 1023.0),
                       c = (unsigned)fmin(fmax(q2 * 1023.0, 0.0), 1023.0);
        codes[i] = spread3(a) | (spread3(b) << 1) | (spread3(c) << 2);
        idx[i] = (int)i;
    }
}
__global__ void __launch_bounds__(THREADS)
gather3_frame_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long n, const double* __restrict__ frame,
                     double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) {
        const long long j = perm[k];
        out[3 * k] = in[3 * j] - frame[4]; out[3 * k + 1] = in[3 * j + 1] - frame[5]; out[3 * k + 2] = in[3 * j + 2] - frame[6];
    }
}
// out[k] = in[perm[k]] - origin   (n x 3)
__global__ void __launch_bounds__(THREADS)
gather3_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long n, double o0, double o1, double o2,
               double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) {
        const long long j = perm[k];
        out[3 * k] = in[3 * j] - o0; out[3 * k + 1] = in[3 * j + 1] - o1; out[3 * k + 2] = in[3 * j + 2] - o2;
    }
}
__global__ void __launch_bounds__(THREADS)
gather1_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long n, double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) out[k] = in[perm[k]];
}
__global__ void __launch_bounds__(THREADS)
gather_f32_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long n, float* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) out[k] = (float)in[perm[k]];
}
// out[perm[k]] = in[k]   (n x ncomp): back to the caller's order
__global__ void __launch_bounds__(THREADS)
scatter_kernel(const double* __restrict__ in, const int* __restrict__ perm, long long n, int ncomp, double* __restrict__ out) {
    const long long k = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (k < n) {
        const long long j = perm[k];
        for (int c = 0; c < ncomp; ++c) out[ncomp * j + c] = in[ncomp * k + c];
    }
}

// per-block {sum(3), min(3), max(3)} of a cloud, then a one-block fold: the centroid and bounding box that
// the Morton ordering needs, without a host pass over the caller's array
__global__ void __launch_bounds__(THREADS)
stats_kernel(const double* __restrict__ pts, long long n, double* __restrict__ part) {
    __shared__ double sh[9][THREADS / 32];
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[9];
    if (i < n) {
        for (int a = 0; a < 3; ++a) { v[a] = pts[3 * i + a]; v[3 + a] = v[a]; v[6 + a] = v[a]; }
    } else {
        for (int a = 0; a < 3; ++a) { v[a] = 0.0; v[3 + a] = 1.0e300; v[6 + a] = -1.0e300; }
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        double x = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double y = __shfl_xor_sync(0xffffffffu, x, o);
            x = k < 3 ? x + y : (k < 6 ? fmin(x, y) : fmax(x, y));
        }
        if (lane == 0) sh[k][wid] = x;
    }
    __syncthreads();
    if (threadIdx.x < 9) {
        const int k = threadIdx.x;
        double x = sh[k][0];
        for (int w = 1; w < THREADS / 32; ++w) x = k < 3 ? x + sh[k][w] : (k < 6 ? fmin(x, sh[k][w]) : fmax(x, sh[k][w]));
        part[(size_t)blockIdx.x * 9 + k] = x;
    }
}
__global__ void __launch_bounds__(288)
stats_fold_kernel(const double* __restrict__ part, int nb, double* __restrict__ out) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;       // one warp per statistic
    double x = k < 3 ? 0.0 : (k < 6 ? 1.0e300 : -1.0e300);
    for (int b = lane; b < nb; b += 32) {
        const double y = part[(size_t)b * 9 + k];
        x = k < 3 ? x + y : (k < 6 ? fmin(x, y) : fmax(x, y));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double y = __shfl_xor_sync(0xffffffffu, x, o);
        x = k < 3 ? x + y : (k < 6 ? fmin(x, y) : fmax(x, y));
    }
    if (lane == 0) out[k] = x;
}

// From the nine statistics of a cloud (sums, minima, maxima) to its frame, on the device:
//   frame[0..2] = lower corner, frame[3] = 1 / longest bounding-box edge (Morton quantisation), frame[4..6] = the origin the cloud is
//   centred on (its centroid, or the caller's frame origin).  The origin and the count also go into the device state (sources: cy, m;
//   targets: cx, n_global); the host mirror of the state catches up when it next needs them (ensure_stats in cpd_b200.cu).
__global__ void cloud_frame_kernel(const double* __restrict__ sums9, long long count, int is_target, long long n_global, int origin_given,
                                   double o0, double o1, double o2, DevState* __restrict__ st, double* __restrict__ frame) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double range = 0.0;
    for (int a = 0; a < 3; ++a) { frame[a] = sums9[3 + a]; range = fmax(range, sums9[6 + a] - sums9[3 + a]); }
    frame[3] = range > 0.0 ? 1.0 / range : 0.0;
    const double og[3] = {o0, o1, o2};
    for (int a = 0; a < 3; ++a) {
        const double o = origin_given ? og[a] : sums9[a] / (double)count;
        frame[4 + a] = o;
        if (is_target) st->cx[a] = o; else st->cy[a] = o;
    }
    if (is_target) st->n_global = n_global; else st->m = count;
}

// sums for sigma^2 initialisation: out[block][0..4) = sum |p|^2, sum p (3)
__global__ void __launch_bounds__(THREADS)
cloud_sums_kernel(const double* __restrict__ pts, long long n, double* __restrict__ out) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    if (i < n) {
        const double a = pts[3 * i], b = pts[3 * i + 1], c = pts[3 * i + 2];
        v[0] = a * a + b * b + c * c; v[1] = a; v[2] = b; v[3] = c;
    }
    block_reduce_store<4>(v, out + (size_t)blockIdx.x * 4);
}
// out[c] = sum_b part[b][c], c < k: one warp per column (launch with k * 32 threads, k <= 32), lanes take the blocks b = lane,
// lane + 32, ..., a fixed shuffle tree joins them -- the same order on every run.
__global__ void __launch_bounds__(1024)
reduce_cols_kernel(const double* __restrict__ part, int nb, int k, double* __restrict__ out) {
    const int c = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (c >= k) return;
    double s = 0.0;
    for (int b = lane; b < nb; b += 32) s += part[(size_t)b * k + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[c] = s;
}

// px = px~ + cx * p1 (un-centre for the API-facing EstepResult)
__global__ void __launch_bounds__(THREADS)
uncentre_px_kernel(const DevState* __restrict__ st, const double* __restrict__ p1, const double* __restrict__ pxc, int m,
                   double* __restrict__ px) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
#pragma unroll
        for (int d = 0; d < 3; ++d) px[3 * (size_t)i + d] = pxc[3 * (size_t)i + d] + st->cx[d] * p1[i];
    }
}
__global__ void __launch_bounds__(THREADS)
centre_px_kernel(const DevState* __restrict__ st, const double* __restrict__ p1, const double* __restrict__ px, int m,
                 double* __restrict__ pxc) {
    const int i = blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
#pragma unroll
        for (int d = 0; d < 3; ++d) pxc[3 * (size_t)i + d] = px[3 * (size_t)i + d] - st->cx[d] * p1[i];
    }
}
// _math.rbf_kernel (cc/math_utils.cc:17-19): float32 Gram matrix, 2*beta in the denominator
__global__ void __launch_bounds__(THREADS)
rbf_kernel_kernel(const float* __restrict__ x, long long nx, const float* __restrict__ y, long long ny, int dim, float two_beta,
                  float* __restrict__ out) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;      // rows on grid.x: grid.y is limited to 65535
    const long long i = blockIdx.x;
    if (j < ny) {
        float d2 = 0.f;
        for (int a = 0; a < dim; ++a) { const float d = x[i * dim + a] - y[j * dim + a]; d2 += d * d; }
        out[i * ny + j] = expf(-d2 / two_beta);          // a division, like (-diff2 / (2.0 * beta)).exp() in cc/math_utils.cc:18
    }
}

// _math.inverse_multiquadric_kernel (cc/math_utils.cc:37-39): float32 (|x_i - y_j|^2 + c)^(-1/2)
__global__ void __launch_bounds__(THREADS)
imq_kernel_kernel(const float* __restrict__ x, long long nx, const float* __restrict__ y, long long ny, int dim, float c,
                  float* __restrict__ out) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;
    const long long i = blockIdx.x;
    if (j < ny) {
        // every operation rounded on its own (no FMA contraction), like Eigen's squaredNorm built without -mfma and the float32
        // numpy restatement the fixtures come from: BCPD inverts this matrix (bcpd.py:117), and the inverse of an inverse
        // multiquadric Gram matrix amplifies a last-bit difference of its entries to the first digits of the M-step
        float d2 = 0.f;
        for (int a = 0; a < dim; ++a) { const float d = __fsub_rn(x[i * dim + a], y[j * dim + a]); d2 = __fadd_rn(d2, __fmul_rn(d, d)); }
        out[i * ny + j] = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(d2, c)));
    }
}

// ---------------------------------------------------------------------------------------------
// Non-rigid CPD, dense G (probreg/cpd.py:247-303, transformation.py:81-102).
// G stays on the device as float32 (the reference's _math.rbf_kernel is float32, cc/types.h:19); the
// M x M system of cpd.py:296 is assembled in FP64 and handed to cuSOLVER's LU (a plain library solve).
// ---------------------------------------------------------------------------------------------
// G[i][j] = exp(-|y_i - y_j|^2 / (2 beta)) from the float32 casts of the ORIGINAL coordinates (cc/math_utils.cc:17-19)
__global__ void __launch_bounds__(THREADS)
nr_gram_kernel(const double* __restrict__ yc, double c0, double c1, double c2, long long m, int dim, float two_beta,
               float* __restrict__ G) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;      // rows on grid.x: grid.y is limited to 65535
    const long long i = blockIdx.x;
    if (j < m) {
        const double cc[3] = {c0, c1, c2};
        float d2 = 0.f;
        for (int a = 0; a < dim; ++a) {
            const float d = (float)(yc[3 * i + a] + cc[a]) - (float)(yc[3 * j + a] + cc[a]);
            d2 += d * d;
        }
        G[i * m + j] = expf(-d2 / two_beta);
    }
}
// ts_i = y_i + sum_j G_ij W_j   (transformation.py:101-102), one warp per row, FP64 accumulation
__global__ void __launch_bounds__(THREADS)
nr_apply_kernel(const float* __restrict__ G, const double* __restrict__ W, const double* __restrict__ yc, double c0, double c1,
                double c2, long long m, double* __restrict__ ts) {
    const long long i = (long long)blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    const float* row = G + i * m;
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
    for (long long j = lane; j < m; j += 32) {
        const double g = (double)row[j];
        a0 += g * W[3 * j]; a1 += g * W[3 * j + 1]; a2 += g * W[3 * j + 2];
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    if (lane == 0) {
        ts[3 * i] = yc[3 * i] + c0 + a0;
        ts[3 * i + 1] = yc[3 * i + 1] + c1 + a1;
        ts[3 * i + 2] = yc[3 * i + 2] + c2 + a2;
    }
}
// A = diag(p1) G + lmd sigma2 I, stored row-major (== column-major A^T for the LU; solved with op(T))   cpd.py:296
__global__ void __launch_bounds__(THREADS)
nr_system_kernel(const float* __restrict__ G, const double* __restrict__ wgt /* p1, or p1 + (sigma2/alpha) p1~ */,
                 const double* __restrict__ sigma2_ptr, double lmd, long long m, double* __restrict__ A) {
    const long long j = (long long)blockIdx.y * THREADS + threadIdx.x;      // rows on grid.x: grid.y is limited to 65535
    const long long i = blockIdx.x;
    if (j < m) A[i * m + j] = wgt[i] * (double)G[i * m + j] + (i == j ? lmd * *sigma2_ptr : 0.0);
}
// B[c*m + i] = px_ic - p1_i y_ic   (right-hand side of cpd.py:296; px = px~ + cx p1, y = y~ + cy)
//               + k (px~prior_ic - p1~prior_i y_ic),  k = sigma2 / alpha   with correspondence priors (cpd.py:395)
__global__ void __launch_bounds__(THREADS)
nr_rhs_kernel(const DevState* __restrict__ st, const double* __restrict__ p1, const double* __restrict__ pxc,
              const double* __restrict__ yc, const double* __restrict__ p1t, const double* __restrict__ pxt, double alpha, long long m,
              double* __restrict__ B) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) {
        const double k = p1t ? st->sigma2 / alpha : 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double y = yc[3 * i + c] + st->cy[c];
            double r = pxc[3 * i + c] + p1[i] * (st->cx[c] - y);
            if (p1t) r += k * (pxt[3 * i + c] - p1t[i] * y);
            B[c * m + i] = r;
        }
    }
}
// wgt = p1 + (sigma2 / alpha) p1~   (cpd.py:391-392)
__global__ void __launch_bounds__(THREADS)
nr_weight_kernel(const double* __restrict__ p1, const double* __restrict__ p1t, const double* __restrict__ sigma2_ptr, double alpha,
                 long long m, double* __restrict__ wgt) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) wgt[i] = p1[i] + (*sigma2_ptr / alpha) * p1t[i];
}
// ts = y (the moved source before the first M-step: W = 0, cpd.py:281)
__global__ void __launch_bounds__(THREADS)
nr_identity_kernel(const double* __restrict__ yc, double c0, double c1, double c2, long long m, double* __restrict__ ts) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) { ts[3 * i] = yc[3 * i] + c0; ts[3 * i + 1] = yc[3 * i + 1] + c1; ts[3 * i + 2] = yc[3 * i + 2] + c2; }
}
__global__ void __launch_bounds__(THREADS)
nr_unpack_kernel(const double* __restrict__ B, long long m, double* __restrict__ W) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (i < m) { W[3 * i] = B[i]; W[3 * i + 1] = B[m + i]; W[3 * i + 2] = B[2 * m + i]; }
}
// residual-form sigma2 (== tr_xp1x - 2 tr_pxt + tr_tpt of cpd.py:298-301, without its cancellation):
//   Q = Srr + sum_m ( 2 e_m . v_m + p1_m |e_m|^2 ),  e = T_old - T_new,  v = px~ - p1 (T_old - cx)
// per-block partials {sum 2 e.v + p1 |e|^2, sum p1}
__global__ void __launch_bounds__(THREADS)
nr_resid_kernel(const DevState* __restrict__ st, const double* __restrict__ p1, const double* __restrict__ pxc,
                const double* __restrict__ ts_old, const double* __restrict__ ts_new, long long m, double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[2] = {0.0, 0.0};
    if (i < m) {
        double acc = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double e = ts_old[3 * i + c] - ts_new[3 * i + c];
            const double vv = pxc[3 * i + c] - p1[i] * (ts_old[3 * i + c] - st->cx[c]);
            acc += 2.0 * e * vv + p1[i] * e * e;
        }
        v[0] = acc; v[1] = p1[i];
    }
    block_reduce_store<2>(v, part + (size_t)blockIdx.x * 2);
}
// The three traces of cpd.py:298-300 from a caller-supplied EstepResult, in the caller's (uncentred) coordinates, FP64:
// per-block partials {sum_n pt1 |x|^2, sum_m px . T, sum_m p1 |T|^2, sum_m p1}; blocks cover max(m, n) points.
__global__ void __launch_bounds__(THREADS)
nr_traces_kernel(const DevState* __restrict__ st, const double* __restrict__ pt1, const double* __restrict__ xc, long long n,
                 const double* __restrict__ p1, const double* __restrict__ pxc, const double* __restrict__ ts, long long m,
                 double* __restrict__ part) {
    const long long i = (long long)blockIdx.x * THREADS + threadIdx.x;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    if (i < n) {
        double x2 = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) { const double x = xc[3 * i + c] + st->cx[c]; x2 += x * x; }
        v[0] = pt1[i] * x2;
    }
    if (i < m) {
        double pt = 0.0, t2 = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double t = ts[3 * i + c];
            pt += (pxc[3 * i + c] + st->cx[c] * p1[i]) * t;
            t2 += t * t;
        }
        v[1] = pt; v[2] = p1[i] * t2; v[3] = p1[i];
    }
    block_reduce_store<4>(v, part + (size_t)blockIdx.x * 4);
}
// sigma2 = (tr_xp1x - 2 tr_pxt + tr_tpt) / (n_p D), q := sigma2   (cpd.py:301-303); tr[0] may have been all-reduced over ranks
__global__ void __launch_bounds__(32)
nr_sigma_api_kernel(DevState* st, const double* __restrict__ tr) {
    if (threadIdx.x == 0) {
        st->sigma2 = (tr[0] - 2.0 * tr[1] + tr[2]) / (tr[3] * st->dim);
        st->q = st->sigma2;
        st->n_p = tr[3];
    }
}
// sigma2 = (Srr / sk^2 + sum part[.][0]) / (Np D);  q := sigma2 (cpd.py:303).  mom[RM_SRR] holds the (all-reduced) Srr.
__global__ void __launch_bounds__(32)
nr_sigma_kernel(DevState* st, const double* __restrict__ part, int nb, const double* __restrict__ mom) {
    if (threadIdx.x == 0) {
        double a = 0.0, np_ = 0.0;
        for (int b = 0; b < nb; ++b) { a += part[2 * (size_t)b]; np_ += part[2 * (size_t)b + 1]; }
        const double sk2 = LOG2E / (2.0 * st->sigma2);
        const double q = mom[RM_SRR] / sk2 + a;
        st->sigma2 = q / (np_ * st->dim);
        st->q = st->sigma2;
        st->n_p = np_;
    }
}

// ---------------------------------------------------------------------------------------------
// Direct Gauss transform (probreg/gauss_transform.py:10-16): the same pair kernel as
// pass 1 without the normalisation:  out[c][i] = sum_j w[c][j] exp(-|t_i - s_j|^2 / h^2),  up to GT_K weight
// vectors per sweep.  Coordinates arrive centred and scaled by sqrt(log2 e)/h, so the exponential is 2^(-u).
// FP32 pair maths, 32-term FP32 groups, FP64 beyond.  Exact (the reference's default for h >= 0.01 is the
// IFGT approximation at eps = 1e-4, gauss_transform.py:42-45).
// ---------------------------------------------------------------------------------------------
constexpr int GT_K = 4, GT_TILE = 256;
__global__ void __launch_bounds__(THREADS)
gauss_transform_kernel(const float4* __restrict__ tg, int n, const float4* __restrict__ sc, const float* __restrict__ wts, int mpad,
                       int k0, int kn, double* __restrict__ out) {
    __shared__ float4 sp[GT_TILE];
    __shared__ float sw[GT_K][GT_TILE];
    const int i = blockIdx.x * THREADS + threadIdx.x;
    const float4 t = tg[i < n ? i : n - 1];
    double acc[GT_K];
#pragma unroll
    for (int c = 0; c < GT_K; ++c) acc[c] = 0.0;
    for (int j0 = 0; j0 < mpad; j0 += GT_TILE) {
        __syncthreads();
        sp[threadIdx.x] = sc[j0 + threadIdx.x];
#pragma unroll
        for (int c = 0; c < GT_K; ++c) sw[c][threadIdx.x] = c < kn ? wts[(size_t)(k0 + c) * mpad + j0 + threadIdx.x] : 0.0f;
        __syncthreads();
#pragma unroll 1
        for (int g = 0; g < GT_TILE; g += 32) {
            float a[GT_K];
#pragma unroll
            for (int c = 0; c < GT_K; ++c) a[c] = 0.0f;
#pragma unroll 8
            for (int jj = 0; jj < 32; ++jj) {
                const float4 b = sp[g + jj];
                const float dx = t.x - b.x, dy = t.y - b.y, dz = t.z - b.z;
                const float e = ex2(-fmaf(dz, dz, fmaf(dy, dy, dx * dx)));
#pragma unroll
                for (int c = 0; c < GT_K; ++c) a[c] = fmaf(e, sw[c][g + jj], a[c]);
            }
#pragma unroll
            for (int c = 0; c < GT_K; ++c) acc[c] += (double)a[c];
        }
    }
    if (i < n)
        for (int c = 0; c < kn; ++c) out[(size_t)(k0 + c) * n + i] = acc[c];
}

// issue-rate probes for the roofline denominators
__global__ void __launch_bounds__(256)
probe_ffma_kernel(float* out, int iters, float seed) {
    float a[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) a[k] = seed + k;
    const float m = 0.9999f + seed * 1e-9f, c = 1e-7f;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 16; ++k) a[k] = fmaf(a[k], m, c);
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) s += a[k];
    if (s == 123.456f) out[0] = s;
}
__global__ void __launch_bounds__(256)
probe_mufu_kernel(float* out, int iters, float seed) {
    float a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = seed * 0.01f - k;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = ex2(a[k]) - 1.5f;   // 1 MUFU + 1 FADD
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += a[k];
    if (s == 123.456f) out[0] = s;
}
// the pair helpers (ffma2: two scalar FMAs on sm_90): the FMA rate the pair loops can reach
__global__ void __launch_bounds__(256)
probe_ffma2_kernel(float* out, int iters, float seed) {
    u64 a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = pack2(seed + k, seed - k);
    const u64 m = pack2(0.9999f + seed * 1e-9f, 0.9998f), c = pack2(1e-7f, 2e-7f);
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = ffma2(a[k], m, c);
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { const float2 v = unpack2(a[k]); s += v.x + v.y; }
    if (s == 123.456f) out[0] = s;
}
// pair FMAs and single FMAs interleaved
__global__ void __launch_bounds__(256)
probe_ffma_mixed_kernel(float* out, int iters, float seed) {
    u64 a[6];
    float b[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { a[k] = pack2(seed + k, seed - k); b[k] = seed + 0.5f * k; }
    const u64 m2 = pack2(0.9999f + seed * 1e-9f, 0.9998f), c2 = pack2(1e-7f, 2e-7f);
    const float m = 0.9999f + seed * 1e-9f, c = 1e-7f;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 6; ++k) { a[k] = ffma2(a[k], m2, c2); b[k] = fmaf(b[k], m, c); }
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) { const float2 v = unpack2(a[k]); s += v.x + v.y + b[k]; }
    if (s == 123.456f) out[0] = s;
}
// instruction mix of the E-step inner loop: NF FP32-pipe instructions + 1 MUFU.EX2 per "pair", 8 chains
template <int NF, bool PACKED>
__global__ void __launch_bounds__(256)
probe_mix_kernel(float* out, int iters, float seed) {
    float x[8], acc[8];
    unsigned long long pa[4];
#pragma unroll
    for (int k = 0; k < 8; ++k) { x[k] = seed * 0.01f - 0.1f * k; acc[k] = 0.f; }
#pragma unroll
    for (int k = 0; k < 4; ++k) pa[k] = pack2(seed, seed + k);
    const float m = 0.999f + seed * 1e-9f;
    const unsigned long long pm = pack2(m, m);
    for (int i = 0; i < iters; ++i) {
        if (PACKED) {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
#pragma unroll
                for (int f = 0; f < NF; ++f) pa[k] = ffma2(pa[k], pm, pm);
                const float2 v = unpack2(pa[k]);
                pa[k] = pack2(ex2(-v.x * v.x), ex2(-v.y * v.y));     // 2 MUFU (+2 FMUL) per 2 pairs
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float t = x[k];
#pragma unroll
                for (int f = 0; f < NF - 1; ++f) t = fmaf(t, m, acc[k]);
                const float e = ex2(-t * t);                          // NF-th FP32 instruction + MUFU
                acc[k] = e;
            }
        }
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += acc[k];
#pragma unroll
    for (int k = 0; k < 4; ++k) { const float2 v = unpack2(pa[k]); s += v.x + v.y; }
    if (s == 123.456f) out[0] = s;
}
__global__ void probe_clock_kernel(long long* out) {
    const long long c0 = clock64();
    const unsigned long long t0 = globaltimer_ns();
    unsigned long long t1;
    do { t1 = globaltimer_ns(); } while (t1 - t0 < 2000000ull);
    out[0] = clock64() - c0;
    out[1] = (long long)(t1 - t0);
}

}  // namespace cpd
