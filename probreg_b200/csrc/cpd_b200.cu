// cpd_b200.cu -- host side of libcpd_b200.so: the C ABI declared in include/cpd_b200.h.
// One handle = one device + one stream; every EM iteration is a fixed sequence of launches on
// that stream (pack, pass 1, finalize 1, pass 2, finalize 2, moments [+ all-reduce] + M-step).
#include "cpd_b200.h"
#include "kernels.cuh"
#include "lowrank.cuh"
#include "gram_i8.cuh"
#include "bcpd.cuh"
#include "gmmtree.cuh"
#include "l2dist.cuh"
#include "ocsvm.cuh"
#include "lattice.cuh"
#include "batch.cuh"

#include <cub/device/device_radix_sort.cuh>
#ifdef CPD_HOST_EMU
#include "emu_nccl.h"
#include "emu_solver.h"
#endif

#include <dlfcn.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <memory>
#include <type_traits>
#include <vector>

using namespace cpd;

// ---------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess)                                                                     \
            return fail(CPD_ERR_CUDA, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(e_)); \
    } while (0)
#define KCHECK() CU(cudaGetLastError())

extern "C" const char* cpd_last_error(void) { return g_err; }
extern "C" int cpd_version(void) { return 100; }
extern "C" int cpd_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// ---------------------------------------------------------------------------------------------
// NCCL, bound at run time (libnccl.so.2 -- torch's bundled copy if it is already loaded)
// ---------------------------------------------------------------------------------------------
namespace {
typedef struct { char internal[128]; } nccl_uid;
typedef void* nccl_comm;
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(nccl_uid*) = nullptr;
    int (*CommInitRank)(nccl_comm*, int, nccl_uid, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm, cudaStream_t) = nullptr;
    int (*CommDestroy)(nccl_comm) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
int load_nccl() {
    if (g_nccl.lib) return CPD_OK;
#ifdef CPD_HOST_EMU   // CPU test build (tests/emu): ranks are threads of one process, the collective is a rendezvous
    static_assert(sizeof(nccl_uid) == sizeof(emu::nccl_uid_t), "unique id layout");
    g_nccl.GetUniqueId = reinterpret_cast<int (*)(nccl_uid*)>(emu::ncclGetUniqueId);
    g_nccl.CommInitRank = reinterpret_cast<int (*)(nccl_comm*, int, nccl_uid, int)>(emu::ncclCommInitRank);
    g_nccl.AllReduce = emu::ncclAllReduce;
    g_nccl.CommDestroy = emu::ncclCommDestroy;
    g_nccl.GetErrorString = emu::ncclGetErrorString;
    g_nccl.lib = (void*)&g_nccl;
    return CPD_OK;
#endif
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    void* lib = nullptr;
    for (const char* nm : names) { lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) return fail(CPD_ERR_NCCL, "cannot dlopen libnccl.so.2: %s", dlerror());
    g_nccl.GetUniqueId = (int (*)(nccl_uid*))dlsym(lib, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(nccl_comm*, int, nccl_uid, int))dlsym(lib, "ncclCommInitRank");
    g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, nccl_comm, cudaStream_t))dlsym(lib, "ncclAllReduce");
    g_nccl.CommDestroy = (int (*)(nccl_comm))dlsym(lib, "ncclCommDestroy");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.CommDestroy)
        return fail(CPD_ERR_NCCL, "libnccl lacks an expected symbol");
    g_nccl.lib = lib;
    return CPD_OK;
}
constexpr int NCCL_DOUBLE = 8, NCCL_SUM = 0;

// cuSOLVER (dense LU of the non-rigid M-step only), bound at run time like NCCL
struct SolverApi {
    void* lib = nullptr;
    int (*Create)(void**) = nullptr;
    int (*Destroy)(void*) = nullptr;
    int (*SetStream)(void*, cudaStream_t) = nullptr;
    int (*CreateParams)(void**) = nullptr;
    int (*DestroyParams)(void*) = nullptr;
    int (*XgetrfBuf)(void*, void*, int64_t, int64_t, int, const void*, int64_t, int, size_t*, size_t*) = nullptr;
    int (*Xgetrf)(void*, void*, int64_t, int64_t, int, void*, int64_t, int64_t*, int, void*, size_t, void*, size_t, int*) = nullptr;
    int (*Xgetrs)(void*, void*, int, int64_t, int64_t, int, const void*, int64_t, const int64_t*, int, void*, int64_t, int*) = nullptr;
};
SolverApi g_sol;
int load_cusolver() {
    if (g_sol.lib) return CPD_OK;
#ifdef CPD_HOST_EMU   // CPU test build (tests/emu): documented-behaviour stand-ins instead of the real library
    g_sol.Create = emu::solverCreate; g_sol.Destroy = emu::solverDestroy; g_sol.SetStream = emu::solverSetStream;
    g_sol.CreateParams = emu::solverCreateParams; g_sol.DestroyParams = emu::solverDestroyParams;
    g_sol.XgetrfBuf = emu::solverXgetrfBuf; g_sol.Xgetrf = emu::solverXgetrf; g_sol.Xgetrs = emu::solverXgetrs;
    g_sol.lib = (void*)&g_sol;
    return CPD_OK;
#endif
    const char* names[] = {"libcusolver.so.11", "/usr/local/cuda/lib64/libcusolver.so.11", "libcusolver.so"};
    void* lib = nullptr;
    for (const char* nm : names) { lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (lib) break; }
    if (!lib) return fail(CPD_ERR_CUDA, "cannot dlopen libcusolver.so.11: %s", dlerror());
#define SOLSYM(field, name) g_sol.field = (decltype(g_sol.field))dlsym(lib, name)
    SOLSYM(Create, "cusolverDnCreate");
    SOLSYM(Destroy, "cusolverDnDestroy");
    SOLSYM(SetStream, "cusolverDnSetStream");
    SOLSYM(CreateParams, "cusolverDnCreateParams");
    SOLSYM(DestroyParams, "cusolverDnDestroyParams");
    SOLSYM(XgetrfBuf, "cusolverDnXgetrf_bufferSize");
    SOLSYM(Xgetrf, "cusolverDnXgetrf");
    SOLSYM(Xgetrs, "cusolverDnXgetrs");
#undef SOLSYM
    if (!g_sol.Create || !g_sol.SetStream || !g_sol.CreateParams || !g_sol.XgetrfBuf || !g_sol.Xgetrf || !g_sol.Xgetrs)
        return fail(CPD_ERR_CUDA, "libcusolver lacks an expected symbol");
    g_sol.lib = lib;
    return CPD_OK;
}
constexpr int CUDA_R_64F_ = 1, CUBLAS_OP_N_ = 0, CUBLAS_OP_T_ = 1;
}  // namespace
#define SOLV(call)                                                                          \
    do {                                                                                    \
        int r_ = (call);                                                                    \
        if (r_ != 0) return fail(CPD_ERR_CUDA, "%s failed with cusolverStatus %d", #call, r_); \
    } while (0)
#define NC(call)                                                                                                   \
    do {                                                                                                           \
        int r_ = (call);                                                                                           \
        if (r_ != 0)                                                                                               \
            return fail(CPD_ERR_NCCL, "%s failed: %s", #call, g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?"); \
    } while (0)

// ---------------------------------------------------------------------------------------------
// owners of the handle's resources
// ---------------------------------------------------------------------------------------------
#define TRY(x) do { int r__ = (x); if (r__ != CPD_OK) return r__; } while (0)
namespace {
// device memory of `n` elements, freed by the destructor
template <typename T>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(n, o.n); return *this; }
    ~DevBuf() { reset(); }
    void reset() {
        if (p) cudaFree(p);
        p = nullptr;
        n = 0;
    }
    // exactly `count` elements (at least one is allocated); the old block is freed first and its contents are not kept
    int alloc(size_t count) {
        reset();
        cudaError_t e = cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
        if (e != cudaSuccess) {
            p = nullptr;
            return fail(CPD_ERR_CUDA, "cudaMalloc(%zu bytes) failed: %s", count * sizeof(T), cudaGetErrorString(e));
        }
        n = count;
        return CPD_OK;
    }
    // grow-only: reallocates (as alloc) only when `count` exceeds what is held
    int reserve(size_t count) { return count > n ? alloc(count) : CPD_OK; }
    size_t bytes() const { return p ? std::max<size_t>(n, 1) * sizeof(T) : 0; }
};
// pinned host memory of `count` elements, freed by the destructor
template <typename T>
struct PinBuf {
    T* p = nullptr;
    PinBuf() = default;
    PinBuf(const PinBuf&) = delete;
    PinBuf& operator=(const PinBuf&) = delete;
    ~PinBuf() { if (p) cudaFreeHost(p); }
    int alloc(size_t count) {
        CU(cudaMallocHost((void**)&p, count * sizeof(T)));
        return CPD_OK;
    }
};
// an event, destroyed with its owner; converts to cudaEvent_t at use sites
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    Event(Event&& o) noexcept : e(o.e) { o.e = nullptr; }
    ~Event() { if (e) cudaEventDestroy(e); }
    operator cudaEvent_t() const { return e; }
};
#ifndef CPD_HOST_EMU
struct GraphExecDelete { void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); } };
using GraphExec = std::unique_ptr<std::remove_pointer_t<cudaGraphExec_t>, GraphExecDelete>;
#endif
// The handle's pinned staging of small host <-> device copies, one field per use: no copy in flight can overwrite another's bytes.
struct PinStage {
    DevState state;          // read_params: the device state
    double sums[8];          // cpd_sigma2_init: target and source sums
    double es[2];            // cpd_estep, cpd_bcpd_estep: {sigma2, w} into DevState.es_sigma2 / es_w
    double bc_ssw[3];        // cpd_bcpd_estep: {scale, sigma2, w} into d_bc_es
    double n_p;              // cpd_last_estep
    int p2p_err;             // cpd_sync: DevState.err
    double nr_sigma2_p;      // cpd_nonrigid_mstep: the E-step's sigma2 into DevState.sigma2
    int nr_info;             // cpd_nonrigid_step / _mstep: getrf's info
    double bc_sigma2;        // cpd_bcpd_step: the new sigma2
    int bc_info[2];          // cpd_bcpd_step: getrf's and getrs's info
    double gmm_lb;           // cpd_gmm_fit: the lower bound of an iteration
    double gt_q;             // cpd_gmmtree_build: the log-likelihood of an iteration
    double gt_rt[12];        // cpd_gmmtree_estep: rot (9) and t (3)
};

// cuSOLVER's dense LU (getrf: the column-major n x n matrix at `a` in place; getrs: op(A) X = B for the nrhs columns of `b`),
// created on first use.  The workspace only grows: a loop that sized it for its system still finds enough after another loop
// sized it for a smaller one.
struct Solver {
    void *h = nullptr, *params = nullptr;
    DevBuf<unsigned char> d_work;
    std::vector<unsigned char> h_work;
    ~Solver() {
        if (params && g_sol.DestroyParams) g_sol.DestroyParams(params);
        if (h && g_sol.Destroy) g_sol.Destroy(h);
    }
    // after load_cusolver: the handle on `stream` and a workspace for the LU of the n x n system stored at `a`
    int reserve(cudaStream_t stream, long long n, double* a) {
        if (!h) {
            SOLV(g_sol.Create(&h));
            SOLV(g_sol.SetStream(h, stream));
            SOLV(g_sol.CreateParams(&params));
        }
        size_t wd = 0, wh = 0;
        SOLV(g_sol.XgetrfBuf(h, params, n, n, CUDA_R_64F_, a, n, CUDA_R_64F_, &wd, &wh));
        TRY(d_work.reserve(std::max<size_t>(wd, 16)));
        if (wh > h_work.size() || h_work.empty()) h_work.resize(std::max<size_t>(wh, 16));
        return CPD_OK;
    }
    int getrf(long long n, double* a, int64_t* ipiv, int* info) {
        SOLV(g_sol.Xgetrf(h, params, n, n, CUDA_R_64F_, a, n, ipiv, CUDA_R_64F_, d_work.p, d_work.n, h_work.data(), h_work.size(), info));
        return CPD_OK;
    }
    int getrs(int op, long long n, long long nrhs, const double* a, const int64_t* ipiv, double* b, int* info) {
        SOLV(g_sol.Xgetrs(h, params, op, n, nrhs, CUDA_R_64F_, a, n, ipiv, CUDA_R_64F_, b, n, info));
        return CPD_OK;
    }
};

// The loops a handle runs between calls keep what they need from one call to the next in records of their own.  The rigid / affine EM loop (cpd_set_state, cpd_em_step): DevState's transformation, shared with the non-rigid loop, which
// ends it (and is ended by it)
enum class EmStatus { none, live, ended };

// whose set-up the low-rank factors hold, hence which kernel function the G X products use
enum class LrOwner { none, nonrigid, bcpd };
// G ~= Q Bc Q^T of rank `rank` (lowrank.cuh): the set-up of the low-rank non-rigid or BCPD loop, whichever began last
struct LowRankFactors {
    LrOwner owner = LrOwner::none;
    int rank = 0;                         // > 0: a set-up finished
    long long m = 0;                      // source count the buffers were sized for (the owner's at its begin)
    double gscale = 1.0;                  // the factor of the products beyond the tile values: c^(-1/2) for the IMQ, 1 for the Gaussian
    bool spd = true;                      // symmetric positive definite K x K system on Qt = Q L (lr_spd_form); CPD_B200_LR_CORE=lu: LU of (c I + Bc S)
    float setup_ms[3] = {0.f, 0.f, 0.f};  // products / orthonormalisations / core of the last profiled set-up
    DevBuf<float4> pts;
    DevBuf<double> Q, X, coef, part, Bc, S, R, sys, rhs, c, out, panel, Lt;
    DevBuf<int> pchol_rank;               // the rank lr_pchol_kernel found
    DevBuf<unsigned char> gi_planes;      // exact int8-digit product: digit planes of X, FP64 chunk partials, column maxima
    DevBuf<double> gi_part, gi_colmax;
};

// non-rigid CPD (host_nonrigid.inl): dense G, or the low-rank factors of LowRankFactors
enum class NrStatus { none, dense, lowrank, ended };
struct NonRigidLoop {
    NrStatus status = NrStatus::none;
    const char* ended_by = nullptr;       // status == ended: the refusal, which names the call that ended the loop
    double lmd = 0.0;
    bool w_stale = false;                 // low-rank: W is formed on demand (cpd_nonrigid_get) from B, wgt, ts and lr.c
    bool prior_on = false;                // the correspondence priors of ConstrainedNonRigidCPD: alpha, p1t, pxt
    double alpha = 1.0;
    DevBuf<float> G;
    DevBuf<double> W, A, B, part;
    DevBuf<double> ts, ts2;               // the moved source T = Y + G W, and the next one while a step forms it (ts: 3 m, allocated last)
    DevBuf<double> wgt;                   // the weights of the last solve: nr_weight_kernel's with priors, else a copy of p1 (low-rank)
    DevBuf<int64_t> ipiv;
    DevBuf<int> info;                     // cuSOLVER's info
    DevBuf<double> p1t, pxt;
    bool live() const { return status == NrStatus::dense || status == NrStatus::lowrank; }
    void end(const char* why) { if (live()) { status = NrStatus::ended; ended_by = why; } }
};

// the BCPD registration loop (host_bcpd.inl): G^-1 (float32), the precision A and Sigma (FP64), all M x M in the internal order
enum class BcStatus { none, running, stopped };   // stopped: a step failed (LU, sigma2); the loop needs a new begin
struct BcpdLoop {
    BcStatus status = BcStatus::none;
    bool lowrank = false;                 // the K x K M-step on the factors of LowRankFactors (cpd_bcpd_lowrank_begin)
    long long m = 0;                      // source count of the last begin
    double sigma2 = 0.0;                  // host copy of the sigma2 the next E-step uses (culling decision)
    DevBuf<BcpdState> state;
    DevBuf<float> ginv;
    DevBuf<double> A, S, v, r, alpha, sdiag, part, sums;
    DevBuf<int64_t> ipiv;
    DevBuf<int> info;                     // [0] getrf's info, [1] getrs's
    // low-rank mode: the K x K system and C = its inverse, C Qt^T ([K][ld]), r in [3][m], w = C Rt (K x 3) and the pivots of the K x K LU
    DevBuf<double> sys, C, CQ, rt, w;
    DevBuf<int64_t> lr_ipiv;
    Event ev[6];
    float ms[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    // the dense loop's M x M buffers (and pivots), released before either begin allocates
    void release_dense() { ginv.reset(); A.reset(); S.reset(); ipiv.reset(); }
};

// GMMTree (host_gmmtree.inl, gmmtree.cuh): the tree (13 doubles per node), its prepared form (16) and the per-point work arrays
struct GmmTree {
    int levels = 0;                       // > 0: a tree is installed (cpd_gmmtree_build / cpd_gmmtree_load)
    long long total = 0, m = 0;           // nodes, source count of the last build (0: loaded)
    DevBuf<double> nodes, prep, pts, spts, g, part, mom, scr;
    DevBuf<unsigned> keys, keys2;
    DevBuf<int> idx, idx2, cur, start, end, asg;
    DevBuf<long long> seeds;
    DevBuf<unsigned char> sort;
    Event ev[7];
    float ms[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // build ms per level (up to 5), ms of the last registration E-step
};
}  // namespace

// ---------------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------------
struct cpd_ctx {
    // declared first, so destroyed last: the stream the handle created (none when the caller passed one)
    struct OwnedStream {
        cudaStream_t s = nullptr;
        ~OwnedStream() { if (s) cudaStreamDestroy(s); }
    } owned_stream;
    int device = 0, dim = 3, sm_count = 132, slots1 = 264, slots2 = 264;
    cudaStream_t stream = nullptr;
    long long m = 0, mpad = 0, n = 0, npad = 0, n_global = 0;
    DevBuf<double> d_yc, d_ts, d_xc, d_raw;
    DevBuf<float4> d_srcP, d_tgtP, d_tgtQ;
    DevBuf<P1Part> d_part1;
    DevBuf<double> d_part2;
    DevBuf<double> d_pt1, d_p1, d_pxc, d_px;
    DevBuf<double> d_mom_src, d_mom_tgt, d_mom, d_sums;
    DevBuf<DevState> d_state;
    DevState h_state;
    PinBuf<PinStage> pin;
    DevBuf<double> d_frame;             // [2][8]: what cloud_frame_kernel derives per cloud (sources, targets)
    PinBuf<double> h_stats;             // [2][9] pinned: the clouds' statistics on their way to the host (ensure_stats)
    Event stats_ev, copy_ev;
    int stats_pending = 0;              // bit 0: sources, bit 1: targets
    long long stats_count[2] = {0, 0};
    bool origin_given = false;
    int it1 = 0, it2 = 0, j1 = 1, j2 = 1, g1 = 1, g2 = 1;   // i-tiles, max partial slots per tile, work items (= grid)
    // exact culling of far blocks (late iterations): stage bounding boxes, per-stage max offset
    DevBuf<float4> d_sbox, d_tbox, d_ssub, d_tsub;
    DevBuf<float> d_omax, d_omax_sub;
    bool cull_on = true, cull_active = false;
    double extent = 0.0;              // largest bounding-box edge of the target shard (caller units)
    DevBuf<int4> d_work1, d_work2;
    DevBuf<int> d_slots1, d_slots2;
    bool have_source = false, have_target = false, prepared = false;
    EmStatus em = EmStatus::none;
    const char* em_ended_by = nullptr;    // em == ended: the call that ended the EM loop
    nccl_comm comm = nullptr;
    int world = 1, rank = 0;
    // Morton ordering (internal permutation; results leave in the caller's order)
    DevBuf<int> d_perm_src, d_perm_tgt, d_idx_tmp;
    DevBuf<unsigned> d_codes, d_codes_out;
    DevBuf<unsigned char> d_sort_tmp;
    DevBuf<double> d_outN, d_outM;      // staging for un-permuted outputs / permuted inputs
    // weighted E-step (BCPD): per-source exponent offsets (FP64 scratch, block minima, the float32 values the passes read) and
    // {log2 c, dead-column shift, la_min} for finalize 1; d_bc_es: {scale, sigma2, w} of a stand-alone cpd_bcpd_estep
    DevBuf<float> d_la;
    DevBuf<double> d_la64, d_la_part, d_bc_es;
    DevBuf<double> d_log2c;
    Solver sol;
    LowRankFactors lr;
    NonRigidLoop nr;
    BcpdLoop bc;
    GmmTree gt;
    DevBuf<P2PMailbox> d_box;             // this rank's mailbox (peers write into it)
    DevBuf<P2PInfo> d_p2p;                // device copy of the peer table; allocated => fused P2P exchange
    void* peer_ptr[P2P_MAX] = {nullptr};  // mappings opened with cudaIpcOpenMemHandle
    Event ev0, ev1, sev[7];
    bool profiling = false;
    int64_t launches = 0;
    // the fused EM iteration as a CUDA graph (cpd_em_step): one graph launch instead of 7-12 kernel launches per iteration
    PinBuf<DevState> h_state_ring;        // pinned staging slots of upload_state
    Event state_ev[8];
    int state_slot = 0;
    bool graph_on = true;
#ifndef CPD_HOST_EMU
    GraphExec em_graph;                   // dropped whenever a buffer or peer table it captured changes (drop_graph)
#endif
    bool em_graph_cull = false;           // the culling choice em_graph was captured with
    int em_graph_launches = 0;
    DevBuf<unsigned char> d_flush;
    std::vector<Event> pool;
};

namespace {
constexpr int STATE_RING = 8;
// A captured EM graph replays the pointers it was captured with: it is dropped whenever one of them may change.
inline void drop_graph(cpd_ctx* h) {
#ifndef CPD_HOST_EMU
    h->em_graph.reset();
#endif
    (void)h;
}

inline unsigned blocks_for(long long n) { return (unsigned)((n + THREADS - 1) / THREADS); }

// Work list of one pass: every i-tile is cut into J contiguous stage ranges ("splits"), one CTA each; J is chosen to
// minimise the makespan  ceil(ntiles*J / slots) * (ceil(nstages/J) + pipeline fill)  over the resident CTA slots, and slots
// left over in a single-wave launch go to extra splits of the first tiles.  All tiles carry the same work, so this is within
// one stage of the optimum whatever N, M and the GPU count are.  (A finer "stream-K" cut that lets one CTA span two tiles needs
// extra live state in the hot loops, which already sit at the 128-register cap.)
struct WorkList {
    std::vector<int4> items;        // {tile, first unit, end unit, slot within the tile}; a unit is a sub-chunk of SUB j-records
    std::vector<int> tile_slots;    // partial slots used per tile
    int max_slots = 1;
};
// Cut ntiles x nunits of work into CTA work items for `slots` resident CTAs.  A tile costs `nunits` (the last one, whose warps
// beyond the end of the i-points leave the kernel at once, `last_cost` = live warps / warps per CTA of that).  Two candidates:
//   * one wave (ntiles <= slots): every tile starts with one item; the next cut always goes to the tile whose longest item is the most
//     expensive, until the slots are used up -- cuts land where the cost is, at the granularity of a sub-chunk (an item may begin
//     and end inside a TMA stage; the kernels load the whole stages and skip the sub-chunks outside the item);
//   * several waves: the same number of cuts j for every tile, j chosen by waves x (item length + item overhead).
// `overhead`: what an item costs before its first unit (offset seeding sweep, pipeline fill), in units: half a stage.
WorkList build_work(int ntiles, int nunits, int slots, double last_cost, double overhead) {
    const double OVERHEAD = overhead;
    WorkList w;
    nunits = std::max(1, nunits);
    auto cost_of = [&](int t) { return t == ntiles - 1 ? last_cost : 1.0; };
    auto span_of = [&](int t, int j) { return cost_of(t) * (double)((nunits + j - 1) / j) + OVERHEAD; };
    // several waves, uniform j
    int best_j = 1;
    double best = 1e300;
    for (int j = 1; j <= nunits; ++j) {
        const long long items = (long long)ntiles * j;
        const double waves = ceil((double)items / slots);
        const double span = waves * ((double)((nunits + j - 1) / j) + OVERHEAD);
        if (span < best - 1e-9) { best = span; best_j = j; }
        if (items > 8LL * slots) break;
    }
    w.tile_slots.assign(ntiles, best_j);
    if (ntiles <= slots) {
        // one wave, cuts by cost
        std::vector<int> cuts(ntiles, 1);
        int used = ntiles;
        while (used < slots) {
            int worst = -1;
            double wv = -1.0;
            for (int t = 0; t < ntiles; ++t) {
                const double v = span_of(t, cuts[t]);
                if (cuts[t] < nunits && v > wv) { wv = v; worst = t; }
            }
            if (worst < 0) break;
            ++cuts[worst];
            ++used;
        }
        double span = 0.0;
        for (int t = 0; t < ntiles; ++t) span = std::max(span, span_of(t, cuts[t]));
        if (span <= best + 1e-9) w.tile_slots = cuts;
    }
    for (int t = 0; t < ntiles; ++t) {
        const int j = w.tile_slots[t];
        for (int s = 0; s < j; ++s) {
            const int a = (int)((long long)nunits * s / j), b = (int)((long long)nunits * (s + 1) / j);
            w.items.push_back(make_int4(t, a, b, s));
        }
        w.max_slots = std::max(w.max_slots, j);
    }
    // longest (most expensive) first: the hardware hands CTAs out in order
    std::stable_sort(w.items.begin(), w.items.end(), [&](const int4& a, const int4& b) {
        return cost_of(a.x) * (a.z - a.y) > cost_of(b.x) * (b.z - b.y);
    });
    return w;
}

// Stream-ordered, no synchronise: the state goes through a small ring of pinned staging slots (a cudaMemcpyAsync from pageable
// memory would synchronise the stream first); a slot is re-used only after the copy that last read it has completed.
int ensure_stats(cpd_ctx* h);
int upload_state(cpd_ctx* h) {
    TRY(ensure_stats(h));
    if (!h->h_state_ring.p) {
        TRY(h->h_state_ring.alloc(STATE_RING));
        for (Event& e : h->state_ev) CU(cudaEventCreateWithFlags(&e.e, cudaEventDisableTiming));
    }
    const int k = h->state_slot;
    h->state_slot = (k + 1) % STATE_RING;
    CU(cudaEventSynchronize(h->state_ev[k]));                  // never recorded: returns at once
    h->h_state_ring.p[k] = h->h_state;
    CU(cudaMemcpyAsync(h->d_state.p, &h->h_state_ring.p[k], sizeof(DevState), cudaMemcpyHostToDevice, h->stream));
    CU(cudaEventRecord(h->state_ev[k], h->stream));
    return CPD_OK;
}

// copy a host cloud (count x dim doubles) into a device count x 3 array
int upload_cloud(cpd_ctx* h, const double* src, long long count, double* dst3) {
    if (h->dim == 3) {
        CU(cudaMemcpyAsync(dst3, src, (size_t)count * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    } else {
        CU(cudaMemsetAsync(dst3, 0, (size_t)count * 3 * sizeof(double), h->stream));
        CU(cudaMemcpy2DAsync(dst3, 3 * sizeof(double), src, 2 * sizeof(double), 2 * sizeof(double), (size_t)count,
                             cudaMemcpyHostToDevice, h->stream));
    }
    return CPD_OK;
}
int download_cloud(cpd_ctx* h, const double* src3, long long count, double* dst) {
    if (h->dim == 3) {
        CU(cudaMemcpyAsync(dst, src3, (size_t)count * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    } else {
        CU(cudaMemcpy2DAsync(dst, 2 * sizeof(double), src3, 3 * sizeof(double), 2 * sizeof(double), (size_t)count,
                             cudaMemcpyDeviceToHost, h->stream));
    }
    return CPD_OK;
}
// a per-source device array (cols 1 or 3, internal order) into the caller's order at `out`; returns once it has arrived
int download_src(cpd_ctx* h, const double* d, int cols, double* out) {
    scatter_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(d, h->d_perm_src.p, h->m, cols, h->d_outM.p);
    KCHECK();
    h->launches += 1;
    if (cols == 3) TRY(download_cloud(h, h->d_outM.p, h->m, out));
    else CU(cudaMemcpyAsync(out, h->d_outM.p, (size_t)h->m * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));        // d_outM is reused
    return CPD_OK;
}

// d_out[0] = sum |p|^2, d_out[1..3] = sum p   over a device count x 3 cloud; stays on the device (stream-ordered, no sync).
// `part`: blocks_for(count) * 4 doubles of scratch.
int cloud_sums_dev(cpd_ctx* h, const double* d_pts, long long count, double* part, double* d_out) {
    const unsigned nb = blocks_for(count);
    cloud_sums_kernel<<<nb, THREADS, 0, h->stream>>>(d_pts, count, part);
    reduce_cols_kernel<<<1, 4 * 32, 0, h->stream>>>(part, (int)nb, 4, d_out);
    KCHECK();
    h->launches += 2;
    return CPD_OK;
}

// A cloud's way into the library, one stream-ordered sequence without a host round trip: upload -> nine statistics (sums, minima,
// maxima) -> frame (cloud_frame_kernel: Morton box, origin; origin and count patched into the device state) -> Morton sort ->
// out[k] = raw[perm[k]] - origin.  The host copy of the statistics travels behind (pinned h_stats, stats_ev) and is read by
// ensure_stats() when the host first needs the centroid or the extent.  The call returns once the upload itself has been
// consumed (copy_ev), so the caller's buffer is free again, as before.
int ingest_cloud(cpd_ctx* h, const double* host_pts, long long count, int is_target, long long n_global, const double* origin,
                 int* d_perm, double* d_out) {
    TRY(h->d_raw.reserve((size_t)count * 3));
    const unsigned nb = blocks_for(count);
    TRY(h->d_sums.reserve((size_t)nb * 9 + 16));
    TRY(h->d_codes.reserve((size_t)count));
    TRY(h->d_codes_out.reserve((size_t)count));
    TRY(h->d_idx_tmp.reserve((size_t)count));
    size_t need = 0;
    CU(cub::DeviceRadixSort::SortPairs(nullptr, need, h->d_codes.p, h->d_codes_out.p, h->d_idx_tmp.p, d_perm, (int)count, 0, 30, h->stream));
    TRY(h->d_sort_tmp.reserve(need));
    TRY(upload_cloud(h, host_pts, count, h->d_raw.p));
    CU(cudaEventRecord(h->copy_ev, h->stream));
    double* frame = h->d_frame.p + 8 * is_target;
    stats_kernel<<<nb, THREADS, 0, h->stream>>>(h->d_raw.p, count, h->d_sums.p + 16);
    stats_fold_kernel<<<1, 288, 0, h->stream>>>(h->d_sums.p + 16, (int)nb, h->d_sums.p);
    cloud_frame_kernel<<<1, 32, 0, h->stream>>>(h->d_sums.p, count, is_target, n_global, origin != nullptr, origin ? origin[0] : 0.0,
                                                origin ? origin[1] : 0.0, origin ? origin[2] : 0.0, h->d_state.p, frame);
    CU(cudaMemcpyAsync(h->h_stats.p + 9 * is_target, h->d_sums.p, 9 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaEventRecord(h->stats_ev, h->stream));
    h->stats_pending |= 1 << is_target;
    h->stats_count[is_target] = count;
    morton_frame_kernel<<<nb, THREADS, 0, h->stream>>>(h->d_raw.p, count, frame, h->d_codes.p, h->d_idx_tmp.p);
    CU(cub::DeviceRadixSort::SortPairs(h->d_sort_tmp.p, need, h->d_codes.p, h->d_codes_out.p, h->d_idx_tmp.p, d_perm, (int)count, 0, 30,
                                       h->stream));
    gather3_frame_kernel<<<nb, THREADS, 0, h->stream>>>(h->d_raw.p, d_perm, count, frame, d_out);
    KCHECK();
    h->launches += 6;
    CU(cudaEventSynchronize(h->copy_ev));
    return CPD_OK;
}

// The host's copy of what cloud_frame_kernel derived on the device (centroid of the sources, frame origin and extent of the targets).
// Every entry point that reads h_state.cx / cy or h->extent, or uploads the host state, calls this first.
int ensure_stats(cpd_ctx* h) {
    if (!h->stats_pending) return CPD_OK;
    CU(cudaEventSynchronize(h->stats_ev));
    if (h->stats_pending & 1)
        for (int a = 0; a < 3; ++a) h->h_state.cy[a] = h->h_stats.p[a] / (double)h->stats_count[0];
    if (h->stats_pending & 2) {
        const double* t = h->h_stats.p + 9;
        if (!h->origin_given) for (int a = 0; a < 3; ++a) h->h_state.cx[a] = t[a] / (double)h->stats_count[1];
        h->extent = std::max(t[6] - t[3], std::max(t[7] - t[4], t[8] - t[5]));
    }
    h->stats_pending = 0;
    return CPD_OK;
}

int require_clouds(cpd_ctx* h) {
    if (!h->have_source || !h->have_target) return fail(CPD_ERR_STATE, "source and target must both be set");
    return CPD_OK;
}

// culling for an E-step at sigma2: a point reaches ~13.3 sigma (2^-127); culling can only pay once that is well inside the cloud
int decide_cull(cpd_ctx* h, double sigma2) {
    TRY(ensure_stats(h));
    h->cull_active = h->extent > 0.0 && 13.3 * sqrt(sigma2) < 0.25 * h->extent;
    return CPD_OK;
}

int prepare(cpd_ctx* h) {
    TRY(ensure_stats(h));
    if (h->prepared) return CPD_OK;
    TRY(require_clouds(h));
    h->it1 = (int)((h->n + ITILE1 - 1) / ITILE1);
    h->it2 = (int)((h->m + ITILE2 - 1) / ITILE2);
    // Pass 1 cuts at sub-chunks, and the warps of its last i-tile whose i-points are all padding leave the kernel at once.  Such a
    // tile is planned at max(0.6, live warps / 8) of a full tile, not live / 8: the live warps get a larger share of the SM's pipes,
    // but a warp on its own is latency-bound.  Pass 2 keeps whole stages as the unit (its kernel is the one closest to the register
    // limit).  The 0.6 and the units are not tuned for the H100; CPD_B200_PLAN_LAST_COST and CPD_B200_PLAN_UNIT switch them.
    const long long in_last = h->n - (long long)(h->it1 - 1) * ITILE1;
    const int live = (int)((in_last + 32 * RI1 - 1) / (32 * RI1));          // warps of the last tile that hold i-points
    double last_cost = live < THREADS / 32 ? std::max(0.6, live / (double)(THREADS / 32)) : 1.0;
    if (const char* e = getenv("CPD_B200_PLAN_LAST_COST")) { const double v = atof(e); if (v > 0.0 && v <= 1.0) last_cost = v; }   // tuning
    WorkList w1;
    if (const char* e = getenv("CPD_B200_PLAN_UNIT"); e && !strcmp(e, "stage")) {      // tuning: items of whole stages, as pass 2
        w1 = build_work(h->it1, (int)(h->mpad / P1_STAGE), h->slots1, last_cost, 0.5);
        for (int4& it : w1.items) { it.y *= P1_STAGE / SUB; it.z *= P1_STAGE / SUB; }
    } else {
        w1 = build_work(h->it1, (int)(h->mpad / SUB), h->slots1, last_cost, 0.5 * (P1_STAGE / SUB));
    }
    const WorkList w2 = build_work(h->it2, (int)(h->npad / P2_STAGE), h->slots2, 1.0, 0.5);
    h->j1 = w1.max_slots; h->g1 = (int)w1.items.size();
    h->j2 = w2.max_slots; h->g2 = (int)w2.items.size();
    TRY(h->d_work1.alloc(w1.items.size()));
    TRY(h->d_work2.alloc(w2.items.size()));
    TRY(h->d_slots1.alloc(w1.tile_slots.size()));
    TRY(h->d_slots2.alloc(w2.tile_slots.size()));
    // on the handle's (non-blocking) stream, which the consuming kernels run on; the vectors live until the synchronise below
    CU(cudaMemcpyAsync(h->d_work1.p, w1.items.data(), w1.items.size() * sizeof(int4), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_work2.p, w2.items.data(), w2.items.size() * sizeof(int4), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_slots1.p, w1.tile_slots.data(), w1.tile_slots.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_slots2.p, w2.tile_slots.data(), w2.tile_slots.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    TRY(h->d_sbox.alloc((size_t)(h->mpad / P1_STAGE) * 2));
    TRY(h->d_tbox.alloc((size_t)(h->npad / P2_STAGE) * 2));
    TRY(h->d_omax.alloc((size_t)(h->npad / P2_STAGE)));
    TRY(h->d_ssub.alloc((size_t)(h->mpad / SUB) * 2));
    TRY(h->d_tsub.alloc((size_t)(h->npad / SUB) * 2));
    TRY(h->d_omax_sub.alloc((size_t)(h->npad / SUB)));
    const size_t need1 = (size_t)h->j1 * h->n, need2 = (size_t)h->j2 * h->m * 4;
    TRY(h->d_part1.reserve(need1));
    TRY(h->d_part2.reserve(need2));
    const size_t ms = (size_t)blocks_for(h->m) * MOM_SRC, mt = (size_t)blocks_for(h->npad) * MOM_TGT;   // MOM_* >= RM_*
    TRY(h->d_mom_src.reserve(ms));
    TRY(h->d_mom_tgt.reserve(mt));
    h->prepared = true;
    drop_graph(h);
    return CPD_OK;
}

int allreduce(cpd_ctx* h, double* buf, size_t count) {
    if (!h->comm) return CPD_OK;
    NC(g_nccl.AllReduce(buf, buf, count, NCCL_DOUBLE, NCCL_SUM, h->comm, h->stream));
    return CPD_OK;
}

// a profiling event (cpd_set_profiling)
inline void mark(cpd_ctx* h, cudaEvent_t e) {
    if (h->profiling) cudaEventRecord(e, h->stream);
}

// pack + pass 1 + finalize 1 + pass 2 + finalize 2; sigma2/w read from the given device scalars; wgt: with the per-source
// exponents of bcpd_weights (BCPD)
int launch_estep(cpd_ctx* h, const double* d_sigma2, const double* d_w, const double* d_ts, bool wgt) {
    TRY(prepare(h));
    const long long cover = std::max(h->mpad, h->n);
    mark(h, h->sev[0]);
    pack_kernel<<<blocks_for(cover), THREADS, 0, h->stream>>>(h->d_state.p, d_sigma2, h->d_yc.p, d_ts, h->d_xc.p, h->m, h->mpad,
                                                              h->n, h->d_srcP.p, h->d_tgtP.p);
    mark(h, h->sev[1]);
    const bool cull = h->cull_on && h->cull_active;
    const int nst1 = (int)(h->mpad / P1_STAGE);
    stage_bbox_kernel<<<(unsigned)nst1, THREADS, 0, h->stream>>>(h->d_srcP.p, (int)h->m, P1_STAGE, h->d_sbox.p);   // offset seeding (always)
    h->launches += 1;
    const int nsub1 = (int)(h->mpad / SUB), nsub2 = (int)(h->npad / SUB);
    if (cull) {
        stage_bbox_kernel<<<(unsigned)(h->npad / P2_STAGE), THREADS, 0, h->stream>>>(h->d_tgtP.p, (int)h->n, P2_STAGE, h->d_tbox.p);
        sub_bbox_kernel<<<(unsigned)((nsub1 + 7) / 8), THREADS, 0, h->stream>>>(h->d_srcP.p, (int)h->m, nsub1, h->d_ssub.p);
        sub_bbox_kernel<<<(unsigned)((nsub2 + 7) / 8), THREADS, 0, h->stream>>>(h->d_tgtP.p, (int)h->n, nsub2, h->d_tsub.p);
        h->launches += 3;
    }
    if (wgt) {
        weight_patch_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_la.p, h->m, h->d_srcP.p);
        h->launches += 1;
    }
#define CPD_PASS1(C, W) pass1_kernel<C, W><<<h->g1, THREADS, PASS1_SMEM, h->stream>>>(h->d_tgtP.p, (int)h->n, h->d_srcP.p, h->d_work1.p, h->d_part1.p, h->d_sbox.p, nst1, (C) ? h->d_ssub.p : nullptr)
    if (cull) { if (wgt) CPD_PASS1(true, true); else CPD_PASS1(true, false); }
    else { if (wgt) CPD_PASS1(false, true); else CPD_PASS1(false, false); }
#undef CPD_PASS1
    mark(h, h->sev[2]);
    finalize1_kernel<<<blocks_for(h->npad), THREADS, 0, h->stream>>>(h->d_state.p, d_sigma2, d_w, h->d_part1.p, h->d_slots1.p, (int)h->n,
                                                                     h->d_tgtP.p, h->d_tgtQ.p, h->npad, h->d_pt1.p, h->d_mom_tgt.p,
                                                                     wgt ? h->d_log2c.p : nullptr);
    mark(h, h->sev[3]);
    if (cull) {
        stage_omax_kernel<<<(unsigned)(h->npad / P2_STAGE), THREADS, 0, h->stream>>>(h->d_tgtQ.p, h->d_omax.p);
        sub_omax_kernel<<<(unsigned)((nsub2 + 7) / 8), THREADS, 0, h->stream>>>(h->d_tgtQ.p, nsub2, h->d_omax_sub.p);
        h->launches += 2;
    }
#define CPD_PASS2(C, W) pass2_kernel<C, W><<<h->g2, THREADS, PASS2_SMEM, h->stream>>>(h->d_srcP.p, (int)h->m, h->d_tgtQ.p, h->d_work2.p, h->d_part2.p, (C) ? h->d_tbox.p : nullptr, (C) ? h->d_omax.p : nullptr, (C) ? h->d_tsub.p : nullptr, (C) ? h->d_omax_sub.p : nullptr)
    if (cull) { if (wgt) CPD_PASS2(true, true); else CPD_PASS2(true, false); }
    else { if (wgt) CPD_PASS2(false, true); else CPD_PASS2(false, false); }
#undef CPD_PASS2
    mark(h, h->sev[4]);
    finalize2_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_state.p, d_sigma2, h->d_part2.p, h->d_slots2.p, (int)h->m, h->d_yc.p,
                                                                  d_ts, h->d_p1.p, h->d_pxc.p, h->d_mom_src.p);
    mark(h, h->sev[5]);
    mark(h, h->sev[6]);          // E-step-only callers end here; cpd_em_step / cpd_nonrigid_step record event 6 again after their M-step
    KCHECK();
    h->launches += 5;
    return CPD_OK;
}

int read_params(cpd_ctx* h, cpd_params* out) {
    const DevState& s = h->pin.p->state;
    CU(cudaMemcpyAsync(&h->pin.p->state, h->d_state.p, sizeof(DevState), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    if (s.err)
        return fail(CPD_ERR_STATE, "a peer rank did not deliver its moments within the P2P exchange timeout");
    const int d = h->dim;
    for (int i = 0; i < 9; ++i) out->lin[i] = 0.0;
    for (int i = 0; i < d; ++i)
        for (int j = 0; j < d; ++j) out->lin[i * d + j] = s.lin[3 * i + j];
    for (int i = 0; i < 3; ++i) out->t[i] = (i < d) ? s.t[i] : 0.0;
    out->scale = s.scale;
    out->sigma2 = s.sigma2;
    TRY(decide_cull(h, out->sigma2));
    out->q = s.q;
    out->n_p = s.n_p;
    return CPD_OK;
}
}  // namespace

// Host-only view of the work list a pass would be launched with (no device needed): lets the CPU tests check that
// every (tile, unit) is covered exactly once and how well the resident CTA slots are filled.
extern "C" int cpd_plan_work(int ntiles, int nunits, int slots, double last_tile_cost, int* items /* 4 ints each, may be NULL */,
                             int capacity, int* n_items, int* max_slots) {
    if (ntiles < 1 || nunits < 1 || slots < 1 || !(last_tile_cost > 0.0 && last_tile_cost <= 1.0) || !n_items || !max_slots)
        return fail(CPD_ERR_ARG, "bad argument");
    const WorkList w = build_work(ntiles, nunits, slots, last_tile_cost, 0.5 * (P1_STAGE / SUB));     // pass 1's units
    *n_items = (int)w.items.size();
    *max_slots = w.max_slots;
    if (items) {
        if (capacity < (int)w.items.size()) return fail(CPD_ERR_ARG, "capacity %d < %d work items", capacity, (int)w.items.size());
        for (size_t i = 0; i < w.items.size(); ++i) {
            items[4 * i] = w.items[i].x; items[4 * i + 1] = w.items[i].y; items[4 * i + 2] = w.items[i].z; items[4 * i + 3] = w.items[i].w;
        }
    }
    return CPD_OK;
}

extern "C" int cpd_create(cpd_ctx** out, int device, int dim, void* stream) {
    if (!out) return fail(CPD_ERR_ARG, "out is NULL");
    if (dim != 2 && dim != 3) return fail(CPD_ERR_ARG, "dim must be 2 or 3, got %d", dim);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(CPD_ERR_CUDA, "no CUDA device: this library has no CPU path");
    }
    if (device < 0 || device >= ndev) return fail(CPD_ERR_ARG, "device %d out of range (%d visible)", device, ndev);
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(CPD_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a (Hopper) only", device, prop.major, prop.minor);
    std::unique_ptr<cpd_ctx> h(new cpd_ctx());
    h->device = device;
    h->dim = dim;
    h->sm_count = prop.multiProcessorCount;
    if (stream) h->stream = (cudaStream_t)stream;
    else { CU(cudaStreamCreateWithFlags(&h->owned_stream.s, cudaStreamNonBlocking)); h->stream = h->owned_stream.s; }
    CU(cudaFuncSetAttribute(pass1_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS1_SMEM));
    CU(cudaFuncSetAttribute(pass2_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS2_SMEM));
    CU(cudaFuncSetAttribute(pass1_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS1_SMEM));
    CU(cudaFuncSetAttribute(pass2_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS2_SMEM));
    CU(cudaFuncSetAttribute(pass1_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS1_SMEM));
    CU(cudaFuncSetAttribute(pass2_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS2_SMEM));
    CU(cudaFuncSetAttribute(pass1_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS1_SMEM));
    CU(cudaFuncSetAttribute(pass2_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PASS2_SMEM));
    int occ1 = 0, occ2 = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, pass1_kernel<false, false>, THREADS, PASS1_SMEM));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, pass2_kernel<false, false>, THREADS, PASS2_SMEM));
    h->slots1 = h->sm_count * std::max(1, occ1);
    h->slots2 = h->sm_count * std::max(1, occ2);
    TRY(h->d_state.alloc(1));
    TRY(h->d_mom.alloc((size_t)MOM_PAD));
    TRY(h->pin.alloc(1));
    TRY(h->d_frame.alloc(16));
    TRY(h->h_stats.alloc(18));
    CU(cudaEventCreateWithFlags(&h->stats_ev.e, cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&h->copy_ev.e, cudaEventDisableTiming));
    CU(cudaEventCreate(&h->ev0.e));
    CU(cudaEventCreate(&h->ev1.e));
    for (Event& e : h->sev) CU(cudaEventCreate(&e.e));
    { const char* e = getenv("CPD_B200_NO_CULL"); h->cull_on = !(e && e[0] == '1'); }
    { const char* e = getenv("CPD_B200_NO_GRAPH"); h->graph_on = !(e && e[0] == '1'); }
    memset(&h->h_state, 0, sizeof(DevState));
    h->h_state.dim = dim;
    h->h_state.scale = 1.0;
    h->h_state.lin[0] = h->h_state.lin[4] = h->h_state.lin[8] = 1.0;
    h->h_state.update_scale = 1;
    TRY(upload_state(h.get()));      // the device state starts as a copy of the host's (cloud_frame_kernel patches single fields)
    *out = h.release();
    return CPD_OK;
}

extern "C" void cpd_destroy(cpd_ctx* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    for (void* p : h->peer_ptr) if (p) cudaIpcCloseMemHandle(p);
    delete h;                        // every buffer, pinned block, event, graph and the solver; the stream the handle created last
}

extern "C" int cpd_set_source(cpd_ctx* h, const double* source, int64_t m) {
    if (!h || !source) return fail(CPD_ERR_ARG, "null argument");
    if (m < 1 || m > 0x7fffffffLL - 65536) return fail(CPD_ERR_ARG, "source count %lld out of range", (long long)m);
    CU(cudaSetDevice(h->device));
    if (m != h->m || !h->d_yc.p) {
        h->m = m;
        h->mpad = (m + P1_STAGE - 1) / P1_STAGE * P1_STAGE;
        TRY(h->d_yc.alloc((size_t)m * 3));
        TRY(h->d_ts.alloc((size_t)m * 3));
        TRY(h->d_srcP.alloc((size_t)h->mpad));
        TRY(h->d_p1.alloc((size_t)m));
        TRY(h->d_pxc.alloc((size_t)m * 3));
        TRY(h->d_px.alloc((size_t)m * 3));
        TRY(h->d_perm_src.alloc((size_t)m));
        TRY(h->d_outM.alloc((size_t)m * 3));
        h->prepared = false;
        if (h->nr.live()) h->nr.status = NrStatus::none;
    }
    TRY(ingest_cloud(h, source, m, 0, 0, nullptr, h->d_perm_src.p, h->d_yc.p));
    h->bc.status = BcStatus::none;       // a BCPD loop starts from its own cpd_set_source + cpd_bcpd_begin
    h->h_state.m = m;
    h->have_source = true;
    return CPD_OK;
}

extern "C" int cpd_set_target(cpd_ctx* h, const double* target, int64_t n_local, int64_t n_global, const double* frame_origin) {
    if (!h || !target) return fail(CPD_ERR_ARG, "null argument");
    if (n_local < 1 || n_local > 0x7fffffffLL - 65536) return fail(CPD_ERR_ARG, "target count %lld out of range", (long long)n_local);
    if (n_global < n_local) return fail(CPD_ERR_ARG, "n_global (%lld) < n_local (%lld)", (long long)n_global, (long long)n_local);
    if (!frame_origin && n_global != n_local) return fail(CPD_ERR_ARG, "a sharded target needs an explicit frame_origin");
    CU(cudaSetDevice(h->device));
    if (n_local != h->n || !h->d_xc.p) {
        h->n = n_local;
        h->npad = (n_local + P2_STAGE - 1) / P2_STAGE * P2_STAGE;
        TRY(h->d_xc.alloc((size_t)n_local * 3));
        TRY(h->d_tgtP.alloc((size_t)n_local));
        TRY(h->d_tgtQ.alloc((size_t)h->npad * 2));
        TRY(h->d_pt1.alloc((size_t)n_local));
        TRY(h->d_perm_tgt.alloc((size_t)n_local));
        TRY(h->d_outN.alloc((size_t)n_local));
        h->prepared = false;
    }
    h->n_global = n_global;
    double origin[3] = {0.0, 0.0, 0.0};
    if (frame_origin) for (int a = 0; a < h->dim; ++a) origin[a] = frame_origin[a];
    h->origin_given = frame_origin != nullptr;
    if (h->origin_given) for (int a = 0; a < 3; ++a) h->h_state.cx[a] = origin[a];
    TRY(ingest_cloud(h, target, n_local, 1, n_global, frame_origin ? origin : nullptr, h->d_perm_tgt.p, h->d_xc.p));
    h->h_state.n_global = n_global;
    h->have_target = true;
    return CPD_OK;
}

extern "C" int cpd_sigma2_init(cpd_ctx* h, double* sigma2) {
    if (!h || !sigma2) return fail(CPD_ERR_ARG, "null argument");
    TRY(require_clouds(h));
    CU(cudaSetDevice(h->device));
    // target sums (summed over the ranks on the device), source sums, ONE read-back: a single host synchronisation
    double sx[4], sy[4];
    const size_t pn = (size_t)blocks_for(h->n) * 4, pm = (size_t)blocks_for(h->m) * 4;
    TRY(h->d_sums.reserve(16 + pn + pm));
    TRY(cloud_sums_dev(h, h->d_xc.p, h->n, h->d_sums.p + 16, h->d_sums.p));
    if (h->comm) TRY(allreduce(h, h->d_sums.p, 4));
    TRY(cloud_sums_dev(h, h->d_yc.p, h->m, h->d_sums.p + 16 + pn, h->d_sums.p + 4));
    CU(cudaMemcpyAsync(h->pin.p->sums, h->d_sums.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    TRY(ensure_stats(h));
    for (int k = 0; k < 4; ++k) { sx[k] = h->pin.p->sums[k]; sy[k] = h->pin.p->sums[4 + k]; }
    *sigma2 = sigma2_closed_form(sx, sy, h->h_state.cx, h->h_state.cy, (double)h->m, (double)h->n_global, h->dim);
    return CPD_OK;
}

extern "C" int cpd_set_state(cpd_ctx* h, int tf_kind, int update_scale, double w, const cpd_params* init) {
    if (!h || !init) return fail(CPD_ERR_ARG, "null argument");
    if (tf_kind != CPD_TF_RIGID && tf_kind != CPD_TF_AFFINE) return fail(CPD_ERR_ARG, "tf_kind %d not supported by the fused EM loop", tf_kind);
    if (!(w >= 0.0 && w < 1.0)) return fail(CPD_ERR_ARG, "w must be in [0, 1), got %g", w);
    if (!(init->sigma2 > 0.0)) return fail(CPD_ERR_ARG, "sigma2 must be positive, got %g", init->sigma2);
    CU(cudaSetDevice(h->device));
    DevState& s = h->h_state;
    const int d = h->dim;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) s.lin[3 * i + j] = (i < d && j < d) ? init->lin[i * d + j] : (i == j ? 1.0 : 0.0);
    for (int i = 0; i < 3; ++i) s.t[i] = (i < d) ? init->t[i] : 0.0;
    s.scale = (tf_kind == CPD_TF_RIGID) ? init->scale : 1.0;
    s.sigma2 = init->sigma2;
    s.q = init->q;
    s.n_p = 0.0;
    s.w = w;
    s.tf_kind = tf_kind;
    s.update_scale = update_scale ? 1 : 0;
    s.dim = d;
    TRY(decide_cull(h, init->sigma2));
    h->em = EmStatus::live;
    h->nr.end("cpd_set_state ended the non-rigid loop of this handle: call cpd_nonrigid_*begin again");
    return upload_state(h);
}

namespace {
// the refusal of an EM step without a live EM loop
int em_check(cpd_ctx* h) {
    if (h->em == EmStatus::none) return fail(CPD_ERR_STATE, "cpd_set_state has not been called");
    if (h->em == EmStatus::ended)
        return fail(CPD_ERR_STATE, "%s ended the rigid/affine EM loop of this handle: call cpd_set_state again", h->em_ended_by);
    return CPD_OK;
}
// the launches of one fused EM iteration, in stream order (also what a graph capture records)
int em_step_launches(cpd_ctx* h) {
    TRY(launch_estep(h, &h->d_state.p->sigma2, &h->d_state.p->w, nullptr, false));
    const int nbs = (int)blocks_for(h->m), nbt = (int)blocks_for(h->npad);
    if (h->d_p2p.p) {
        moments_p2p_kernel<<<1, 256, 0, h->stream>>>(h->d_state.p, h->d_mom_src.p, nbs, RM_SRC, h->d_mom_tgt.p, nbt, RM_TGT, h->d_mom.p,
                                                     h->d_p2p.p);
        h->launches += 1;
    } else if (h->comm) {
        moments_kernel<0><<<1, 256, 0, h->stream>>>(h->d_state.p, h->d_mom_src.p, nbs, RM_SRC, h->d_mom_tgt.p, nbt, RM_TGT, h->d_mom.p);
        TRY(allreduce(h, h->d_mom.p, MOM_PAD));
        mstep_residual_kernel<<<1, 32, 0, h->stream>>>(h->d_state.p, h->d_mom.p);
        h->launches += 2;
    } else {
        moments_kernel<1><<<1, 256, 0, h->stream>>>(h->d_state.p, h->d_mom_src.p, nbs, RM_SRC, h->d_mom_tgt.p, nbt, RM_TGT, h->d_mom.p);
        h->launches += 1;
    }
    mark(h, h->sev[6]);
    KCHECK();
    return CPD_OK;
}
}  // namespace

// One EM iteration (probreg/cpd.py:111-113).  The launch sequence is fixed per {culling on/off, buffer generation}, so it is
// captured once into a CUDA graph and replayed: one graph launch per iteration.  Not captured: profiling runs (events between
// the kernels) and the ncclAllReduce variant of the multi-rank exchange (CPD_B200_NO_P2P=1); CPD_B200_NO_GRAPH=1 turns it off.
extern "C" int cpd_em_step(cpd_ctx* h, cpd_params* out) {
    if (!h) return fail(CPD_ERR_ARG, "null handle");
    TRY(em_check(h));
    CU(cudaSetDevice(h->device));
#ifndef CPD_HOST_EMU
    const bool use_graph = h->graph_on && !h->profiling && !(h->comm && !h->d_p2p.p);
#else
    const bool use_graph = false;
#endif
    if (!use_graph) {
        TRY(em_step_launches(h));
    }
#ifndef CPD_HOST_EMU
    else {
        TRY(prepare(h));                                    // allocations and uploads happen outside the capture
        const bool cull = h->cull_on && h->cull_active;
        if (!h->em_graph || h->em_graph_cull != cull) {
            h->em_graph.reset();
            const int64_t before = h->launches;
            cudaGraph_t g = nullptr;
            CU(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
            const int rc = em_step_launches(h);
            const cudaError_t ce = cudaStreamEndCapture(h->stream, &g);
            h->em_graph_launches = (int)(h->launches - before);
            h->launches = before;
            if (rc != CPD_OK) { if (g) cudaGraphDestroy(g); return rc; }
            if (ce != cudaSuccess) return fail(CPD_ERR_CUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(ce));
            cudaGraphExec_t exec = nullptr;
            const cudaError_t ie = cudaGraphInstantiate(&exec, g, 0);
            cudaGraphDestroy(g);
            if (ie != cudaSuccess) return fail(CPD_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ie));
            h->em_graph.reset(exec);
            h->em_graph_cull = cull;
        }
        CU(cudaGraphLaunch(h->em_graph.get(), h->stream));
        h->launches += h->em_graph_launches;                // kernels executed, whatever carried them to the device
    }
#endif
    if (out) return read_params(h, out);
    return CPD_OK;
}

extern "C" int cpd_em_run(cpd_ctx* h, int maxiter, double tol, cpd_params* out, int* iters_run, double* trace) {
    if (!h || !out) return fail(CPD_ERR_ARG, "null argument");
    TRY(em_check(h));
    double q = h->h_state.q;
    int it = 0;
    cpd_params cur;
    memset(&cur, 0, sizeof(cur));
    for (it = 0; it < maxiter; ++it) {
        TRY(cpd_em_step(h, &cur));
        if (trace) { trace[2 * it] = cur.sigma2; trace[2 * it + 1] = cur.q; }
        if (fabs(cur.q - q) < tol) { ++it; break; }          // cpd.py:117
        q = cur.q;
    }
    if (maxiter <= 0) TRY(read_params(h, &cur));
    *out = cur;
    if (iters_run) *iters_run = it;
    return CPD_OK;
}

namespace {
// The stand-alone E-step at the caller's moved source, sigma2 and w (weighted: with the exponents bcpd_weights formed) into the
// E-step's buffers, summed over the ranks
int run_estep(cpd_ctx* h, const double* t_source, double sigma2, double w, bool weighted) {
    TRY(h->d_raw.reserve((size_t)h->m * 3));
    TRY(upload_cloud(h, t_source, h->m, h->d_raw.p));
    gather3_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_raw.p, h->d_perm_src.p, h->m, 0.0, 0.0, 0.0, h->d_ts.p);
    h->launches += 1;
    TRY(decide_cull(h, sigma2));
    h->pin.p->es[0] = sigma2;
    h->pin.p->es[1] = w;
    CU(cudaMemcpyAsync(&h->d_state.p->es_sigma2, h->pin.p->es, 2 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    TRY(launch_estep(h, &h->d_state.p->es_sigma2, &h->d_state.p->es_w, h->d_ts.p, weighted));
    if (h->comm) {
        TRY(allreduce(h, h->d_p1.p, (size_t)h->m));
        TRY(allreduce(h, h->d_pxc.p, (size_t)h->m * 3));
    }
    return CPD_OK;
}
}  // namespace

extern "C" int cpd_estep(cpd_ctx* h, const double* t_source, double sigma2, double w, double* pt1, double* p1, double* px, double* n_p) {
    if (!h || !t_source) return fail(CPD_ERR_ARG, "null argument");
    if (!(sigma2 > 0.0)) return fail(CPD_ERR_ARG, "sigma2 must be positive, got %g", sigma2);
    if (!(w >= 0.0 && w < 1.0)) return fail(CPD_ERR_ARG, "w must be in [0, 1), got %g", w);
    TRY(require_clouds(h));
    CU(cudaSetDevice(h->device));
    TRY(run_estep(h, t_source, sigma2, w, false));
    return cpd_last_estep(h, pt1, p1, px, n_p);
}

namespace {
// The per-source exponents of the weighted E-step, on the device: la_m = -log2(weight_m) in FP64 (bcpd_la_kernel), their minimum,
// the constants of finalize 1 (bcpd_la_finish_kernel) and la_m - la_min in float32 (bcpd_la_apply_kernel; perm != null: alpha and
// sdiag are in the caller's order and are gathered into the internal one).  ssw: {scale, sigma2, w} in device memory.
int bcpd_weights(cpd_ctx* h, const double* alpha, const double* sdiag, const int* perm, const double* ssw) {
    const long long m = h->m;
    const unsigned nb = blocks_for(m);
    bcpd_la_kernel<<<nb, THREADS, 0, h->stream>>>(alpha, sdiag, m, ssw, h->dim, h->d_la64.p, h->d_la_part.p);
    bcpd_la_finish_kernel<<<1, 32, 0, h->stream>>>(h->d_la_part.p, (int)nb, ssw, h->dim, h->n_global, h->d_log2c.p);
    bcpd_la_apply_kernel<<<nb, THREADS, 0, h->stream>>>(h->d_la64.p, perm, m, h->d_log2c.p, h->d_la.p);
    KCHECK();
    h->launches += 3;
    return CPD_OK;
}
int ensure_weight_buffers(cpd_ctx* h) {
    const long long m = h->m;
    TRY(h->d_la.reserve((size_t)m));
    TRY(h->d_la64.reserve((size_t)m));
    TRY(h->d_la_part.reserve((size_t)blocks_for(m)));
    if (!h->d_log2c.p) TRY(h->d_log2c.alloc(3));
    if (!h->d_bc_es.p) TRY(h->d_bc_es.alloc(3));
    return CPD_OK;
}
}  // namespace

// BayesianCoherentPointDrift.expectation_step (probreg/bcpd.py:53-72): the CPD E-step with a weight per source,
//   pmat_nm = exp(-|x_n - t_m|^2 / 2 sigma2) (2 pi sigma2)^(-D/2) * exp(-scale^2 / (2 sigma2) * sigma_mm * D) * (1 - w) * alpha_m,
//   den_n = w / N + sum_m pmat_nm,  P = pmat / den,  nu_d = sum_m P (n),  nu = sum_n P (m),  px = P x (m x D),  n_p = sum nu.
// The weights enter the exponent as la_m = -log2(weight_m) (FP64, minus their minimum so that la >= 0 and FP32 keeps
// them to ~1e-7 absolute); the constant w / N moves to the same units.  x_hat = px / nu is left to the caller (bcpd.py:70-71).
// Dead columns (bcpd.py:64-65: den == 0 -> eps, so P = 0): a term of the reference's float64 sum is exactly 0 when
// exp(-d2 / 2 sigma2) underflows (log2 < -1075) or when its product with the factors does.  In kernel units
// (S' = sum_m 2^-(u + la')) the first is log2 S' < -1075 -- exact for equal weights, the dominant-term approximation
// otherwise -- and the second log2 S' - la_min - (D/2) log2(2 pi sigma2) < -1075: the smaller of the two shifts decides.
// The exponents and constants are formed on the device by bcpd_weights, the routine the device-resident loop (host_bcpd.inl) uses.
extern "C" int cpd_bcpd_estep(cpd_ctx* h, const double* t_source, double scale, const double* alpha, const double* sigma_diag,
                              double sigma2, double w, double* nu_d, double* nu, double* px, double* n_p) {
    if (!h || !t_source || !alpha || !sigma_diag) return fail(CPD_ERR_ARG, "null argument");
    if (!(sigma2 > 0.0)) return fail(CPD_ERR_ARG, "sigma2 must be positive, got %g", sigma2);
    if (!(w >= 0.0 && w < 1.0)) return fail(CPD_ERR_ARG, "w must be in [0, 1), got %g", w);
    TRY(require_clouds(h));
    CU(cudaSetDevice(h->device));
    const long long m = h->m;
    bool any_weight = false;
    for (long long i = 0; i < m; ++i) {
        if (!(alpha[i] >= 0.0) || !(sigma_diag[i] >= 0.0)) return fail(CPD_ERR_ARG, "alpha and diag(sigma_mat) must be non-negative");
        any_weight = any_weight || (alpha[i] > 0.0 && sigma_diag[i] < INFINITY);
    }
    if (!any_weight) return fail(CPD_ERR_ARG, "every source has zero weight");
    TRY(ensure_weight_buffers(h));
    // alpha and sigma_diag (caller's order) into d_outM [0, m) and [m, 2m), {scale, sigma2, w} into d_bc_es
    h->pin.p->bc_ssw[0] = scale;
    h->pin.p->bc_ssw[1] = sigma2;
    h->pin.p->bc_ssw[2] = w;
    CU(cudaMemcpyAsync(h->d_bc_es.p, h->pin.p->bc_ssw, 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_outM.p, alpha, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_outM.p + m, sigma_diag, (size_t)m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    TRY(bcpd_weights(h, h->d_outM.p, h->d_outM.p + m, h->d_perm_src.p, h->d_bc_es.p));
    TRY(run_estep(h, t_source, sigma2, w, true));
    return cpd_last_estep(h, nu_d, nu, px, n_p);
}

extern "C" int cpd_last_estep(cpd_ctx* h, double* pt1, double* p1, double* px, double* n_p) {
    if (!h) return fail(CPD_ERR_ARG, "null handle");
    if (!h->prepared) return fail(CPD_ERR_STATE, "no E-step has run on this handle");
    CU(cudaSetDevice(h->device));
    if (pt1) {
        scatter_kernel<<<blocks_for(h->n), THREADS, 0, h->stream>>>(h->d_pt1.p, h->d_perm_tgt.p, h->n, 1, h->d_outN.p);
        CU(cudaMemcpyAsync(pt1, h->d_outN.p, (size_t)h->n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
        h->launches += 1;
    }
    if (p1) TRY(download_src(h, h->d_p1.p, 1, p1));
    if (px) {
        uncentre_px_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_state.p, h->d_p1.p, h->d_pxc.p, (int)h->m, h->d_px.p);
        h->launches += 1;
        TRY(download_src(h, h->d_px.p, 3, px));
    }
    if (n_p) {
        // n_p = sum(p1) (cpd.py:88): block partials of the (possibly all-reduced) p1
        const unsigned nb = blocks_for(h->m);
        TRY(h->d_sums.reserve((size_t)nb * 4 + 4));
        src_moments_api_kernel<<<nb, THREADS, 0, h->stream>>>((int)h->m, h->d_yc.p, h->d_p1.p, h->d_pxc.p, h->d_mom_src.p);
        reduce_cols_kernel<<<1, MOM_SRC * 32, 0, h->stream>>>(h->d_mom_src.p, (int)nb, MOM_SRC, h->d_mom.p);
        KCHECK();
        h->launches += 2;
        CU(cudaMemcpyAsync(&h->pin.p->n_p, h->d_mom.p, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    }
    CU(cudaStreamSynchronize(h->stream));
    if (n_p) *n_p = h->pin.p->n_p;
    return CPD_OK;
}

namespace {
// a caller's E-step result (pt1, p1, px as cpd_estep returns them) into d_pt1, d_p1 and d_px, caller's order -> internal (Morton) order
int upload_estep(cpd_ctx* h, const double* pt1, const double* p1, const double* px) {
    CU(cudaMemcpyAsync(h->d_outN.p, pt1, (size_t)h->n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    gather1_kernel<<<blocks_for(h->n), THREADS, 0, h->stream>>>(h->d_outN.p, h->d_perm_tgt.p, h->n, h->d_pt1.p);
    CU(cudaMemcpyAsync(h->d_outM.p, p1, (size_t)h->m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    gather1_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_outM.p, h->d_perm_src.p, h->m, h->d_p1.p);
    TRY(h->d_raw.reserve((size_t)h->m * 3));
    TRY(upload_cloud(h, px, h->m, h->d_raw.p));
    gather3_kernel<<<blocks_for(h->m), THREADS, 0, h->stream>>>(h->d_raw.p, h->d_perm_src.p, h->m, 0.0, 0.0, 0.0, h->d_px.p);
    KCHECK();
    h->launches += 3;
    return CPD_OK;
}
}  // namespace

extern "C" int cpd_mstep(cpd_ctx* h, int tf_kind, int update_scale, const double* pt1, const double* p1, const double* px, double n_p,
                         cpd_params* out) {
    (void)n_p;   // recomputed as sum(p1), which is what the reference passes (cpd.py:88)
    if (!h || !pt1 || !p1 || !px || !out) return fail(CPD_ERR_ARG, "null argument");
    if (tf_kind != CPD_TF_RIGID && tf_kind != CPD_TF_AFFINE) return fail(CPD_ERR_ARG, "tf_kind %d not supported", tf_kind);
    TRY(require_clouds(h));
    CU(cudaSetDevice(h->device));
    TRY(prepare(h));
    h->nr.end("cpd_mstep ended the non-rigid loop of this handle: call cpd_nonrigid_*begin again");
    h->h_state.tf_kind = tf_kind;
    h->h_state.update_scale = update_scale ? 1 : 0;
    // only the two selectors: the rest of the device state may be ahead of the host mirror
    CU(cudaMemcpyAsync(&h->d_state.p->tf_kind, &h->h_state.tf_kind, 2 * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    TRY(upload_estep(h, pt1, p1, px));
    const int nbs = (int)blocks_for(h->m), nbt = (int)blocks_for(h->n);
    centre_px_kernel<<<nbs, THREADS, 0, h->stream>>>(h->d_state.p, h->d_p1.p, h->d_px.p, (int)h->m, h->d_pxc.p);
    src_moments_api_kernel<<<nbs, THREADS, 0, h->stream>>>((int)h->m, h->d_yc.p, h->d_p1.p, h->d_pxc.p, h->d_mom_src.p);
    tgt_moments_api_kernel<<<nbt, THREADS, 0, h->stream>>>(h->d_pt1.p, h->d_xc.p, (int)h->n, h->d_mom_tgt.p);
    moments_kernel<0><<<1, 256, 0, h->stream>>>(h->d_state.p, h->d_mom_src.p, nbs, MOM_SRC, h->d_mom_tgt.p, nbt, MOM_TGT, h->d_mom.p);
    KCHECK();
    if (h->comm) TRY(allreduce(h, h->d_mom.p + MOM_SRC, MOM_TGT));   // p1/px are already global; pt1 is per shard
    mstep_api_kernel<<<1, 32, 0, h->stream>>>(h->d_state.p, h->d_mom.p);
    KCHECK();
    h->launches += 5;
    return read_params(h, out);
}

// The remaining entry points live in the .inl files of this same translation unit:
#include "host_nonrigid.inl"     // cpd_nonrigid_* (dense G, low-rank factors, priors)
#include "host_bcpd.inl"         // cpd_bcpd_begin / step / get, cpd_bcpd_step_times (the BCPD loop on the device)
#include "host_gmmtree.inl"      // cpd_gmmtree_* (the GMMTree build and registration E-step)
#include "host_stateless.inl"    // cpd_rbf_kernel, cpd_imq_kernel, cpd_gauss_transform, cpd_squared_kernel_sum
#include "host_l2dist.inl"       // cpd_gmm_fit, cpd_l2_dist, cpd_tps_kernel (GMMReg)
#include "host_ocsvm.inl"        // cpd_ocsvm_fit (the one-class SVM of SVR)
#include "host_filterreg.inl"    // cpd_lattice_filter, cpd_filterreg_estep (the permutohedral lattice of FilterReg)
#include "host_multi.inl"        // cpd_comm_*, cpd_p2p_*
#include "host_measure.inl"      // cpd_timer_*, cpd_event_*, cpd_stage_times, cpd_flush_l2, cpd_microbench
#include "host_batch.inl"        // cpd_batch_register (many small rigid / affine registrations, one CTA per pair)
