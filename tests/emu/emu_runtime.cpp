// tests/emu/emu_runtime.cpp -- TEST INFRASTRUCTURE: the fiber scheduler and the host stand-ins behind
// tests/emu/cuda_runtime.h.  See that header for the execution model.
#include "cuda_runtime.h"

#include <stdio.h>
#include <stdlib.h>
#include <sys/mman.h>
#include <ucontext.h>

#include <algorithm>
#include <chrono>
#include <mutex>
#include <vector>

#undef threadIdx
#undef blockIdx
#undef blockDim
#undef gridDim

namespace emu {
uint3 g_threadIdx, g_blockIdx;
dim3 g_blockDim, g_gridDim;
unsigned char* g_dyn_smem = nullptr;

namespace {
constexpr size_t STACK = 512 << 10;
// Context switch between the scheduler and a fiber.  On x86-64 a hand-written switch of the callee-saved registers and the stack
// pointer (no system call; glibc's swapcontext saves the signal mask on every switch, which is most of the cost of a warp
// shuffle here); elsewhere, or with -DEMU_UCONTEXT (AddressSanitizer understands that one better), plain ucontext.
#if defined(__x86_64__) && !defined(EMU_UCONTEXT)
#define EMU_FAST_SWITCH 1
struct Ctx { void* sp; };
extern "C" void emu_switch(Ctx* from, Ctx* to);
asm(".text\n"
    ".globl emu_switch\n"
    ".type emu_switch,@function\n"
    "emu_switch:\n"
    "    pushq %rbp\n    pushq %rbx\n    pushq %r12\n    pushq %r13\n    pushq %r14\n    pushq %r15\n"
    "    movq %rsp, (%rdi)\n"
    "    movq (%rsi), %rsp\n"
    "    popq %r15\n    popq %r14\n    popq %r13\n    popq %r12\n    popq %rbx\n    popq %rbp\n"
    "    ret\n"
    ".size emu_switch, .-emu_switch\n");
#else
struct Ctx { ucontext_t uc; };
static void emu_switch(Ctx* from, Ctx* to) { swapcontext(&from->uc, &to->uc); }
#endif
struct Fiber {
    Ctx ctx;
    bool done = false;
};
struct Warp {
    int alive = 0, count = 0;
    unsigned gen = 0;
    unsigned char slot[32][16];
    bool pred[32];
    bool present[32];
};
Ctx g_sched;
std::vector<Fiber> g_fibers;
std::vector<Warp> g_warps;
char* g_stacks = nullptr;
size_t g_stack_count = 0;
int g_cur = -1, g_nthreads = 0, g_alive = 0, g_bar_count = 0;
unsigned g_bar_gen = 0;
const std::function<void()>* g_body = nullptr;
long long g_launches = 0;
std::vector<unsigned char> g_smem_store;

void release_block_barrier_if_complete() {
    if (g_alive > 0 && g_bar_count == g_alive) { g_bar_count = 0; ++g_bar_gen; }
}
void release_warp_barrier_if_complete(Warp& w) {
    if (w.alive > 0 && w.count == w.alive) { w.count = 0; ++w.gen; }
}
void trampoline() {
    (*g_body)();
    Fiber& f = g_fibers[g_cur];
    f.done = true;
    --g_alive;
    Warp& w = g_warps[g_cur >> 5];
    --w.alive;
    w.present[g_cur & 31] = false;
    release_block_barrier_if_complete();     // exited threads count as arrived (CUDA semantics)
    release_warp_barrier_if_complete(w);
    emu_switch(&f.ctx, &g_sched);
    abort();                                  // a finished fiber is never resumed
}
void warp_barrier() {
    Warp& w = g_warps[g_cur >> 5];
    const unsigned gen = w.gen;
    ++w.count;
    release_warp_barrier_if_complete(w);
    while (w.gen == gen) yield();
}
}  // namespace

void yield() {
    Fiber& f = g_fibers[g_cur];
    emu_switch(&f.ctx, &g_sched);
}
void syncthreads() {
    const unsigned gen = g_bar_gen;
    ++g_bar_count;
    release_block_barrier_if_complete();
    while (g_bar_gen == gen) yield();
}
void syncwarp() { warp_barrier(); }
void exchange(const void* mine, size_t bytes, int src_lane, void* out) {
    if (bytes > 16) { fprintf(stderr, "emu: shuffle of %zu bytes\n", bytes); abort(); }
    Warp& w = g_warps[g_cur >> 5];
    memcpy(w.slot[g_cur & 31], mine, bytes);
    warp_barrier();
    // a shuffle from an exited / out-of-range lane returns the caller's own value on hardware (undefined in
    // general); the library never relies on that, so flag it
    if (!w.present[src_lane]) { fprintf(stderr, "emu: shuffle from an inactive lane\n"); abort(); }
    memcpy(out, w.slot[src_lane], bytes);
    warp_barrier();
}
unsigned vote_any(bool pred) {
    Warp& w = g_warps[g_cur >> 5];
    w.pred[g_cur & 31] = pred;
    warp_barrier();
    unsigned m = 0;
    for (int l = 0; l < 32; ++l) if (w.present[l] && w.pred[l]) m |= 1u << l;
    warp_barrier();
    return m;
}
long long launches() { return g_launches; }

// Order in which the runnable fibers of a block get the CPU in each scheduling round.  CPD_EMU_SCHED = "rr" (default:
// thread 0, 1, 2, ...), "reverse", or "random[:seed]" (a fresh permutation every round).  A kernel whose result depends on
// the order is missing a barrier; the test-suite runs under all three.
static void next_order(std::vector<size_t>& order, size_t n) {
    static int mode = -1;
    static unsigned long long rng = 0x9e3779b97f4a7c15ull;
    if (mode < 0) {
        const char* e = getenv("CPD_EMU_SCHED");
        mode = (!e || !strncmp(e, "rr", 2)) ? 0 : (!strncmp(e, "reverse", 7) ? 1 : 2);
        if (mode == 2 && e[6] == ':') rng ^= strtoull(e + 7, nullptr, 10) * 0xbf58476d1ce4e5b9ull;
    }
    if (order.size() != n) {
        order.resize(n);
        for (size_t i = 0; i < n; ++i) order[i] = mode == 1 ? n - 1 - i : i;
    }
    if (mode == 2)
        for (size_t i = n - 1; i > 0; --i) {
            rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
            std::swap(order[i], order[rng % (i + 1)]);
        }
}

void launch(const char* name, dim3 grid, dim3 block, size_t smem, cudaStream_t, const std::function<void()>& body) {
    // one kernel at a time in the whole process: ranks of a multi-rank test are OS threads, and the scheduler state, the
    // `static` stand-ins for __shared__ and the mbarrier table are process-wide
    static std::mutex kernel_lock;
    std::lock_guard<std::mutex> lk(kernel_lock);
    const size_t nthreads = (size_t)block.x * block.y * block.z;
    static std::vector<size_t> order;
    // the hardware limits a blind launch would trip over
    if (nthreads == 0 || nthreads > 1024 || grid.x == 0 || grid.y == 0 || grid.z == 0 || grid.x > 2147483647u || grid.y > 65535u ||
        grid.z > 65535u || smem > 227u * 1024u) {
        fprintf(stderr, "emu: invalid launch configuration for %s: grid (%u,%u,%u) block (%u,%u,%u) smem %zu\n", name, grid.x, grid.y,
                grid.z, block.x, block.y, block.z, smem);
        abort();
    }
    ++g_launches;
    if (g_stack_count < nthreads) {
        if (g_stacks) munmap(g_stacks, g_stack_count * STACK);
        g_stacks = (char*)mmap(nullptr, nthreads * STACK, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (g_stacks == MAP_FAILED) { perror("emu: mmap"); abort(); }
        g_stack_count = nthreads;
    }
    g_smem_store.assign(smem + 256, 0xcd);
    g_dyn_smem = g_smem_store.data() + (128 - ((uintptr_t)g_smem_store.data() % 128)) % 128;
    g_blockDim = block;
    g_gridDim = grid;
    g_body = &body;
    g_nthreads = (int)nthreads;
    g_fibers.resize(nthreads);
    g_warps.resize((nthreads + 31) / 32);
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                g_blockIdx = uint3{bx, by, bz};
                g_alive = (int)nthreads;
                g_bar_count = 0;
                for (Warp& w : g_warps) { w.alive = 0; w.count = 0; for (int l = 0; l < 32; ++l) w.present[l] = false; }
                for (size_t t = 0; t < nthreads; ++t) {
                    Fiber& f = g_fibers[t];
                    f.done = false;
#ifdef EMU_FAST_SWITCH
                    {   // first switch "returns" into trampoline with the stack aligned as after a call
                        void** top = reinterpret_cast<void**>(g_stacks + (t + 1) * STACK);
                        top[-2] = reinterpret_cast<void*>(&trampoline);
                        for (int r = 3; r <= 8; ++r) top[-r] = nullptr;      // rbp, rbx, r12..r15
                        f.ctx.sp = &top[-8];
                    }
#else
                    getcontext(&f.ctx.uc);
                    f.ctx.uc.uc_stack.ss_sp = g_stacks + t * STACK;
                    f.ctx.uc.uc_stack.ss_size = STACK;
                    f.ctx.uc.uc_link = &g_sched.uc;
                    makecontext(&f.ctx.uc, trampoline, 0);
#endif
                    g_warps[t >> 5].alive++;
                    g_warps[t >> 5].present[t & 31] = true;
                }
                int remaining = (int)nthreads;
                long long idle_rounds = 0;
                while (remaining > 0) {
                    int progressed = 0;
                    next_order(order, nthreads);
                    for (size_t oi = 0; oi < nthreads; ++oi) {
                        const size_t t = order[oi];
                        Fiber& f = g_fibers[t];
                        if (f.done) continue;
                        g_cur = (int)t;
                        g_threadIdx = uint3{(unsigned)(t % block.x), (unsigned)((t / block.x) % block.y), (unsigned)(t / ((size_t)block.x * block.y))};
                        emu_switch(&g_sched, &f.ctx);
                        if (f.done) { --remaining; ++progressed; }
                    }
                    // a round in which nobody finished is normal (barriers); a very long run of them is a deadlock
                    idle_rounds = progressed ? 0 : idle_rounds + 1;
                    if (idle_rounds > 2000000ll) { fprintf(stderr, "emu: %s appears deadlocked\n", name); abort(); }
                }
            }
    g_cur = -1;
}
}  // namespace emu

long long clock64() {
    return (long long)std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
namespace cpd {
unsigned long long globaltimer_ns() { return (unsigned long long)clock64(); }
}

// ---- runtime API ---------------------------------------------------------------------------
struct emu_stream { int unused; };
struct emu_event { double t_ms; bool recorded; };
static int emu_sms() {
    const char* e = getenv("CPD_EMU_SMS");
    const int v = e ? atoi(e) : 0;
    return v > 0 ? v : 132;
}
static int emu_devices() {
    const char* e = getenv("CPD_EMU_DEVICES");
    const int v = e ? atoi(e) : 0;
    return v > 0 ? v : 1;
}
cudaError_t cudaGetDeviceCount(int* n) { *n = emu_devices(); return cudaSuccess; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated CUDA error"; }
cudaError_t cudaSetDevice(int d) { return (d >= 0 && d < emu_devices()) ? cudaSuccess : cudaErrorInvalidValue; }
cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    memset(p, 0, sizeof(*p));
    p->major = 9; p->minor = 0; p->multiProcessorCount = emu_sms();
    snprintf(p->name, sizeof(p->name), "CPU emulation (tests/emu)");
    return cudaSuccess;
}
cudaError_t cudaMalloc(void** p, size_t bytes) {
    void* q = nullptr;
    if (posix_memalign(&q, 256, bytes ? bytes : 1) != 0) return cudaErrorMemoryAllocation;
    memset(q, 0xa5, bytes);                 // device memory is not zero-initialised: make reliance on that visible
    *p = q;
    return cudaSuccess;
}
cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaMallocHost(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void* dst, const void* src, size_t bytes, cudaMemcpyKind) { memmove(dst, src, bytes); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind, cudaStream_t) { memmove(dst, src, bytes); return cudaSuccess; }
cudaError_t cudaMemcpy2DAsync(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width, size_t height, cudaMemcpyKind, cudaStream_t) {
    for (size_t r = 0; r < height; ++r) memmove((char*)dst + r * dpitch, (const char*)src + r * spitch, width);
    return cudaSuccess;
}
cudaError_t cudaMemset(void* p, int v, size_t bytes) { memset(p, v, bytes); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void* p, int v, size_t bytes, cudaStream_t) { memset(p, v, bytes); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = new emu_stream(); return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { delete s; return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emu_event(); (*e)->t_ms = 0.0; (*e)->recorded = false; return cudaSuccess; }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t_ms = (double)clock64() * 1e-6; e->recorded = true; return cudaSuccess; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
    if (!a->recorded || !b->recorded) return cudaErrorInvalidValue;      // the real runtime refuses events that were never recorded
    *ms = (float)(b->t_ms - a->t_ms);
    return cudaSuccess;
}
cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return cudaErrorNotSupported; }
cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) { return cudaErrorNotSupported; }
cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
cudaError_t emu_func_set_attribute(const void*, int, int value) { return value <= 227 * 1024 ? cudaSuccess : cudaErrorInvalidValue; }
cudaError_t emu_occupancy(int* out, const void*, int, size_t smem) {
    *out = smem > 0 ? (int)((227u * 1024u) / (smem + 1024)) : 8;
    if (*out > 2) *out = 2;                 // the E-step kernels are register-limited to 2 CTAs/SM on the real part
    return cudaSuccess;
}

extern "C" long long cpd_emu_launches(void) { return emu::launches(); }
extern "C" int cpd_is_emulation(void) { return 1; }
