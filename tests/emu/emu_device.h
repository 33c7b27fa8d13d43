// tests/emu/emu_device.h -- TEST INFRASTRUCTURE: host stand-ins for the inline-PTX helpers of
// probreg_b200/csrc/kernels.cuh (included from there only when CPD_HOST_EMU is defined).
//   ex2.approx.ftz      -> exp2f with results below FLT_MIN flushed to 0 (the property exact culling relies on)
//   FP32 pair helpers   -> two scalar IEEE operations per call (compile with -ffp-contract=off)
//   mbarrier + TMA bulk -> the copy is performed when the barrier is waited on; until then the destination
//                          holds a NaN pattern, so reading a stage before its wait, or re-arming a stage that
//                          a slower thread still reads, corrupts the results visibly
#pragma once
#include <float.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

namespace cpd {
typedef unsigned long long u64;

// CPD_EMU_EX2=mufu: perturb the result by a smooth function of the argument's fractional part, up to 2^-22 relative -- the
// size and kind of error MUFU.EX2 has.  The library's parity must not depend on ex2 being exact (it relies on both passes
// seeing the SAME argument so that the error cancels in K / sum K); the test-suite also runs in this mode.
static inline float ex2(float x) {
    static const int mode = [] { const char* e = getenv("CPD_EMU_EX2"); return (e && !strcmp(e, "mufu")) ? 1 : 0; }();
    float r = exp2f(x);
    if (mode == 1 && x > -1000.0f && x < 1000.0f) {
        const float fr = x - floorf(x);
        r *= 1.0f + 2.3841858e-07f * sinf(6.2831853f * (3.0f * fr + 0.17f));
    }
    return (r < FLT_MIN) ? 0.0f : r;
}
static inline u64 pack2(float lo, float hi) {
    uint32_t a, b;
    memcpy(&a, &lo, 4); memcpy(&b, &hi, 4);
    return (u64)a | ((u64)b << 32);
}
static inline float2 unpack2(u64 v) {
    const uint32_t a = (uint32_t)v, b = (uint32_t)(v >> 32);
    float2 r;
    memcpy(&r.x, &a, 4); memcpy(&r.y, &b, 4);
    return r;
}
static inline u64 fsub2(u64 a, u64 b) { const float2 x = unpack2(a), y = unpack2(b); return pack2(x.x - y.x, x.y - y.y); }
static inline u64 fadd2(u64 a, u64 b) { const float2 x = unpack2(a), y = unpack2(b); return pack2(x.x + y.x, x.y + y.y); }
static inline u64 fmul2(u64 a, u64 b) { const float2 x = unpack2(a), y = unpack2(b); return pack2(x.x * y.x, x.y * y.y); }
static inline u64 ffma2(u64 a, u64 b, u64 c) {
    const float2 x = unpack2(a), y = unpack2(b), z = unpack2(c);
    return pack2(fmaf(x.x, y.x, z.x), fmaf(x.y, y.y, z.y));
}

// one mbarrier = 8 bytes of shared memory: {completed phases (u32), index+1 into the pending-copy table (u32)}
struct EmuPending { void* dst; const void* src; uint32_t bytes; };
struct EmuBarrier { uint32_t phases; uint32_t armed; };
inline std::vector<std::vector<EmuPending>>& emu_pending() { static std::vector<std::vector<EmuPending>> t; return t; }
static inline void mbar_init(uint64_t* bar, uint32_t) {
    EmuBarrier* b = reinterpret_cast<EmuBarrier*>(bar);
    b->phases = 0; b->armed = 0;
}
static inline void mbar_fence_init() {}
static inline void mbar_expect_tx(uint64_t* bar, uint32_t) {
    EmuBarrier* b = reinterpret_cast<EmuBarrier*>(bar);
    auto& tab = emu_pending();
    tab.emplace_back();
    b->armed = (uint32_t)tab.size();
}
static inline void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    EmuBarrier* b = reinterpret_cast<EmuBarrier*>(bar);
    if (!b->armed) { fprintf(stderr, "emu: TMA copy on an mbarrier without expect_tx\n"); abort(); }
    if (bytes % 16 || ((uintptr_t)dst % 16) || ((uintptr_t)src % 16)) { fprintf(stderr, "emu: misaligned bulk copy\n"); abort(); }
    memset(dst, 0xff, bytes);                                  // poison until the barrier completes
    emu_pending()[b->armed - 1].push_back({dst, src, bytes});
}
static inline void mbar_wait(uint64_t* bar, uint32_t parity) {
    EmuBarrier* b = reinterpret_cast<EmuBarrier*>(bar);
    while ((b->phases & 1u) == parity) {                       // the phase with this parity has not completed yet
        if (!b->armed) { emu::yield(); continue; }             // nobody armed it yet: spin like the hardware would
        for (const EmuPending& p : emu_pending()[b->armed - 1]) memcpy(p.dst, p.src, p.bytes);
        emu_pending()[b->armed - 1].clear();
        b->armed = 0;
        b->phases += 1;
    }
}
static inline uint32_t smem_u32(const void*) { return 0; }
static inline void st_release_sys(unsigned long long* p, unsigned long long v) { *(volatile unsigned long long*)p = v; }
static inline unsigned long long ld_acquire_sys(const unsigned long long* p) { return *(const volatile unsigned long long*)p; }
static inline double ld_relaxed_sys(const double* p) { return *(const volatile double*)p; }
unsigned long long globaltimer_ns();
}  // namespace cpd
