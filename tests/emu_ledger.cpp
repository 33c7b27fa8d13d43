// tests/emu_ledger.cpp -- TEST INFRASTRUCTURE: a ledger in front of the CPU emulation's allocation and event stand-ins.
//
// tests/test_emulated_ownership.py links this file into its own copy of the emulated library, with tests/emu/emu_runtime.cpp
// compiled under -DcudaMalloc=emu_base_cudaMalloc (and the same for cudaFree, cudaMallocHost, cudaFreeHost, cudaEventCreate
// and cudaEventDestroy): the library's calls land here, are recorded, and are passed on.  Nothing is injected: every call
// does what the emulation does, and a free of a pointer the ledger never handed out is refused and counted.
#include "cuda_runtime.h"

#include <mutex>
#include <unordered_map>
#include <utility>

cudaError_t emu_base_cudaMalloc(void** p, size_t bytes);
cudaError_t emu_base_cudaFree(void* p);
cudaError_t emu_base_cudaMallocHost(void** p, size_t bytes);
cudaError_t emu_base_cudaFreeHost(void* p);
cudaError_t emu_base_cudaEventCreate(cudaEvent_t* e);
cudaError_t emu_base_cudaEventDestroy(cudaEvent_t e);

namespace {
struct Ledger {
    std::mutex mu;
    std::unordered_map<void*, std::pair<size_t, bool>> live;      // block -> (bytes, pinned)
    long long blocks[2] = {0, 0}, bytes[2] = {0, 0}, allocs[2] = {0, 0}, unknown_frees = 0, ev_created = 0, ev_destroyed = 0;
};
Ledger& ledger() {
    static Ledger l;
    return l;
}
cudaError_t record_alloc(cudaError_t e, void* p, size_t bytes, bool pinned) {
    if (e != cudaSuccess) return e;
    Ledger& l = ledger();
    std::lock_guard<std::mutex> lk(l.mu);
    l.live[p] = {bytes, pinned};
    l.blocks[pinned] += 1;
    l.bytes[pinned] += (long long)bytes;
    l.allocs[pinned] += 1;
    return e;
}
// true: p is a live block of this kind, now forgotten; false: counted as an unknown free
bool record_free(void* p, bool pinned) {
    Ledger& l = ledger();
    std::lock_guard<std::mutex> lk(l.mu);
    auto it = l.live.find(p);
    if (it == l.live.end() || it->second.second != pinned) {
        l.unknown_frees += 1;
        return false;
    }
    l.blocks[pinned] -= 1;
    l.bytes[pinned] -= (long long)it->second.first;
    l.live.erase(it);
    return true;
}
}  // namespace

cudaError_t cudaMalloc(void** p, size_t bytes) {
    const cudaError_t e = emu_base_cudaMalloc(p, bytes);
    return record_alloc(e, *p, bytes, false);
}
cudaError_t cudaMallocHost(void** p, size_t bytes) {
    const cudaError_t e = emu_base_cudaMallocHost(p, bytes);
    return record_alloc(e, *p, bytes, true);
}
cudaError_t cudaFree(void* p) {
    if (!p) return cudaSuccess;
    return record_free(p, false) ? emu_base_cudaFree(p) : cudaErrorInvalidValue;
}
cudaError_t cudaFreeHost(void* p) {
    if (!p) return cudaSuccess;
    return record_free(p, true) ? emu_base_cudaFreeHost(p) : cudaErrorInvalidValue;
}
cudaError_t cudaEventCreate(cudaEvent_t* e) {
    const cudaError_t r = emu_base_cudaEventCreate(e);
    std::lock_guard<std::mutex> lk(ledger().mu);
    if (r == cudaSuccess) ledger().ev_created += 1;
    return r;
}
cudaError_t cudaEventDestroy(cudaEvent_t e) {
    {
        std::lock_guard<std::mutex> lk(ledger().mu);
        ledger().ev_destroyed += 1;
    }
    return emu_base_cudaEventDestroy(e);
}

// out: live device blocks, device bytes, device allocation calls, live pinned blocks, pinned bytes, pinned allocation calls,
// unknown frees, events created, events destroyed
extern "C" void cpd_emu_alloc_stats(long long out[9]) {
    Ledger& l = ledger();
    std::lock_guard<std::mutex> lk(l.mu);
    const long long v[9] = {l.blocks[0], l.bytes[0], l.allocs[0], l.blocks[1], l.bytes[1], l.allocs[1], l.unknown_frees, l.ev_created,
                            l.ev_destroyed};
    for (int k = 0; k < 9; ++k) out[k] = v[k];
}
