// simt.h -- thin portability layer for the kernel bodies.
//
// Under nvcc the wrappers are the sm_90a intrinsics, nothing more. Under
// -DSB_EMU (tests/emu only) the same kernel bodies are compiled by g++ against a
// fiber-based warp emulator so their LOGIC can be checked on a machine without a
// GPU. The emulator is test tooling: the product library is only ever built
// from the __CUDACC__ branch and has no CPU execution path.
#pragma once
#include <stdint.h>
#include <stddef.h>

#if defined(SB_EMU)
// the emulator build (tests/emu/emu_kernels.cpp) includes its own simt_emu.h BEFORE any kernel header
#ifndef SB_EMU_PRIMITIVES
#error "SB_EMU builds must include tests/emu/simt_emu.h first (it defines the warp primitives)"
#endif
namespace sbk {
// the emulator has no caches: a prefetch is a hint with nothing to do
SB_DEVICE void prefetch_l2(const void*) {}
// fibers switch only at warp collectives, so a plain compare-and-swap is atomic
SB_DEVICE unsigned long long atomic_cas(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
    const unsigned long long o = *p;
    if (o == cmp) *p = v;
    return o;
}
}
#else

#include <cuda_runtime.h>

#define SB_DEVICE __device__ __forceinline__
#define SB_DEVICE_NOINLINE __device__ __noinline__
#define SB_FULL 0xFFFFFFFFu

namespace sbk {

SB_DEVICE unsigned lane_id() { return threadIdx.x & 31u; }
SB_DEVICE unsigned warp_id() { return threadIdx.x >> 5; }
SB_DEVICE unsigned thread_idx() { return threadIdx.x; }
SB_DEVICE unsigned block_dim() { return blockDim.x; }
SB_DEVICE unsigned block_idx() { return blockIdx.x; }
SB_DEVICE unsigned grid_dim() { return gridDim.x; }

SB_DEVICE uint32_t shfl(uint32_t v, unsigned src) { return __shfl_sync(SB_FULL, v, src); }
SB_DEVICE int shfl(int v, unsigned src) { return __shfl_sync(SB_FULL, v, src); }
SB_DEVICE uint64_t shfl(uint64_t v, unsigned src) { return __shfl_sync(SB_FULL, v, src); }
SB_DEVICE uint32_t shfl_up(uint32_t v, unsigned d) { return __shfl_up_sync(SB_FULL, v, d); }
SB_DEVICE uint32_t shfl_down(uint32_t v, unsigned d) { return __shfl_down_sync(SB_FULL, v, d); }
SB_DEVICE uint32_t shfl_xor(uint32_t v, unsigned m) { return __shfl_xor_sync(SB_FULL, v, m); }
SB_DEVICE uint32_t ballot(bool p) { return __ballot_sync(SB_FULL, p); }
SB_DEVICE bool any(bool p) { return __any_sync(SB_FULL, p); }
SB_DEVICE bool all(bool p) { return __all_sync(SB_FULL, p); }
SB_DEVICE uint32_t match_any(uint32_t v) { return __match_any_sync(SB_FULL, v); }
SB_DEVICE void syncwarp() { __syncwarp(); }
SB_DEVICE void syncthreads() { __syncthreads(); }
// named barrier over `nthreads` threads (multiple of 32), id in [1,15]
SB_DEVICE void bar_sync(unsigned id, unsigned nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// non-blocking arrival on a named barrier (producer side of a bar.sync/bar.arrive pair)
SB_DEVICE void bar_arrive(unsigned id, unsigned nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

SB_DEVICE int popc(uint32_t v) { return __popc(v); }
SB_DEVICE int ffs(uint32_t v) { return __ffs(v); }          // 1-based, 0 if none
SB_DEVICE int clz(uint32_t v) { return __clz(v); }
SB_DEVICE int ffsll(uint64_t v) { return __ffsll((long long)v); }
SB_DEVICE uint32_t funnel_r(uint32_t lo, uint32_t hi, unsigned sh) { return __funnelshift_r(lo, hi, sh); }
SB_DEVICE uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t s) { return __byte_perm(a, b, s); }

SB_DEVICE uint32_t atomic_add(uint32_t* p, uint32_t v) { return atomicAdd(p, v); }
SB_DEVICE unsigned long long atomic_add(unsigned long long* p, unsigned long long v) { return atomicAdd(p, v); }
SB_DEVICE uint32_t atomic_min(uint32_t* p, uint32_t v) { return atomicMin(p, v); }
SB_DEVICE unsigned long long atomic_cas(unsigned long long* p, unsigned long long cmp, unsigned long long v) {
    return atomicCAS(p, cmp, v);
}
SB_DEVICE void threadfence() { __threadfence(); }
SB_DEVICE void threadfence_block() { __threadfence_block(); }
SB_DEVICE uint32_t reduce_or(uint32_t v) { return __reduce_or_sync(SB_FULL, v); }
SB_DEVICE uint32_t reduce_add(uint32_t v) { return __reduce_add_sync(SB_FULL, v); }
SB_DEVICE uint32_t reduce_max(uint32_t v) { return __reduce_max_sync(SB_FULL, v); }
// polite spin-wait hint inside producer/consumer polling loops
SB_DEVICE void spin() { __nanosleep(32); }
// consumer side: latency matters little, issue slots do. (The per-instruction counts of an ncu --set full capture
// overstate this poll loop: they come from the instrumented replay, which runs many times longer than the kernel, and
// polls scale with time; the hardware counter of the same capture puts polling at ~2-3% of issued instructions.)
SB_DEVICE void spin_long() { __nanosleep(1500); }
SB_DEVICE uint32_t ld_volatile(const uint32_t* p) { return *(const volatile uint32_t*)p; }
SB_DEVICE void st_volatile(uint32_t* p, uint32_t v) { *(volatile uint32_t*)p = v; }
SB_DEVICE uint64_t ld_volatile64(const uint64_t* p) { return *(const volatile uint64_t*)p; }
// L2 prefetch: no destination register, so nothing waits for it
SB_DEVICE void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// read-only / streaming global accessors
SB_DEVICE uint32_t ldg32(const void* p) { return __ldg((const uint32_t*)p); }
SB_DEVICE uint4 ldg128(const void* p) { return __ldg((const uint4*)p); }
SB_DEVICE uint8_t ldg8(const void* p) { return __ldg((const uint8_t*)p); }
// streaming (evict-first) 16-byte store for write-once output
SB_DEVICE void stcs128(void* p, uint4 v) { __stcs((uint4*)p, v); }

// mbarrier in shared memory (8 bytes, 8-aligned): producer arrives, consumer blocks in hardware instead of polling
SB_DEVICE void mbar_init(uint64_t* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
SB_DEVICE void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
}
// true once the phase of the given parity has completed; otherwise returns false after a hardware-bounded suspend
SB_DEVICE bool mbar_try_wait(uint64_t* bar, unsigned parity, unsigned hint_ns) {
    uint32_t done;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(parity), "r"(hint_ns) : "memory");
    return done != 0;
}
// write-once output bytes: evict-first in L2 so they do not displace data that is re-read
SB_DEVICE void st8_stream(uint8_t* p, uint8_t v) { __stcs(p, v); }
extern __shared__ __align__(128) unsigned char sb_dyn_smem[];
SB_DEVICE unsigned char* smem() { return sb_dyn_smem; }

}  // namespace sbk
#endif
