// k18_host_gather.cuh -- K18: the gathers of K17 over streams that stay in page-locked host memory
// (sb_frame_table_gather_host_streams_ws, sb_raw_table_gather_host_streams_ws).
//
// A stream in page-locked host memory mapped into the device's address space is readable by the kernels at its host
// address, but every load crosses PCIe: a decode that reads its body element by element waits one dependent round trip
// (~1-2 us) per cache line. K18 gives the gathers a source policy instead. The warp that decodes a chunk or block first
// copies its compressed body [src, src + len) from stream memory into a compressed slot of its own, in wide
// independent loads, then decodes from the slot. Only bodies the call decodes cross the bus, once per decode.
//   fetch   k18_fetch: the slot copy sits at src's offset within 16 bytes (src & 15), so the aligned middle moves in
//           16-byte loads and stores, K18_UNROLL of them in flight per lane; the unaligned head and tail move byte by
//           byte. No byte outside the body is read.
//   slots   K18_CSLOT bytes each: K5_MAX_CBLOCK (76,490, the largest body k13_rec_ok lets a frame record have) rounded up
//           to 256, so every frame body fits at any alignment. A raw block's body is bounded only by its stream (a legal
//           block may spend up to 5 compressed bytes per output byte); one that does not fit is decoded in place from
//           stream memory: correct, and slow.
//   where   the edge decodes (k17_*_gather_body<true>) and the interior decodes (k13_decode_body<true, true>,
//           k15_decode_body<true, true>), which in host mode run on the pool's warps (k12_pool_warps), so that every
//           decoding warp owns one compressed slot beside its 64 KiB decode slot. The error-only re-decodes of the
//           finish bodies read in place.
// The device gathers instantiate the same bodies with HOST = false, where the policy is the stream pointer itself.
#pragma once
#include "common.cuh"

namespace sbk {

static const uint64_t K18_CSLOT = (76490 + 255) / 256 * 256;   // K5_MAX_CBLOCK rounded up to 256: 76,544 bytes
static const uint32_t K18_UNROLL = 4;                         // 16-byte loads in flight per lane

// Emulator builds count the compressed bytes the host gathers copy into their slots, so the tests can check the cost
// contract: every decoded body once per decode, and nothing else
#if defined(SB_EMU)
inline uint64_t g_emu_fetched = 0;
#define K18_COUNT_FETCH(n) do { if (lane_id() == 0) sbk::g_emu_fetched += (n); } while (0)
SB_DEVICE uint4 k18_ld16(const uint8_t* p) { return ldg128(p); }
SB_DEVICE void k18_st16(uint8_t* p, uint4 v) { memcpy(p, &v, 16); }
#else
#define K18_COUNT_FETCH(n) do {} while (0)
// plain loads and stores: stream memory may be host memory, and the slot is read back by the same warp
SB_DEVICE uint4 k18_ld16(const uint8_t* p) { return *(const uint4*)p; }
SB_DEVICE void k18_st16(uint8_t* p, uint4 v) { *(uint4*)p = v; }
#endif

// The calling warp copies [src, src + len) to cslot + (src & 15) and returns the copy's address. cslot is 16-byte
// aligned and holds (src & 15) + len bytes.
SB_DEVICE const uint8_t* k18_fetch(const uint8_t* src, uint32_t len, uint8_t* cslot) {
    const uint32_t mis = (uint32_t)((uintptr_t)src & 15u), lane = lane_id();
    uint8_t* dst = cslot + mis;
    const uint32_t lead = (16u - mis) & 15u, head = lead < len ? lead : len;     // bytes before src's next 16-byte line
    const uint32_t nv = (len - head) >> 4, at = head + (nv << 4), tail = len - at;
    if (lane < head) dst[lane] = src[lane];
    if (lane < tail) dst[at + lane] = src[at + lane];
    const uint8_t* vs = src + head + ((uint64_t)lane << 4);             // 16-byte aligned, lane's first line
    uint8_t* vd = dst + head + ((uint64_t)lane << 4);
    uint32_t i = lane;
    for (; i + 32 * (K18_UNROLL - 1) < nv; i += 32 * K18_UNROLL, vs += 512 * K18_UNROLL, vd += 512 * K18_UNROLL) {
        uint4 v[K18_UNROLL];
#pragma unroll
        for (uint32_t k = 0; k < K18_UNROLL; k++) v[k] = k18_ld16(vs + 512 * k);
#pragma unroll
        for (uint32_t k = 0; k < K18_UNROLL; k++) k18_st16(vd + 512 * k, v[k]);
    }
    for (; i < nv; i += 32, vs += 512, vd += 512) k18_st16(vd, k18_ld16(vs));
    K18_COUNT_FETCH(len);
    syncwarp();
    return dst;
}

// the body a decode reads: the stream bytes themselves (HOST false, or a body the slot cannot hold), else their copy
template <bool HOST>
SB_DEVICE const uint8_t* k18_body(const uint8_t* src, uint32_t len, uint8_t* cslot) {
    if (!HOST || ((uintptr_t)src & 15u) + (uint64_t)len > K18_CSLOT) return src;
    return k18_fetch(src, len, cslot);
}

// Scratch of a host gather: the device gather's (k17_carve, `gather_bytes` of it from `scratch`), then `slots`
// compressed slots, 256-byte aligned. Returns the bytes used; *cpool (when not null) receives the first slot.
inline uint64_t k18_carve(void* scratch, uint64_t gather_bytes, uint64_t slots, uint8_t** cpool) {
    if (cpool) *cpool = (uint8_t*)(((uintptr_t)scratch + 255) / 256 * 256 + gather_bytes - 256);
    return gather_bytes + slots * K18_CSLOT;
}

}  // namespace sbk
