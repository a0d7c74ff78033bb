// common.cuh -- shared definitions for the sm_90a Snappy kernels.
#pragma once
#include "simt.h"
#include "../../include/snapb200.h"

namespace sbk {

static const uint32_t kMaxBlock = 65536;       // reference src/lib.rs:97
static const uint64_t kMaxInput = 0xFFFFFFFFull;  // reference src/lib.rs:93
static const uint32_t kSlotStride = 76544;     // >= max_compress_len(65536)=76490, multiple of 128

// One independent unit of work = one raw stream in, one buffer out (sb_batch,
// include/snapb200.h): pointer arrays, or base + i*stride when they are null.
typedef sb_batch BatchDesc;

SB_DEVICE const uint8_t* unit_in(const BatchDesc& b, uint32_t i) {
    return b.in_ptrs ? b.in_ptrs[i] : b.in_base + (uint64_t)i * b.in_stride;
}
SB_DEVICE uint8_t* unit_out(const BatchDesc& b, uint32_t i) {
    return b.out_ptrs ? b.out_ptrs[i] : b.out_base + (uint64_t)i * b.out_stride;
}
SB_DEVICE uint32_t unit_in_len(const BatchDesc& b, uint32_t i) {
    return b.in_lens ? b.in_lens[i] : b.in_len_uniform;
}
SB_DEVICE uint32_t unit_out_cap(const BatchDesc& b, uint32_t i) {
    return b.out_caps ? b.out_caps[i] : b.out_cap_uniform;
}

SB_DEVICE void set_status(sb_error* st, uint32_t code, uint64_t a, uint64_t b, uint64_t c) {
    if (st) { st->code = code; st->_pad = 0; st->a = a; st->b = b; st->c = c; }
}

// ---------------------------------------------------------------------------
// Warp-cooperative byte copy, global/shared -> global/shared, non-overlapping.
// All 32 lanes call it with identical arguments. 4-byte-aligned stores with
// funnel-shifted aligned loads; every load stays inside [src, src+n).
// EF: the destination is write-once output -> evict-first stores (kept out of the L2 working set).
template <bool EF>
SB_DEVICE void warp_copy_t(uint8_t* dst, const uint8_t* src, uint32_t n) {
    auto put8 = [](uint8_t* p, uint8_t v) { if (EF) st8_stream(p, v); else *p = v; };
    auto put128 = [](uint8_t* p, uint4 v) { if (EF) stcs128(p, v); else *(uint4*)p = v; };
    const unsigned lane = lane_id();
    if (n < 64) {
        for (uint32_t k = lane; k < n; k += 32) put8(dst + k, src[k]);
        return;
    }
    // head: bring dst to 16-byte alignment
    uint32_t head = (uint32_t)((0 - (uintptr_t)dst) & 15u);
    if (lane < head) put8(dst + lane, src[lane]);
    dst += head; src += head; n -= head;
    const uint32_t m = (uint32_t)((uintptr_t)src & 3u);
    uint32_t nvec = n >> 4;
    if (m == 0) {
        if ((((uintptr_t)src) & 15u) == 0) {
            for (uint32_t v = lane; v < nvec; v += 32)
                put128(dst + 16 * v, *(const uint4*)(src + 16 * v));
        } else {
            for (uint32_t v = lane; v < nvec; v += 32) {
                const uint32_t* s = (const uint32_t*)(src + 16 * v);
                put128(dst + 16 * v, make_uint4(s[0], s[1], s[2], s[3]));
            }
        }
    } else {
        // aligned words w[j] at (src - m) + 4j; output word j = funnel(w[j], w[j+1], 8m).
        // The first word starts m bytes before src and the word after the last
        // vector may end past src+n: keep one vector on each side for the byte path.
        const uint32_t* w = (const uint32_t*)(src - m);
        const unsigned sh = 8 * m;
        uint32_t v0 = 1, v1 = nvec > 0 ? nvec - 1 : 0;   // vectors [v0, v1) use word loads
        if (v1 < v0) v1 = v0;
        for (uint32_t v = v0 + lane; v < v1; v += 32) {
            const uint32_t* p = w + 4 * v;
            uint32_t a = p[0], b = p[1], c = p[2], d = p[3], e = p[4];
            put128(dst + 16 * v, make_uint4(funnel_r(a, b, sh), funnel_r(b, c, sh), funnel_r(c, d, sh), funnel_r(d, e, sh)));
        }
        if (nvec > 0) {
            if (lane < 16) put8(dst + lane, src[lane]);
            if (nvec > 1 && lane >= 16) put8(dst + 16 * (nvec - 1) + (lane - 16), src[16 * (nvec - 1) + (lane - 16)]);
        }
    }
    uint32_t done = nvec << 4;
    if (done + lane < n) put8(dst + done + lane, src[done + lane]);   // tail < 16 bytes
}
SB_DEVICE void warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n) { warp_copy_t<false>(dst, src, n); }

}  // namespace sbk
