// k10_frame_batch_encode.cuh -- K10: frame encode of a batch of units of any length (sb_frame_encode_batch_device_ws).
//
// Replaces, per unit, `FrameEncoder::new(vec![]).write_all(input); into_inner()` (reference src/write.rs:123-192 with
// src/frame.rs:62-104): the stream identifier, then one chunk per <= 65,536-byte slice, each compressed or stored by
// K4's chunk rule. Chunks are independent, so K10 has K9's shape: every chunk of every unit goes through ONE K1 launch,
// unchanged, in frame mode (each chunk's varint and its masked CRC-32C in the emitter warp):
//   k10_plan       thread per unit: the cap check and the unit's class in K9's classes (rejected, empty, one chunk,
//                  more than one chunk); Σ n over multi-chunk units -> ctl.
//   k9_scan_*      K9's scan of the slot counts (K9's kernels over the embedded RawCompressPlan).
//   k10_iscan_*    with an index: the same scan of every unit's chunk count; unit i's index starts at i + that prefix.
//   k10_fill       thread per K1 entry. Entry u < count is unit u's single chunk, compressed in place at out_u + 10 + 8
//                  (cap >= sb_frame_max_len(n) = 10 + 8 + 76,490 holds max_compress_len(65536) behind both headers);
//                  entry count + g is slot g. Every other entry is empty and writes its one-byte varint to `sink`.
//   K1             flags 1 (chunk varint), crcs of nk entries, slots of kSlotStride.
//   k10_bscan_local + k9_bscan_tiles: the scan over the slots' final chunk sizes 8 + (stored ? n_c : c).
//   k10_gather     warp per slot: the chunk's header and body to out_u + 10 + (its offset inside the unit), and its
//                  index entry.
//   k10_finish     warp per unit, always: the identifier, a single chunk's header (its body copied over K1's output
//                  when it is stored uncompressed), out_lens, the status, the first and last index entries.
// The scratch depends only on (count, in_bytes), as K9's does; K9's layout with the CRCs, the index scan and the sink
// appended.
#pragma once
#include "k9_raw_batch_compress.cuh"

namespace sbk {

static const uint32_t K10_IDENT = 10;                  // stream identifier (src/frame.rs:18)
static const uint32_t K10_CHUNK_HDR = 8;               // type, u24 length, masked CRC (src/frame.rs:26)
static const uint32_t K10_MAX_CBLOCK = 76490;          // src/frame.rs:12

struct FrameBatchPlan {
    RawCompressPlan r;                 // K9's plan: units, classes (K9_*), slot scan, K1 entries, body scan, slots
    uint64_t* idx;                     // d_chunk_offs (may be null)
    uint32_t* crcs;                    // nk: K1's masked CRC per entry
    uint64_t *ix_offs, *ix_tiles;      // scan over units (count + 1 entries) of their chunk counts
    uint8_t* sink;                     // where K1's empty entries write their varint
};

inline uint64_t k10_carve(void* scratch, uint32_t count, uint64_t in_bytes, FrameBatchPlan* q) {
    const uint64_t k9 = k9_carve(scratch, count, in_bytes, q ? &q->r : nullptr);
    if (k9 == ~0ull) return k9;
    const uint64_t nk = (uint64_t)count + k9_slot_bound(count, in_bytes);
    const uintptr_t base = ((uintptr_t)scratch + k9 + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    uint32_t* crcs = (uint32_t*)take(nk * 4);
    uint64_t* ix_offs = (uint64_t*)take(((uint64_t)count + 2) * 8);
    uint64_t* ix_tiles = (uint64_t*)take(((uint64_t)count + 1) / K4_TILE * 8 + 24);
    uint8_t* sink = (uint8_t*)take(256);
    if (q) { q->crcs = crcs; q->ix_offs = ix_offs; q->ix_tiles = ix_tiles; q->sink = sink; }
    return k9 + at + 256;
}

// sb_frame_max_len(n)
SB_DEVICE uint64_t k10_need(uint64_t n) { return K10_IDENT + (n + kMaxBlock - 1) / kMaxBlock * (K10_CHUNK_HDR + K10_MAX_CBLOCK); }
SB_DEVICE uint32_t k10_chunks(uint64_t n) { return (uint32_t)((n + kMaxBlock - 1) / kMaxBlock); }
// first index entry of unit u
SB_DEVICE uint64_t k10_index_base(const FrameBatchPlan& q, uint32_t u) { return u + k8b_at(q.ix_offs, q.ix_tiles, u); }

SB_DEVICE void k10_plan_body(const FrameBatchPlan& q) {
    const RawCompressPlan& r = q.r;
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    uint64_t multi = 0;
    if (i < r.b.count) {
        const uint64_t n = unit_in_len(r.b, (uint32_t)i), cap = unit_out_cap(r.b, (uint32_t)i);
        uint32_t c;
        if (n == 0) c = K9_EMPTY;                                      // nothing is written (src/write.rs:155-157)
        else if (cap < k10_need(n)) c = K9_TOO_SMALL;
        else if (n <= kMaxBlock) c = K9_SINGLE;
        else { c = K9_MULTI; multi = n; }
        r.cls[i] = c;
    }
#pragma unroll
    for (unsigned m = 16; m; m >>= 1) multi += shfl(multi, lane_id() ^ m);
    if (lane_id() == 0 && multi) atomic_add(&r.ctl->in_total, (unsigned long long)multi);
}

SB_DEVICE void k10_iscan_local_body(const FrameBatchPlan& q) {
    const uint32_t count = q.r.b.count;
    scan_local_body(count + 1, [&](uint32_t u) { return u < count ? k10_chunks(unit_in_len(q.r.b, u)) : 0u; }, q.ix_offs,
                    q.ix_tiles);
}
SB_DEVICE void k10_iscan_tiles_body(const FrameBatchPlan& q) { scan_tiles_body(q.r.b.count + 1, 0, q.ix_tiles); }

SB_DEVICE void k10_fill_body(const FrameBatchPlan& q) {
    const RawCompressPlan& r = q.r;
    const uint64_t e = (uint64_t)block_idx() * block_dim() + thread_idx();
    if (e >= r.nk) return;
    const uint32_t count = r.b.count;
    const uint8_t* in = nullptr;
    uint8_t* out = q.sink;
    uint32_t len = 0;
    if (e < count) {
        const uint32_t u = (uint32_t)e;
        if (r.cls[u] == K9_SINGLE) {
            len = unit_in_len(r.b, u);
            in = unit_in(r.b, u);
            out = unit_out(r.b, u) + K10_IDENT + K10_CHUNK_HDR;
        }
    } else {
        const uint64_t g = e - count;
        if (g < k8b_at(r.sl_offs, r.sl_tiles, count)) {
            const uint32_t u = k8b_unit_of(r.sl_offs, r.sl_tiles, count, g);
            const uint64_t j = g - k8b_at(r.sl_offs, r.sl_tiles, u), n = unit_in_len(r.b, u);
            const uint64_t left = n - j * kMaxBlock;
            len = left > kMaxBlock ? kMaxBlock : (uint32_t)left;
            in = unit_in(r.b, u) + j * kMaxBlock;
            out = r.slots + g * kSlotStride;
        }
    }
    r.k1_in[e] = in; r.k1_out[e] = out; r.k1_lens[e] = len;
}

// bytes slot g occupies in its unit's stream
SB_DEVICE uint32_t k10_slot_size(const RawCompressPlan& r, uint32_t g) {
    const uint32_t n = r.k1_lens[r.b.count + g], c = r.k1_clens[r.b.count + g];
    return K10_CHUNK_HDR + (K4_CHUNK_RAW(c, n) ? n : c);
}
SB_DEVICE void k10_bscan_local_body(const FrameBatchPlan& q) {
    const uint32_t nslot = q.r.nslot;
    scan_local_body(nslot + 1, [&](uint32_t g) { return g < nslot ? k10_slot_size(q.r, g) : 0u; }, q.r.bo_offs, q.r.bo_tiles);
}

// the 8-byte chunk header of a chunk of n input bytes, c compressed: lane k < 8 writes byte k (src/frame.rs:91-93)
SB_DEVICE void k10_put_header(uint8_t* dst, uint32_t c, uint32_t n, uint32_t crc) {
    const bool raw = K4_CHUNK_RAW(c, n);
    const uint64_t hdr = (uint64_t)(raw ? 1u : 0u) | ((uint64_t)(4 + (raw ? n : c)) << 8) | ((uint64_t)crc << 32);
    if (lane_id() < 8) dst[lane_id()] = (uint8_t)(hdr >> (8 * lane_id()));
}

SB_DEVICE void k10_gather_body(const FrameBatchPlan& q) {
    const RawCompressPlan& r = q.r;
    const uint32_t count = r.b.count;
    const uint64_t total = k8b_at(r.sl_offs, r.sl_tiles, count);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < total; g += nwarps) {
        const uint32_t u = k8b_unit_of(r.sl_offs, r.sl_tiles, count, g);
        const uint64_t first = k8b_at(r.sl_offs, r.sl_tiles, u);
        const uint64_t at = K10_IDENT + k8b_at(r.bo_offs, r.bo_tiles, g) - k8b_at(r.bo_offs, r.bo_tiles, first);
        const uint32_t n = r.k1_lens[count + g], c = r.k1_clens[count + g];
        uint8_t* dst = unit_out(r.b, u) + at;
        k10_put_header(dst, c, n, q.crcs[count + g]);
        const bool raw = K4_CHUNK_RAW(c, n);
        warp_copy_t<true>(dst + K10_CHUNK_HDR, raw ? unit_in(r.b, u) + (g - first) * kMaxBlock : r.slots + g * kSlotStride,
                          raw ? n : c);
        if (q.idx && lane_id() == 0) q.idx[k10_index_base(q, u) + (g - first)] = at;
    }
}

SB_DEVICE void k10_finish_body(const FrameBatchPlan& q) {
    const RawCompressPlan& r = q.r;
    const BatchDesc& b = r.b;
    const unsigned wpb = block_dim() >> 5, lane = lane_id();
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t i = (uint64_t)block_idx() * wpb + warp_id(); i < b.count; i += nwarps) {
        const uint32_t u = (uint32_t)i, c = r.cls[u];
        const uint64_t n = unit_in_len(b, u);
        sb_error* st = b.statuses ? &b.statuses[u] : nullptr;
        syncwarp();
        if (c == K9_TOO_SMALL) {
            if (lane == 0) { b.out_lens[u] = 0; set_status(st, SB_BUFFER_TOO_SMALL, unit_out_cap(b, u), k10_need(n), 0); }
            continue;
        }
        if (c == K9_MULTI && k9_over(r)) {
            if (lane == 0) { b.out_lens[u] = 0; set_status(st, SB_E_INVALID, r.ctl->in_total, r.in_bytes, 0); }
            continue;
        }
        uint8_t* out = unit_out(b, u);
        uint64_t len = 0;
        if (c == K9_SINGLE) {
            const uint32_t cl = r.k1_clens[u];
            const bool raw = K4_CHUNK_RAW(cl, (uint32_t)n);
            k10_put_header(out + K10_IDENT, cl, (uint32_t)n, q.crcs[u]);
            if (raw) warp_copy_t<true>(out + K10_IDENT + K10_CHUNK_HDR, unit_in(b, u), (uint32_t)n);
            len = K10_IDENT + K10_CHUNK_HDR + (raw ? n : cl);
        } else if (c == K9_MULTI) {
            const uint64_t s0 = k8b_at(r.sl_offs, r.sl_tiles, u), s1 = k8b_at(r.sl_offs, r.sl_tiles, u + 1);
            len = K10_IDENT + k8b_at(r.bo_offs, r.bo_tiles, s1) - k8b_at(r.bo_offs, r.bo_tiles, s0);
        }
        if (len && lane < K10_IDENT) out[lane] = (uint8_t)("\xff\x06\x00\x00sNaPpY"[lane]);
        if (lane == 0) {
            b.out_lens[u] = (uint32_t)len;
            set_status(st, SB_OK, 0, 0, 0);
            if (q.idx) {
                const uint64_t x = k10_index_base(q, u);
                if (c == K9_SINGLE) q.idx[x] = K10_IDENT;
                q.idx[x + k10_chunks(n)] = len;
            }
        }
    }
}

}  // namespace sbk
