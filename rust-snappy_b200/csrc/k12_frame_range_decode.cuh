// k12_frame_range_decode.cuh -- K12: decode byte ranges of one frame stream (sb_frame_decode_ranges_device_ws).
//
// Range r asks for decoded bytes [lo_r, lo_r + len_r). K12 runs K5's index phase unchanged (K7 or the caller's index,
// parse, walk when needed, scan of decoded lengths), so every chunk k of the table has its output offset off_k and
// decoded length dlen_k before anything is decoded. Then only the (range, chunk) pairs the ranges cover are decoded:
//   k12_plan        thread per range: the range's first and last verified chunk by binary search over the scanned
//                   offsets (k8b_at), its pair count; K4's generic scan of the counts (k12_plan_tiles finishes it).
//   k12_decode      warp per pair, grid-striding over the pair total that only the device knows: the pair's range by
//                   k8b_unit_of, then K5's decode + CRC (k5_decode_chunk). An interior chunk (inside [lo, end) in full)
//                   decodes straight into the range's buffer; a head or tail chunk (straddling lo or end) decodes into
//                   one of the range's two 64 KiB staging slots in scratch and a warp copy writes only its slice: the
//                   whole chunk must be decoded to check its CRC, and in place it would overrun the range's buffer. The
//                   first failing chunk per range by atomic_min.
//   k12_finish      thread per range: status and out_len in the order below; the stream's result.
//
// Which chunks a range verifies. With end = min(lo + len, total), range r verifies chunk k iff
// off_k < end && off_k + max(dlen_k, 1) > lo: every chunk that produces a byte of [lo, end), and every empty chunk at an
// offset inside it. Both tests are monotone in k (off_k + max(dlen_k, 1) never decreases), so the verified chunks are one
// run [first, last]. Only the first can straddle lo and only the last can straddle end, so two slots per range suffice.
//
// Why the per-range result is exact. `FrameDecoder::new(stream).read_to_end()` yields the chunks in stream order and
// stops at the first one that fails. If every chunk the range does not verify is valid, the reader reaches lo, and the
// first failing chunk it meets while producing [lo, end) is the first failing verified chunk k*: it has produced
// max(off_k*, lo) - lo bytes of the range by then, with k*'s own status (K5's, byte for byte). When none fails and the
// range ends inside the stream, what follows end does not change those bytes; when the range reaches past total, the
// reader goes on to the end of the header chain and returns the walk's stopping error (Ok at a clean end: a short read).
// A table that is too small leaves total a lower bound, so every range reports it first, as k5_finish does.
//
// Costs. A chunk shared by several ranges is decoded once per range, and each range takes 128 KiB of staging whatever
// its length; callers with very many small ranges over tabled streams use the gathers (k17_table_gather.cuh).
#pragma once
#include "k5_frame_decode.cuh"
#include "k8_raw_split.cuh"
#include "k18_host_gather.cuh"

namespace sbk {

// max_chunks limit: a range verifies at most max_chunks chunks, and 1,024 pair counts (one scan tile) stay below 2^32
static const uint32_t K12_MAX_CHUNKS = (1u << 22) - 2;
static const uint32_t K12_MAX_RANGES = 1u << 31;
static const uint64_t K12_SLOT = kMaxBlock;            // staging bytes per slot: the largest decoded chunk
static const uint32_t K12_NONE = 0xFFFFFFFFu;

struct RangeRec { uint32_t first; uint32_t pairs; uint32_t first_bad; uint32_t _pad; };

struct RangePlan {
    DecodePlan d;                      // K5's index phase: cap UINT64_MAX, out null; d.result receives the stream's result
    const uint64_t *lo, *len;          // nranges each
    uint8_t* const* outs;              // range r's buffer holds len[r] bytes
    uint64_t* out_lens;
    sb_error* statuses;
    uint32_t nranges;
    RangeRec* rec;                     // nranges
    uint64_t *pr_offs, *pr_tiles;      // scan over ranges of their pair counts (nranges + 1 entries)
    uint8_t* staging;                  // 2 slots of K12_SLOT bytes per range
};

// Scratch layout of the range part (host side), behind K5's decode scratch: every array 256-byte aligned from
// `scratch` (null: just the size). Returns the bytes used.
inline uint64_t k12_carve(void* scratch, uint32_t nranges, RangePlan* q) {
    const uint64_t units = (uint64_t)nranges + 1;
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    RangeRec* rec = (RangeRec*)take(nranges * sizeof(RangeRec));
    uint64_t* offs = (uint64_t*)take((units + 1) * 8);
    uint64_t* tiles = (uint64_t*)take((units / K4_TILE + 3) * 8);
    uint8_t* staging = (uint8_t*)take(2 * nranges * K12_SLOT);
    if (q) { q->nranges = nranges; q->rec = rec; q->pr_offs = offs; q->pr_tiles = tiles; q->staging = staging; }
    return at + 256;
}

// The gather calls (k17_table_gather.cuh) replace the two staging slots per range by a pool of k17_pool_slots(nranges)
// slots of K12_SLOT bytes, one per warp that decodes into staging: the gather decode and K13's finish body run only the
// first k12_pool_warps warps of their grid, warp w on slot w. The one definition of the pool's size, for the carve, the
// launch grids and the bodies.
static const uint32_t K17_SLOTS = 4096;
#if defined(SB_EMU)
static inline uint64_t k17_pool_slots(uint32_t nranges)
#else
__host__ __device__ __forceinline__ uint64_t k17_pool_slots(uint32_t nranges)
#endif
{
    return 2ull * nranges < K17_SLOTS ? 2ull * nranges : K17_SLOTS;
}
SB_DEVICE uint64_t k12_pool_warps(uint64_t nwarps, uint32_t nranges) {
    const uint64_t slots = k17_pool_slots(nranges);
    return nwarps < slots ? nwarps : slots;
}
// Emulator builds count the chunk and block decodes of the gather calls, so the tests can check their cost contract
#if defined(SB_EMU)
inline uint64_t g_emu_decodes = 0;
#define K17_COUNT_DECODE() do { if (lane_id() == 0) sbk::g_emu_decodes++; } while (0)
#else
#define K17_COUNT_DECODE() do {} while (0)
#endif

SB_DEVICE bool k12_table_full(const DecodeCtl* c) { return c->walk_err.code == SB_E_INVALID && c->walk_err.b == 1; }
// min(lo + len, total) without overflow
SB_DEVICE uint64_t k12_end(uint64_t lo, uint64_t len, uint64_t total) { return lo > total || len > total - lo ? total : lo + len; }
SB_DEVICE uint64_t k12_off(const RangePlan& q, uint32_t k) { return k8b_at(q.d.ooff, q.d.tiles, k); }

SB_DEVICE void k12_plan_body(const RangePlan& q) {
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    const DecodeCtl* ctl = q.d.ctl;
    uint32_t v = 0;
    if (i < q.nranges) {
        const uint32_t n = k12_table_full(ctl) ? 0 : ctl->nchunks;
        const uint64_t lo = q.lo[i], end = k12_end(lo, q.len[i], ctl->produced);
        const FChunk* ch = q.d.chunks;
        uint32_t a = 0, b = n;                                           // first k with off_k + max(dlen_k, 1) > lo
        while (a < b) {
            const uint32_t m = a + (b - a) / 2;
            const uint32_t dl = ch[m].dlen;
            if (k12_off(q, m) + (dl ? dl : 1) > lo) b = m; else a = m + 1;
        }
        const uint32_t first = a;
        b = n;                                                           // first k >= first with off_k >= end
        while (a < b) {
            const uint32_t m = a + (b - a) / 2;
            if (k12_off(q, m) >= end) b = m; else a = m + 1;
        }
        v = a - first;
        RangeRec r;
        r.first = first; r.pairs = v; r.first_bad = K12_NONE; r._pad = 0;
        q.rec[i] = r;
    }
    scan_local_body(q.nranges + 1, [&](uint32_t) { return v; }, q.pr_offs, q.pr_tiles);
}
SB_DEVICE void k12_plan_tiles_body(const RangePlan& q) { scan_tiles_body(q.nranges + 1, 0, q.pr_tiles); }

SB_DEVICE void k12_decode_body(const RangePlan& q) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const uint64_t pairs = k8b_at(q.pr_offs, q.pr_tiles, q.nranges), total = q.d.ctl->produced;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < pairs; g += nwarps) {
        const uint32_t r = k8b_unit_of(q.pr_offs, q.pr_tiles, q.nranges, g);
        const uint32_t first = q.rec[r].first, k = first + (uint32_t)(g - k8b_at(q.pr_offs, q.pr_tiles, r));
        const FChunk c = q.d.chunks[k];
        const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], total), off = k12_off(q, k);
        const bool inside = off >= lo && off + c.dlen <= end;
        uint8_t* dst = inside ? q.outs[r] + (off - lo) : q.staging + ((uint64_t)r * 2 + (k == first ? 0 : 1)) * K12_SLOT;
        // a chunk verified by several ranges gets the same status from each: its header and body decide it
        const uint32_t code = k5_decode_chunk(tab, elems, c, q.d.in, dst, &q.d.statuses[k]);
        if (code != SB_OK) { if (lane_id() == 0) atomic_min(&q.rec[r].first_bad, k); }
        else if (!inside) {                                              // the slice of [lo, end) a head or tail chunk holds
            const uint64_t a = off > lo ? off : lo, e = off + c.dlen < end ? off + c.dlen : end;
            warp_copy(q.outs[r] + (a - lo), dst + (a - off), (uint32_t)(e - a));
        }
        syncwarp();
    }
}

// per range, in priority order: chunk table too small, the first failing verified chunk, past the end: the walk's
// stopping error (Ok at a clean end), else Ok
SB_DEVICE void k12_finish_body(const RangePlan& q) {
    const DecodeCtl* ctl = q.d.ctl;
    const bool full = k12_table_full(ctl);
    const uint64_t total = ctl->produced;
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx(); i < q.nranges; i += nthreads) {
        const uint64_t lo = q.lo[i], len = q.len[i], end = k12_end(lo, len, total);
        const uint32_t bad = q.rec[i].first_bad;
        sb_error* st = &q.statuses[i];
        uint64_t got = end > lo ? end - lo : 0;
        if (full) { set_status(st, SB_E_INVALID, q.d.cap_chunks, 1, 0); got = 0; }
        else if (bad != K12_NONE) { const uint64_t off = k12_off(q, bad); *st = q.d.statuses[bad]; got = off > lo ? off - lo : 0; }
        else if (lo > total || len > total - lo) *st = ctl->walk_err;
        else set_status(st, SB_OK, 0, 0, 0);
        q.out_lens[i] = got;
    }
    if (block_idx() == 0 && thread_idx() == 0) {
        sb_frame_result r;
        r.status = ctl->walk_err; r.bytes = total; r.nchunks = ctl->nchunks; r._pad = 0;
        *q.d.result = r;
    }
}

}  // namespace sbk
