// k11_frame_batch_decode.cuh -- K11: frame decode of a batch of streams (sb_frame_decode_batch_device_ws).
//
// Replaces, per unit, `FrameDecoder::new(unit).read_to_end()` (reference src/read.rs:104-239) with exactly the result
// sb_frame_decode_device_ws gives that unit. The per-stream pieces are K5's and K7's own device functions; K11 adds the
// unit dimension, the way K8b adds it to K8: per-unit scans (K4's generic scan, k8b_at / k8b_unit_of for lookups) turn
// per-unit counts into slices of shared arrays, and every pass is one grid over a global item list.
//   k11_plan        thread per unit: without a caller index, the unit's K7 segment count (Σ in_lens -> ctl); with one,
//                   the unit's index entries from d_index_at. Scanned over units (k11_plan_tiles finishes it).
//   k11_survivors   (no caller index) warp per global segment: K7's survivor search on the unit's IndexPlan view.
//   k11_stitch      (no caller index) CTAs grid-striding over units: K7's stitch -> chunk count or NOT_INDEXABLE.
//   k11_link        (caller index) thread per index entry: the linkage check (below). A unit that fails is walked.
//   k11_count       thread per unit: the unit's table range -- K7's count, the caller's count, or the count of the
//                   reader's walk (k5_walk without a sink) -- capped at max_chunks + 1, and the scan of the ranges.
//                   Units take ranges in batch order; a unit fits when its range ends at or below max_chunks.
//   k11_emit        (no caller index) thread per global segment: K7's emit into the unit's slice of the index table.
//   k11_parse       thread per table slot: K5's per-chunk check (k5_check_chunk) against the unit's index.
//   k11_fill        thread per unit that is walked (never indexed, or a chunk the parse rejected): the reader's walk
//                   (k5_walk) writes its chunk records into the unit's range. Every unit: live chunks, walk error.
//   k11_oscan_*     scan of the decoded lengths of every live slot; a unit needs prefix(end) - prefix(start) bytes.
//   k11_decode      warp per live slot of a unit that fits its cap: K5's decode + CRC (k5_decode_chunk); the first
//                   failing chunk per unit by atomic_min.
//   k11_finish      thread per unit: status and out_lens in k5_finish's priority order, d_unit_chunks.
//
// Why fixed ranges are safe. A unit's range is sized before the parse or the walk fill runs. The reader's walk follows
// header linkage (pos += 4 + len for every chunk type) from offset 0 and stops no later than the end of that chain,
// recording only data chunks. When a chain's linkage has been verified -- by K7's hops (type, length and bounds of every
// chunk, the identifier, the chain ending at n) or by k11_link (the first entry is 10 and the identifier bytes are
// right, or 0 for a fragment; every entry has 4 <= len and at + 4 + len == next inside the stream; the last entry is n)
// -- any walk of that unit visits a prefix of the same chain and so records at most its entries. K7's count, or the
// caller's count once linked, therefore bounds the walk fill; a unit whose linkage was not verified gets its range from
// its own walk count. Where the parse and the walk disagree -- a short-body varint the parse rejects and the walk accepts
// through the reader's persistent buffer (src/read.rs:216), a padding or skippable chunk inside a caller-indexed chain
// -- only the live count changes, never the range. Every data chunk occupies at least 8 bytes, so a range never exceeds
// n / 8.
//
// Why the results are the single call's. A unit whose parse accepts every chunk of a verified chain is exactly what the
// reader's walk would record (the argument of k7_frame_index.cuh), so both paths give the reader's chunk list and
// stopping error; decode, CRC and the choice of the reported error are K5's, per unit.
#pragma once
#include "k5_frame_decode.cuh"
#include "k7_frame_index.cuh"
#include "k8_raw_split.cuh"

namespace sbk {

// max_chunks limit: a unit's range is capped at max_chunks + 1, and 1,024 of them (one scan tile) stay below 2^32
static const uint32_t K11_MAX_CHUNKS = (1u << 22) - 2;
static const uint32_t K11_MAX_COUNT = 1u << 31;
static const uint64_t K11_MAX_IN_BYTES = 1ull << 36;   // larger bounds are clamped, as in K8b
static const uint32_t K11_NONE = 0xFFFFFFFFu;

enum { K11_WALK = 0, K11_K7 = 1, K11_CALLER = 2 };       // how a unit's range was sized

struct FrameUnitCtl {
    uint32_t mode;        // K11_*: K7's or the caller's verified chain, or the walk count
    uint32_t k7_count;    // K7's chunk count, or SB_FRAME_NOT_INDEXABLE
    uint32_t range;       // slots in the chunk table (<= max_chunks + 1)
    uint32_t reparse;     // the parse rejected a chunk: the walk fills the range
    uint32_t nchunks;     // live chunks in the range
    uint32_t first_bad;   // first failing chunk (unit-local), K11_NONE
    sb_error walk_err;    // the reader's stopping error (Ok for a parsed unit)
};

struct FrameDecodeBatchPlan {
    sb_batch b;
    uint32_t fragment;                 // flags bit0: no stream identifier expected
    uint32_t max_chunks;               // chunk table slots
    uint64_t in_bytes;                 // the caller's bound on Σ in_lens (clamped)
    uint64_t seg;                      // K7 segment length
    const uint64_t *cidx, *cidx_at;    // optional caller index: unit i's is cidx[cidx_at[i] .. cidx_at[i+1])
    uint32_t* unit_chunks;             // optional: chunks the parallel parse placed per unit, 0 when walked
    unsigned long long* in_total;      // Σ in_lens (zeroed before k11_plan)
    FrameUnitCtl* uctl;                // count
    uint64_t *sg_offs, *sg_tiles;      // scan over units of their K7 segments (caller index: their index entries)
    uint64_t *rg_offs, *rg_tiles;      // scan over units of their table ranges
    K7Seg* segs;                       // global segment list
    uint32_t *nsurv, *ent, *base;
    uint32_t nseg_cap;
    uint64_t* idx;                     // K7's index: unit u's at range start + u (max_chunks + count + 1 entries)
    FChunk* chunks;                    // max_chunks
    sb_error* cst;                     // max_chunks: each chunk's status
    uint64_t *o_offs, *o_tiles;        // scan of the slots' decoded lengths
};

// Scratch layout (host side): every array 256-byte aligned from `scratch` (null: just the size). Returns the bytes used.
inline uint64_t k11_carve(void* scratch, uint32_t count, uint64_t in_bytes, uint32_t max_chunks, FrameDecodeBatchPlan* q) {
    const uint64_t in = in_bytes < K11_MAX_IN_BYTES ? in_bytes : K11_MAX_IN_BYTES;
    const uint64_t units = (uint64_t)count + 1, slots = (uint64_t)max_chunks + 1;
    const uint64_t segs = in / K7_SEG_MIN + count;                      // Σ ceil((n_i - s0) / seg)
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    FrameDecodeBatchPlan p;
    p.in_bytes = in;
    p.nseg_cap = (uint32_t)segs;
    p.in_total = (unsigned long long*)take(8);
    p.uctl = (FrameUnitCtl*)take(count * sizeof(FrameUnitCtl));
    p.sg_offs = (uint64_t*)take((units + 1) * 8); p.sg_tiles = (uint64_t*)take((units / K4_TILE + 3) * 8);
    p.rg_offs = (uint64_t*)take((units + 1) * 8); p.rg_tiles = (uint64_t*)take((units / K4_TILE + 3) * 8);
    p.segs = (K7Seg*)take(segs * sizeof(K7Seg));
    p.nsurv = (uint32_t*)take(segs * 4);
    p.ent = (uint32_t*)take(segs * 4);
    p.base = (uint32_t*)take(segs * 4);
    p.idx = (uint64_t*)take((slots + count) * 8);
    p.chunks = (FChunk*)take(max_chunks * sizeof(FChunk));
    p.cst = (sb_error*)take(max_chunks * sizeof(sb_error));
    p.o_offs = (uint64_t*)take((slots + 1) * 8); p.o_tiles = (uint64_t*)take((slots / K4_TILE + 3) * 8);
    if (q) {
        p.b = q->b; p.fragment = q->fragment; p.max_chunks = max_chunks; p.seg = q->seg;
        p.cidx = q->cidx; p.cidx_at = q->cidx_at; p.unit_chunks = q->unit_chunks;
        *q = p;
    }
    return at + 256;
}

SB_DEVICE bool k11_over(const FrameDecodeBatchPlan& q) { return *q.in_total > q.in_bytes; }
// start of unit u's table range; the unit fits when its range ends at or below max_chunks (ranges in batch order)
SB_DEVICE uint64_t k11_range(const FrameDecodeBatchPlan& q, uint32_t u) { return k8b_at(q.rg_offs, q.rg_tiles, u); }
SB_DEVICE bool k11_fits(const FrameDecodeBatchPlan& q, uint32_t u) { return k11_range(q, u + 1) <= q.max_chunks; }
SB_DEVICE uint64_t k11_out_at(const FrameDecodeBatchPlan& q, uint64_t j) { return k8b_at(q.o_offs, q.o_tiles, j); }
// slots of the table that belong to some unit (they may reach past max_chunks: those units do not fit)
SB_DEVICE uint64_t k11_slots(const FrameDecodeBatchPlan& q) {
    const uint64_t t = k11_range(q, q.b.count);
    return t < q.max_chunks ? t : q.max_chunks;
}

// K7 segments of a unit of n bytes (k7_make_plan's decisions with the batch's segment length); 0 and *decline = 1
// when K7 does not index it (no room for the identifier, more chunks than the table holds)
SB_DEVICE uint32_t k11_k7_nseg(const FrameDecodeBatchPlan& q, uint64_t n, uint32_t* decline) {
    const uint64_t s0 = q.fragment ? 0 : 10, body = n > s0 ? n - s0 : 0;
    *decline = (n < s0 || (body + K7_SPAN - 1) / K7_SPAN > q.max_chunks) ? 1u : 0u;
    return *decline ? 0 : (uint32_t)((body + q.seg - 1) / q.seg);
}
// unit u as one K7 stream: its bytes and its slices of the batch's arrays
SB_DEVICE IndexPlan k11_index_view(const FrameDecodeBatchPlan& q, uint32_t u) {
    IndexPlan p;
    p.in = unit_in(q.b, u); p.n = unit_in_len(q.b, u);
    p.s0 = q.fragment ? 0 : 10; p.seg = q.seg; p.fragment = q.fragment; p.max_chunks = q.max_chunks;
    p.nseg = k11_k7_nseg(q, p.n, &p.decline);
    const uint64_t s = k8b_at(q.sg_offs, q.sg_tiles, u);
    p.segs = q.segs + s; p.nsurv = q.nsurv + s; p.ent = q.ent + s; p.base = q.base + s;
    p.index = q.idx + k11_range(q, u) + u;                          // meaningful once the ranges are scanned
    p.count = &q.uctl[u].k7_count;
    return p;
}
// unit u's index: the caller's, or K7's slice
SB_DEVICE const uint64_t* k11_index(const FrameDecodeBatchPlan& q, uint32_t u) {
    return q.cidx ? q.cidx + q.cidx_at[u] : q.idx + k11_range(q, u) + u;
}

SB_DEVICE void k11_plan_body(const FrameDecodeBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    uint64_t n = 0;
    if (i < count) {
        const uint32_t u = (uint32_t)i;
        n = unit_in_len(q.b, u);
        FrameUnitCtl c;
        memset(&c, 0, sizeof c);
        c.mode = K11_WALK; c.k7_count = SB_FRAME_NOT_INDEXABLE;
        if (q.cidx) {
            const uint64_t a0 = q.cidx_at[u], a1 = q.cidx_at[u + 1];
            if (a1 > a0 && a1 - a0 - 1 <= q.max_chunks) { v = (uint32_t)(a1 - a0); c.mode = K11_CALLER; }
        } else {
            uint32_t decline;
            v = k11_k7_nseg(q, n, &decline);
        }
        q.uctl[u] = c;
    }
#pragma unroll
    for (unsigned m = 16; m; m >>= 1) n += shfl(n, lane_id() ^ m);
    if (lane_id() == 0 && n) atomic_add(q.in_total, (unsigned long long)n);
    scan_local_body(count + 1, [&](uint32_t) { return v; }, q.sg_offs, q.sg_tiles);
}
SB_DEVICE void k11_plan_tiles_body(const FrameDecodeBatchPlan& q) { scan_tiles_body(q.b.count + 1, 0, q.sg_tiles); }

SB_DEVICE void k11_survivors_body(const FrameDecodeBatchPlan& q) {
    if (k11_over(q)) return;
    const uint32_t count = q.b.count;
    const uint64_t total = k8b_at(q.sg_offs, q.sg_tiles, count);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t g = (uint64_t)block_idx() * wpb + warp_id(); g < total; g += nwarps) {
        const uint32_t u = k8b_unit_of(q.sg_offs, q.sg_tiles, count, g);
        k7_survivors_seg(k11_index_view(q, u), g - k8b_at(q.sg_offs, q.sg_tiles, u));
    }
}
SB_DEVICE void k11_stitch_body(const FrameDecodeBatchPlan& q) {
    const bool over = k11_over(q);
    for (uint32_t u = block_idx(); u < q.b.count; u += grid_dim()) {
        const IndexPlan p = k11_index_view(q, u);
        if (over || p.decline) {                                     // the same for every thread
            if (thread_idx() == 0) *p.count = SB_FRAME_NOT_INDEXABLE;
            continue;
        }
        k7_stitch_body(p);
        syncthreads();
    }
}

// thread per entry of the caller's index: the chain from s0 to n, linked by the chunk headers (see the file comment)
SB_DEVICE void k11_link_body(const FrameDecodeBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t total = k8b_at(q.sg_offs, q.sg_tiles, count);
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = (uint64_t)block_idx() * block_dim() + thread_idx(); g < total; g += nthreads) {
        const uint32_t u = k8b_unit_of(q.sg_offs, q.sg_tiles, count, g);
        const uint64_t e0 = k8b_at(q.sg_offs, q.sg_tiles, u), k = g - e0;
        const uint64_t ents = k8b_at(q.sg_offs, q.sg_tiles, u + 1) - e0;
        const uint8_t* in = unit_in(q.b, u);
        const uint64_t n = unit_in_len(q.b, u), s0 = q.fragment ? 0 : 10;
        const uint64_t* ix = k11_index(q, u);
        const uint64_t at = ix[k];
        bool ok;
        if (k + 1 == ents) ok = at == n;
        else {
            const uint64_t next = ix[k + 1];
            ok = at < n && n - at >= 4;
            if (ok) {
                const uint32_t len = (uint32_t)in[at + 1] | ((uint32_t)in[at + 2] << 8) | ((uint32_t)in[at + 3] << 16);
                ok = len >= 4 && n - at - 4 >= len && at + 4 + len == next;
            }
        }
        if (k == 0) {
            ok = ok && at == s0;
            if (ok && !q.fragment) { const uint8_t id[10] = {0xFF, 6, 0, 0, 's', 'N', 'a', 'P', 'p', 'Y'}; for (int m = 0; m < 10; m++) ok = ok && in[m] == id[m]; }
        }
        if (!ok) q.uctl[u].mode = K11_WALK;
    }
}

SB_DEVICE void k11_count_body(const FrameDecodeBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < count) {
        const uint32_t u = (uint32_t)i;
        FrameUnitCtl* c = &q.uctl[u];
        uint32_t mode = c->mode, range;
        if (!q.cidx && c->k7_count != SB_FRAME_NOT_INDEXABLE) { mode = K11_K7; range = c->k7_count; }
        else if (mode == K11_CALLER) range = (uint32_t)(k8b_at(q.sg_offs, q.sg_tiles, u + 1) - k8b_at(q.sg_offs, q.sg_tiles, u) - 1);
        else {                                                       // the reader's walk, counting (max_chunks + 1 do not fit)
            sb_error e;
            uint64_t produced;
            range = k5_walk(unit_in(q.b, u), unit_in_len(q.b, u), q.fragment != 0, q.max_chunks + 1,
                            [](uint32_t, const FChunk&) {}, &e, &produced);
        }
        v = range <= q.max_chunks ? range : q.max_chunks + 1;
        c->mode = mode; c->range = v; c->first_bad = K11_NONE;
    }
    scan_local_body(count + 1, [&](uint32_t) { return v; }, q.rg_offs, q.rg_tiles);
}
SB_DEVICE void k11_range_tiles_body(const FrameDecodeBatchPlan& q) { scan_tiles_body(q.b.count + 1, 0, q.rg_tiles); }

SB_DEVICE void k11_emit_body(const FrameDecodeBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t total = k11_over(q) ? 0 : k8b_at(q.sg_offs, q.sg_tiles, count);
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = (uint64_t)block_idx() * block_dim() + thread_idx(); g < total; g += nthreads) {
        const uint32_t u = k8b_unit_of(q.sg_offs, q.sg_tiles, count, g);
        if (q.uctl[u].mode != K11_K7 || !k11_fits(q, u)) continue;
        const IndexPlan p = k11_index_view(q, u);
        const uint64_t k = g - k8b_at(q.sg_offs, q.sg_tiles, u);
        if (k == 0) p.index[q.uctl[u].k7_count] = p.n;
        k7_emit_seg(p, k);
    }
}

SB_DEVICE void k11_parse_body(const FrameDecodeBatchPlan& q) {
    const uint32_t count = q.b.count;
    const uint64_t total = k11_slots(q);
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t j = (uint64_t)block_idx() * block_dim() + thread_idx(); j < total; j += nthreads) {
        const uint32_t u = k8b_unit_of(q.rg_offs, q.rg_tiles, count, j);
        if (q.uctl[u].mode == K11_WALK || !k11_fits(q, u)) continue;
        const uint64_t k = j - k11_range(q, u);
        const uint64_t* ix = k11_index(q, u);
        FChunk c;
        if (!k5_check_chunk(unit_in(q.b, u), unit_in_len(q.b, u), ix[k], ix[k + 1], &c)) { q.uctl[u].reparse = 1; c.dlen = 0; }
        q.chunks[j] = c;
    }
}

SB_DEVICE void k11_fill_body(const FrameDecodeBatchPlan& q) {
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx(); i < q.b.count; i += nthreads) {
        const uint32_t u = (uint32_t)i;
        FrameUnitCtl* c = &q.uctl[u];
        if (!k11_fits(q, u)) continue;
        sb_error werr;
        uint32_t live = c->range;
        set_status(&werr, SB_OK, 0, 0, 0);
        if (c->mode == K11_WALK || c->reparse) {
            FChunk* chunks = q.chunks + k11_range(q, u);
            uint64_t produced;
            live = k5_walk(unit_in(q.b, u), unit_in_len(q.b, u), q.fragment != 0, c->range,
                           [&](uint32_t k, const FChunk& ch) { chunks[k] = ch; }, &werr, &produced);
        }
        c->nchunks = live;
        c->walk_err = werr;
    }
}

// slot j's unit when the slot holds a live chunk of a unit that fits, else K11_NONE
SB_DEVICE uint32_t k11_live_unit(const FrameDecodeBatchPlan& q, uint64_t j) {
    const uint32_t u = k8b_unit_of(q.rg_offs, q.rg_tiles, q.b.count, j);
    return k11_fits(q, u) && j - k11_range(q, u) < q.uctl[u].nchunks ? u : K11_NONE;
}
SB_DEVICE void k11_oscan_local_body(const FrameDecodeBatchPlan& q) {
    const uint64_t total = k11_slots(q);
    const FChunk* ch = q.chunks;
    scan_local_body(q.max_chunks + 1, [&](uint32_t j) { return j < total && k11_live_unit(q, j) != K11_NONE ? ch[j].dlen : 0u; },
                    q.o_offs, q.o_tiles);
}
SB_DEVICE void k11_oscan_tiles_body(const FrameDecodeBatchPlan& q) { scan_tiles_body(q.max_chunks + 1, 0, q.o_tiles); }

// bytes unit u decodes to (its live chunks' lengths)
SB_DEVICE uint64_t k11_need(const FrameDecodeBatchPlan& q, uint32_t u) {
    return k11_out_at(q, k11_range(q, u + 1)) - k11_out_at(q, k11_range(q, u));
}

SB_DEVICE void k11_decode_body(const FrameDecodeBatchPlan& q) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const uint64_t total = k11_slots(q);
    const unsigned wpb = block_dim() >> 5;
    const uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    for (uint64_t j = (uint64_t)block_idx() * wpb + warp_id(); j < total; j += nwarps) {
        const uint32_t u = k11_live_unit(q, j);
        if (u == K11_NONE || k11_need(q, u) > unit_out_cap(q.b, u)) continue;
        const uint64_t r = k11_range(q, u), base = k11_out_at(q, r);
        const uint32_t code = k5_decode_chunk(tab, elems, q.chunks[j], unit_in(q.b, u), unit_out(q.b, u) + (k11_out_at(q, j) - base),
                                              &q.cst[j]);
        if (code != SB_OK && lane_id() == 0) atomic_min(&q.uctl[u].first_bad, (uint32_t)(j - r));
        syncwarp();
    }
}

// k5_finish's order per unit: chunk table too small, BufferTooSmall, the first failing chunk, the walk's error
SB_DEVICE void k11_finish_body(const FrameDecodeBatchPlan& q) {
    const sb_batch& b = q.b;
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx(); i < b.count; i += nthreads) {
        const uint32_t u = (uint32_t)i;
        const FrameUnitCtl c = q.uctl[u];
        const bool fits = k11_fits(q, u);
        sb_error* st = &b.statuses[u];
        uint64_t bytes = 0;
        if (!fits || (c.walk_err.code == SB_E_INVALID && c.walk_err.b == 1)) set_status(st, SB_E_INVALID, q.max_chunks, 1, 0);
        else {
            const uint64_t r = k11_range(q, u), need = k11_need(q, u);
            if (need > unit_out_cap(b, u)) set_status(st, SB_BUFFER_TOO_SMALL, unit_out_cap(b, u), need, 0);
            else if (c.first_bad != K11_NONE) { *st = q.cst[r + c.first_bad]; bytes = k11_out_at(q, r + c.first_bad) - k11_out_at(q, r); }
            else { *st = c.walk_err; bytes = need; }
        }
        b.out_lens[u] = (uint32_t)bytes;
        if (q.unit_chunks) q.unit_chunks[u] = fits && c.mode != K11_WALK && !c.reparse ? c.nchunks : 0;
    }
}

}  // namespace sbk
