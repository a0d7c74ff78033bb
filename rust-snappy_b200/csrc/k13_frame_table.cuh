// k13_frame_table.cuh -- K13: seek tables of frame streams, and byte ranges over many tabled streams in one call
// (sb_frame_table_build_device_ws, sb_frame_table_decode_ranges_device_ws).
//
// A seek table is what K12 learns about a stream before it decodes anything, kept: a header, then one 32-byte record per
// data chunk in stream order (K5's FChunk and the chunk's decoded offset). It holds no pointers, and the header plus
// its first nchunks records is a complete table, so a table may be cut to k13_table_bytes(nchunks) or moved.
//   build     K5's index phase unchanged (K7 or the caller's index, parse, walk when needed, scan), then
//   k13_export  thread per chunk slot: record k = chunks[k] + its scanned offset; one more thread writes the header
//               and the stream's result.
//
// A read takes ranges (unit, lo, len) over `count` tabled streams and runs K12's per-range logic inside each unit's
// records, with no pass over any stream's headers:
//   k13_plan        thread per range: the unit and its table header checked, then K12's two binary searches over the
//                   unit's records give the verified run [first, last] (see k12_frame_range_decode.cuh for which chunks
//                   a range verifies and why the result is exact); K4's generic scan of the pair counts.
//   k13_decode      warp per pair, grid-striding over the pair total: K12's interior / head / tail handling and its two
//                   64 KiB staging slots per range, k5_decode_chunk unchanged. First failing chunk per range by
//                   atomic_min. Chunk statuses go to a per-warp sink: tables are read-only and have no status array.
//   k13_finish      warp per range: the status and out_len in K12's order behind the two table checks; a range whose
//                   first failing chunk is set decodes that one chunk again into its staging to get the chunk's status.
//
// Tables are trusted only as far as is cheap to check. The header must carry the magic and the stream length the
// caller passes; every record a decode touches must stay within the bounds every build writes (body inside [0, n), a
// data chunk type, body <= 76,490 bytes, decoded <= 65,536 bytes, a stored body as long as its output, a non-negative
// slice of [lo, end)), else it fails as its chunk with Invalid{k, 0, 3}. Every decoded chunk is CRC-checked, so a table
// paired with other bytes of the same length gives errors, and no table content makes a read leave the stream or a
// write leave a range's buffer, its staging or the scratch.
//
// K13 does not share K12's plan and decode bodies through a template: see DESIGN.md section 4 (K13).
#pragma once
#include "k12_frame_range_decode.cuh"

namespace sbk {

static const uint64_t K13_MAGIC = 0x0001000042545342ull;   // "BSTB", format version 1 in the high half
static const uint32_t K13_MAX_COUNT = 1u << 31;

struct TableHead {                 // 64 bytes
    uint64_t magic;
    uint64_t n;                    // compressed length of the stream the table was built over
    uint64_t total;                // decoded length of the chunks in the table
    uint32_t nchunks;
    uint32_t full;                 // 1: the chunk table was too small (walk_err = Invalid{max_chunks, 1})
    sb_error walk_err;             // the walk's stopping status
};
struct TableRec { uint64_t body_off; uint32_t body_len; uint32_t dlen; uint32_t want_crc; uint32_t type; uint64_t off; };

inline uint64_t k13_table_bytes(uint32_t nchunks) { return sizeof(TableHead) + (uint64_t)nchunks * sizeof(TableRec); }

struct TablePlan {
    const void* const* tables; const uint8_t* const* ins; const uint64_t* in_lens; uint32_t count;
    const uint32_t* unit; const uint64_t *lo, *len;
    uint8_t* const* outs;
    uint64_t* out_lens;
    sb_error* statuses;
    uint32_t nranges;
    RangeRec* rec;                 // nranges
    uint64_t *pr_offs, *pr_tiles;  // scan over ranges of their pair counts
    uint8_t* staging;              // 2 slots of K12_SLOT bytes per range
};

// Scratch of a read: K12's range part exactly (records, pair scan, staging). Returns the bytes used.
inline uint64_t k13_carve(void* scratch, uint32_t nranges, TablePlan* q) {
    RangePlan r;
    const uint64_t bytes = k12_carve(scratch, nranges, &r);
    if (q) { q->nranges = nranges; q->rec = r.rec; q->pr_offs = r.pr_offs; q->pr_tiles = r.pr_tiles; q->staging = r.staging; }
    return bytes;
}

SB_DEVICE const TableRec* k13_recs(const TableHead* h) { return (const TableRec*)(h + 1); }
SB_DEVICE bool k13_is_table(const TableHead* h) { return h && h->magic == K13_MAGIC && h->nchunks <= K12_MAX_CHUNKS; }

// range r's table header when the unit is in range and the table is one of this format built over a stream of the
// length given for the unit; null otherwise
SB_DEVICE const TableHead* k13_head(const TablePlan& q, uint32_t r) {
    const uint32_t u = q.unit[r];
    if (u >= q.count) return nullptr;
    const TableHead* h = (const TableHead*)q.tables[u];
    const uint64_t n = q.in_lens[u];
    return k13_is_table(h) && h->n == n && (q.ins[u] || n == 0) ? h : nullptr;
}

// the bounds every build writes, and a non-negative slice [max(off, lo), min(off + dlen, end)) of [lo, end). A range
// that starts past total has end = total < lo: no chunk of a valid table is verified by it, and a record that claims to
// be must fail here, before its slice length end - lo wraps around.
SB_DEVICE bool k13_rec_ok(const TableRec& t, uint64_t n, uint64_t lo, uint64_t end) {
    return t.body_off <= n && t.body_len <= n - t.body_off && t.body_len <= K5_MAX_CBLOCK && t.dlen <= kMaxBlock &&
           (t.type == 0 || (t.type == 1 && t.body_len == t.dlen)) && t.off <= ~0ull - t.dlen && lo <= end &&
           t.off <= end && t.off + t.dlen >= lo;
}
SB_DEVICE FChunk k13_chunk(const TableRec& t) {
    FChunk c;
    c.body_off = t.body_off; c.body_len = t.body_len; c.dlen = t.dlen; c.want_crc = t.want_crc; c.type = t.type;
    return c;
}

// ---- build: thread per chunk slot, and thread cap_chunks for the header and the stream's result
SB_DEVICE void k13_export_body(const DecodePlan& p, TableHead* table) {
    const uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx();
    const DecodeCtl* ctl = p.ctl;
    if (i < ctl->nchunks) {
        const FChunk c = p.chunks[i];
        TableRec t;
        t.body_off = c.body_off; t.body_len = c.body_len; t.dlen = c.dlen; t.want_crc = c.want_crc; t.type = c.type;
        t.off = k8b_at(p.ooff, p.tiles, i);
        ((TableRec*)(table + 1))[i] = t;
    }
    if (i == p.cap_chunks) {
        TableHead h;
        h.magic = K13_MAGIC; h.n = p.n; h.total = ctl->produced; h.nchunks = ctl->nchunks;
        h.full = k12_table_full(ctl) ? 1u : 0u; h.walk_err = ctl->walk_err;
        *table = h;
        sb_frame_result r;
        r.status = ctl->walk_err; r.bytes = ctl->produced; r.nchunks = ctl->nchunks; r._pad = 0;
        *p.result = r;
    }
}

// ---- read
SB_DEVICE void k13_plan_body(const TablePlan& q) {
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < q.nranges) {
        const TableHead* h = k13_head(q, (uint32_t)i);
        uint32_t first = 0;
        if (h && !h->full) {
            const TableRec* t = k13_recs(h);
            const uint64_t lo = q.lo[i], end = k12_end(lo, q.len[i], h->total);
            uint32_t a = 0, b = h->nchunks;                              // first k with off_k + max(dlen_k, 1) > lo
            while (a < b) {
                const uint32_t m = a + (b - a) / 2;
                const uint32_t dl = t[m].dlen;
                if (t[m].off + (dl ? dl : 1) > lo) b = m; else a = m + 1;
            }
            first = a;
            b = h->nchunks;                                              // first k >= first with off_k >= end
            while (a < b) {
                const uint32_t m = a + (b - a) / 2;
                if (t[m].off >= end) b = m; else a = m + 1;
            }
            v = a - first;
        }
        RangeRec r;
        r.first = first; r.pairs = v; r.first_bad = K12_NONE; r._pad = 0;
        q.rec[i] = r;
    }
    scan_local_body(q.nranges + 1, [&](uint32_t) { return v; }, q.pr_offs, q.pr_tiles);
}
SB_DEVICE void k13_plan_tiles_body(const TablePlan& q) { scan_tiles_body(q.nranges + 1, 0, q.pr_tiles); }

// GATHER (the gather call, k17_table_gather.cuh): only pairs inside [lo, end) decode here, on the whole grid. The head
// and tail pairs that are not inside are left to K17's gather decode. A middle pair that is not inside (only a table
// whose offsets were tampered with has one) sets rec[r]._pad, and the gather's finish walks that range's run for it.
// HOST (the host-stream gather, k18_host_gather.cuh): only the pool's warps decode, warp w fetching each body into its
// compressed slot cpool + w * K18_CSLOT first.
template <bool GATHER = false, bool HOST = false>
SB_DEVICE void k13_decode_body(const TablePlan& q, uint8_t* cpool = nullptr) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const unsigned wpb = block_dim() >> 5;
    sb_error* sink = (sb_error*)(smem() + K3_TABLE_BYTES + wpb * K2_SMEM_PER_WARP) + warp_id();
    const uint64_t pairs = k8b_at(q.pr_offs, q.pr_tiles, q.nranges);
    uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id();
    if (HOST) { nwarps = k12_pool_warps(nwarps, q.nranges); if (w >= nwarps) return; }
    uint8_t* const cslot = HOST ? cpool + w * K18_CSLOT : nullptr;
    for (uint64_t g = w; g < pairs; g += nwarps) {
        const uint32_t r = k8b_unit_of(q.pr_offs, q.pr_tiles, q.nranges, g);
        const uint32_t first = q.rec[r].first, k = first + (uint32_t)(g - k8b_at(q.pr_offs, q.pr_tiles, r));
        const uint32_t u = q.unit[r];                                    // a range with pairs passed k13_head
        const TableHead* h = (const TableHead*)q.tables[u];
        const TableRec t = k13_recs(h)[k];
        const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->total);
        uint32_t code = SB_E_INVALID;
        if (k13_rec_ok(t, h->n, lo, end)) {
            const bool inside = t.off >= lo && t.off + t.dlen <= end;
            if (GATHER && !inside) {
                if (k != first && k + 1 != first + q.rec[r].pairs && lane_id() == 0) q.rec[r]._pad = 1;
                syncwarp();
                continue;
            }
            uint8_t* dst = inside ? q.outs[r] + (t.off - lo) : q.staging + ((uint64_t)r * 2 + (k == first ? 0 : 1)) * K12_SLOT;
            if (GATHER) K17_COUNT_DECODE();
            FChunk c = k13_chunk(t);
            const uint8_t* in = q.ins[u];
            if (HOST) { in = k18_body<true>(in + t.body_off, t.body_len, cslot); c.body_off = 0; }
            code = k5_decode_chunk(tab, elems, c, in, dst, sink);
            if (code == SB_OK && !inside) {                               // the slice of [lo, end) a head or tail chunk holds
                const uint64_t a = t.off > lo ? t.off : lo, e = t.off + t.dlen < end ? t.off + t.dlen : end;
                warp_copy(q.outs[r] + (a - lo), dst + (a - t.off), (uint32_t)(e - a));
            }
        }
        if (code != SB_OK && lane_id() == 0) atomic_min(&q.rec[r].first_bad, k);
        syncwarp();
    }
}

// per range, in priority order: unit out of range, not a table of this stream, chunk table too small, the first failing
// verified chunk, past the end: the walk's stopping error (Ok at a clean end), else Ok. GATHER: a range whose rec._pad the
// interior decode set first decodes its middle pairs that are not inside [lo, end) into the warp's pool slot, as the
// range call decodes them into its staging; the failing chunk decodes again into that slot.
template <bool GATHER = false>
SB_DEVICE void k13_finish_body(const TablePlan& q) {
    uint32_t* tab = (uint32_t*)smem();
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const unsigned wpb = block_dim() >> 5;
    const bool lead = lane_id() == 0;
    uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id();
    if (GATHER) { nwarps = k12_pool_warps(nwarps, q.nranges); if (w >= nwarps) return; }
    for (uint64_t r = w; r < q.nranges; r += nwarps) {
        const uint32_t u = q.unit[r];
        const TableHead* h = k13_head(q, (uint32_t)r);
        sb_error* st = &q.statuses[r];
        uint64_t got = 0;
        if (!h) {
            if (lead) {
                if (u >= q.count) set_status(st, SB_E_INVALID, u, q.count, 1);
                else {
                    const TableHead* t = (const TableHead*)q.tables[u];
                    set_status(st, SB_E_INVALID, q.in_lens[u], k13_is_table(t) ? t->n : 0, 2);
                }
            }
        } else {
            const uint64_t total = h->total, lo = q.lo[r], len = q.len[r], end = k12_end(lo, len, total);
            if (GATHER && q.rec[r]._pad) {
                const RangeRec rr = q.rec[r];
                uint8_t* slot = q.staging + w * K12_SLOT;
                for (uint32_t k = rr.first + 1; k + 1 < rr.first + rr.pairs; k++) {
                    const TableRec t = k13_recs(h)[k];
                    if (!k13_rec_ok(t, h->n, lo, end) || (t.off >= lo && t.off + t.dlen <= end)) continue;
                    // st takes the chunk's status for now; every branch below writes the range's own
                    if (k5_decode_chunk(tab, elems, k13_chunk(t), q.ins[u], slot, st) != SB_OK) {
                        if (lead) atomic_min(&q.rec[r].first_bad, k);
                    } else {
                        const uint64_t a = t.off > lo ? t.off : lo, e = t.off + t.dlen < end ? t.off + t.dlen : end;
                        warp_copy(q.outs[r] + (a - lo), slot + (a - t.off), (uint32_t)(e - a));
                    }
                    syncwarp();
                }
            }
            const uint32_t bad = q.rec[r].first_bad;
            got = end > lo ? end - lo : 0;
            if (h->full) { if (lead) *st = h->walk_err; got = 0; }
            else if (bad != K12_NONE) {
                const TableRec t = k13_recs(h)[bad];
                if (!k13_rec_ok(t, h->n, lo, end)) { if (lead) set_status(st, SB_E_INVALID, bad, 0, 3); }
                else k5_decode_chunk(tab, elems, k13_chunk(t), q.ins[u], q.staging + (GATHER ? w : r * 2) * K12_SLOT, st);
                const uint64_t stop = t.off < end ? t.off : end;           // off_k* for a valid table
                got = stop > lo ? stop - lo : 0;
            }
            else if (lo > total || len > total - lo) { if (lead) *st = h->walk_err; }
            else if (lead) set_status(st, SB_OK, 0, 0, 0);
        }
        if (lead) q.out_lens[r] = got;
        syncwarp();
    }
}

}  // namespace sbk
