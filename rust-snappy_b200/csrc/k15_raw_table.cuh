// k15_raw_table.cuh -- K15: seek tables of raw streams built from K8's block cuts, and byte ranges over many tabled raw
// streams in one call (sb_raw_table_build_batch_device_ws, sb_raw_table_decode_ranges_device_ws).
//
// A raw seek table is a 64-byte header and one 8-byte record per 64 KiB output block: the compressed offset of the
// block's first element and the masked CRC-32C of its decoded bytes. Block j's decoded offset (65536 * j) and length
// (min(65536, dn - 65536 * j)) are implied; its compressed bytes end where block j + 1's start (n for the last). The table
// holds no pointers and may be copied or moved.
//
// A stream is seekable when the reference's Decoder::decompress returns Ok and every block decodes alone to the same
// bytes: a multi-block unit (dn > 65536) that sb_decompress_batch_device_ws splits and decodes block-parallel with Ok,
// or a single-block unit (dn <= 65536, dn == 0 included) that decodes Ok. Anything else gets a header that says it is
// not seekable, with the reason (for diagnostics only).
//
// Build, over a batch:
//   K8b's split part unchanged (k8b_plan .. k8b_cuts, uniform cap 2^32 - 1, no output): every split unit's cut table.
//   k15_validate   warp per block of K8b's global block list, then warp per unit: a block is decoded with block-local
//                  bounds (k2_decode_stream<false>, as k8_block does) and a single-block unit as a whole stream
//                  (k2_decode_stream<true>), into the warp's own 64 KiB staging slot, and its masked CRC-32C is kept. A
//                  failing block marks its unit's control record (decline = 2), exactly where k8b_blocks would decline.
//   k15_size_*     K4's two-level scan of the table sizes (64, plus 8 per block for a seekable unit).
//   k15_export     thread per block of the global list: its record; thread per unit: d_table_offs, header, d_results.
// Why a seekable multi-block unit is exact: its cuts are those sb_decompress_batch_device_ws would decode with, and every
// block decodes Ok with block-local bounds; by K8's argument (k8_raw_split.cuh) the reference then returns Ok with the
// same bytes, which are the concatenation of the blocks'. A single-block unit is decoded exactly as K2 decodes it.
//
// Read: ranges (unit, lo, len) over `count` tabled streams. With end = min(lo + len, dn), range r decodes exactly the
// blocks that overlap [lo, end): [lo >> 16, (end - 1) >> 16], found without a search.
//   k15_plan       thread per range: the unit and its header checked, the range's first block and block count; K4's
//                  generic scan of the counts (k15_plan_tiles finishes it).
//   k15_decode     warp per (range, block) pair: the record checked against the build's bounds, the block decoded
//                  (interior blocks straight into the range's buffer, the head and tail block into the range's two
//                  64 KiB staging slots, of which a warp copy writes only the slice), then its CRC checked against the
//                  record. First failing block per range by atomic_min.
//   k15_finish     thread per range: status and out_len.
// No table content makes a read leave a stream (every block's bytes lie in [hl, n) of the stream it names, n checked
// against the caller's length) or write outside a range's buffer (block j's output is bounded by its implied length and
// the slice of [lo, end) it holds), its staging or the scratch.
//
// K15 does not share K13's plan and decode bodies through a template: see DESIGN.md section 4 (K13).
#pragma once
#include "k12_frame_range_decode.cuh"

namespace sbk {

static const uint64_t K15_MAGIC = 0x0001000042545352ull;   // "RSTB", format version 1 in the high half
static const uint32_t K15_MAX_COUNT = 1u << 31;
// Validation staging: 64 KiB per slot, one slot per warp of k15_validate. 4,096 slots (256 MiB) keep 31 warps per SM of
// an H100 decoding; a batch with fewer blocks than that gets one slot per block (DESIGN.md section 5 has the speed).
static const uint32_t K15_SLOTS = 4096;

// why a stream is not seekable (RawTableHead::reason)
enum : uint32_t { K15_SEEKABLE = 0, K15_BAD_HEADER = 1, K15_OVER_IN_BYTES = 2, K15_NOT_SPLIT = 3, K15_BLOCK_FAILED = 4 };

struct RawTableHead {              // 64 bytes
    uint64_t magic;
    uint64_t n;                    // compressed length of the stream the table was built over
    uint64_t dn;                   // decoded length (0 when not seekable)
    uint32_t hl;                   // varint header length (0 when not seekable)
    uint32_t nblocks;              // ceil(dn / 65536)
    uint32_t seekable;             // 1 or 0
    uint32_t reason;               // K15_* (0 when seekable)
    uint64_t _pad[3];
};
struct RawTableRec { uint32_t off; uint32_t crc; };

inline uint64_t k15_table_bytes(uint32_t nblocks) { return sizeof(RawTableHead) + (uint64_t)nblocks * sizeof(RawTableRec); }

// what k15_validate learns about unit u. kind 0: not seekable (reason); 1: seekable single-block (dn, crc); 2: the header
// announces more than one block, and the verdict is K8b's (uctl, the in_bytes bound)
struct RawUnit { uint32_t kind, dn, crc, reason; };

struct RawTableBuildPlan {
    RawBatchPlan q;                // K8b's plan and scratch: its out fields are not read
    RawUnit* units;                // count
    uint32_t* crc;                 // the global block list's masked CRCs
    uint8_t* slots;                // nslots * 64 KiB
    uint32_t nslots;
    uint8_t* tables;               // 8-byte aligned, the tables back to back
    uint64_t* table_offs;          // count + 1
    sb_frame_result* results;      // count
    uint64_t *sz_offs, *sz_tiles;  // scan over units of their table sizes
};

// the bound on Σ blocks of split units (k8b_carve sizes its cut array by it): a split unit announces at most 64 bytes per
// 3 compressed bytes, so it has at most n / 3072 + 1 blocks
inline uint64_t k15_blocks_bound(uint32_t count, uint64_t in_bytes) {
    const uint64_t in = in_bytes < K8B_MAX_IN_BYTES ? in_bytes : K8B_MAX_IN_BYTES;
    return in / 3072 + count;
}
inline uint64_t k15_tables_bytes(uint32_t count, uint64_t in_bytes) {
    return (uint64_t)count * sizeof(RawTableHead) + k15_blocks_bound(count, in_bytes) * sizeof(RawTableRec);
}

// K8b's carve, then the unit verdicts, the block CRCs, the size scan and the staging slots. Returns the bytes used (a pure
// function of count and in_bytes).
inline uint64_t k15_carve(void* scratch, uint32_t count, uint64_t in_bytes, RawTableBuildPlan* t) {
    const uint64_t k8 = k8b_carve(scratch, count, in_bytes, t ? &t->q : nullptr);
    const uint64_t blocks = k15_blocks_bound(count, in_bytes), units = (uint64_t)count + 1;
    const uint64_t slots = blocks + count < K15_SLOTS ? blocks + count : K15_SLOTS;
    const uintptr_t base = ((uintptr_t)scratch + k8 + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    RawUnit* u = (RawUnit*)take(count * sizeof(RawUnit));
    uint32_t* crc = (uint32_t*)take(blocks * 4);
    uint64_t* offs = (uint64_t*)take((units + 1) * 8);
    uint64_t* tiles = (uint64_t*)take((units / K4_TILE + 3) * 8);
    uint8_t* sl = (uint8_t*)take(slots * kMaxBlock);
    if (t) { t->units = u; t->crc = crc; t->sz_offs = offs; t->sz_tiles = tiles; t->slots = sl; t->nslots = (uint32_t)slots; }
    return k8 + at + 256;
}

SB_DEVICE uint64_t k15_blocks(const RawBatchPlan& q) { return k8b_over(q) ? 0 : k8b_at(q.bk_offs, q.bk_tiles, q.b.count); }

// ---- build
SB_DEVICE void k15_validate_body(const RawTableBuildPlan& t) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const RawBatchPlan& q = t.q;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id(), nw = (uint64_t)grid_dim() * wpb;
    const uint64_t active = nw < t.nslots ? nw : t.nslots;            // warps with a slot of their own
    if (w >= active) return;
    uint8_t* slot = t.slots + w * kMaxBlock;
    const uint32_t count = q.b.count;
    const uint64_t blocks = k15_blocks(q);
    for (uint64_t g = w; g < blocks + count; g += active) {
        if (g < blocks) {
            const uint32_t u = k8b_unit_of(q.bk_offs, q.bk_tiles, count, g);
            const RawPlan p = k8b_view(q, u);
            if (k8_declined(p)) continue;
            const uint64_t j = g - (uint64_t)(p.cut - q.cut - u);
            const uint32_t a = p.cut[j], b = p.cut[j + 1];
            const uint64_t dn = p.ctl->dn, want = dn - (j << 16) < 65536 ? dn - (j << 16) : 65536;
            uint32_t code = SB_E_INVALID;                              // bad cuts cannot happen once they were accepted
            if (a <= b && b <= p.n) code = k2_decode_stream<false>(p.in + a, b - a, slot, want, nullptr, nullptr, elems);
            syncwarp();
            const uint32_t crc = code == SB_OK ? k3_warp_crc32c_masked(tab, slot, (uint32_t)want) : 0u;
            if (lane_id() == 0) {
                t.crc[g] = crc;
                if (code != SB_OK) p.ctl->decline = 2;
            }
        } else {
            const uint32_t u = (uint32_t)(g - blocks), n = unit_in_len(q.b, u);
            const uint8_t* in = unit_in(q.b, u);
            uint64_t v = 0;
            const uint32_t hl = n ? k2_read_header(in, n, &v) : 0;
            RawUnit r;
            r.kind = 0; r.dn = 0; r.crc = 0; r.reason = K15_BAD_HEADER;
            if (hl && v <= kMaxInput) {
                if (v > kMaxBlock) { r.kind = 2; r.reason = K15_SEEKABLE; }
                else {
                    const uint32_t code = k2_decode_stream<true>(in, n, slot, kMaxBlock, nullptr, nullptr, elems);
                    syncwarp();
                    if (code == SB_OK) {
                        r.kind = 1; r.dn = (uint32_t)v; r.reason = K15_SEEKABLE;
                        r.crc = k3_warp_crc32c_masked(tab, slot, (uint32_t)v);
                    } else r.reason = K15_BLOCK_FAILED;
                }
            }
            if (lane_id() == 0) t.units[u] = r;
        }
        syncwarp();
    }
}

struct RawVerdict { uint32_t seekable, dn, hl, nblocks, reason; };
SB_DEVICE RawVerdict k15_verdict(const RawTableBuildPlan& t, uint32_t u) {
    const RawUnit r = t.units[u];
    const RawCtl& c = t.q.uctl[u];
    RawVerdict v;
    v.seekable = 0; v.dn = 0; v.hl = 0; v.nblocks = 0; v.reason = r.reason;
    if (r.kind == 1) { v.seekable = 1; v.dn = r.dn; v.hl = c.hl; v.nblocks = (r.dn + 65535) >> 16; }
    else if (r.kind == 2) {
        if (k8b_over(t.q)) v.reason = K15_OVER_IN_BYTES;
        else if (c.decline) v.reason = c.decline == 2 ? K15_BLOCK_FAILED : K15_NOT_SPLIT;
        else { v.seekable = 1; v.dn = (uint32_t)c.dn; v.hl = c.hl; v.nblocks = c.nblk; }
    }
    return v;
}

SB_DEVICE uint64_t k15_table_at(const RawTableBuildPlan& t, uint32_t u) { return k8b_at(t.sz_offs, t.sz_tiles, u); }

// Σ sizes of a tile stays below 2^32: at most 1,024 headers and 1,024 * 65,536 records
SB_DEVICE void k15_size_local_body(const RawTableBuildPlan& t) {
    const uint32_t count = t.q.b.count;
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < count) {
        const RawVerdict r = k15_verdict(t, (uint32_t)i);
        v = (uint32_t)sizeof(RawTableHead) + (r.seekable ? r.nblocks * (uint32_t)sizeof(RawTableRec) : 0u);
    }
    scan_local_body(count + 1, [&](uint32_t) { return v; }, t.sz_offs, t.sz_tiles);
}
SB_DEVICE void k15_size_tiles_body(const RawTableBuildPlan& t) { scan_tiles_body(t.q.b.count + 1, 0, t.sz_tiles); }

// threads over the global block list: the records of seekable split units; then threads over units [0, count]: the
// offsets, headers, single-block records and results. Every field is written, padding included.
SB_DEVICE void k15_export_body(const RawTableBuildPlan& t) {
    const RawBatchPlan& q = t.q;
    const uint32_t count = q.b.count;
    const uint64_t blocks = k15_blocks(q);
    const uint64_t i0 = (uint64_t)block_idx() * block_dim() + thread_idx(), nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = i0; g < blocks; g += nthreads) {
        const uint32_t u = k8b_unit_of(q.bk_offs, q.bk_tiles, count, g);
        if (q.uctl[u].decline) continue;
        const uint64_t b0 = k8b_at(q.bk_offs, q.bk_tiles, u), j = g - b0;
        RawTableRec rec;
        rec.off = q.cut[b0 + u + j]; rec.crc = t.crc[g];
        ((RawTableRec*)(t.tables + k15_table_at(t, u) + sizeof(RawTableHead)))[j] = rec;
    }
    for (uint64_t i = i0; i <= count; i += nthreads) {
        const uint32_t u = (uint32_t)i;
        const uint64_t at = k15_table_at(t, u);
        t.table_offs[u] = at;
        if (u == count) continue;
        const RawVerdict v = k15_verdict(t, u);
        RawTableHead h;
        h.magic = K15_MAGIC; h.n = unit_in_len(q.b, u); h.dn = v.dn; h.hl = v.hl; h.nblocks = v.nblocks;
        h.seekable = v.seekable; h.reason = v.reason; h._pad[0] = h._pad[1] = h._pad[2] = 0;
        *(RawTableHead*)(t.tables + at) = h;
        if (v.seekable && t.units[u].kind == 1 && v.nblocks) {
            RawTableRec rec;
            rec.off = v.hl; rec.crc = t.units[u].crc;
            *(RawTableRec*)(t.tables + at + sizeof(RawTableHead)) = rec;
        }
        sb_frame_result res;
        if (v.seekable) set_status(&res.status, SB_OK, 0, 0, 0);
        else set_status(&res.status, SB_E_INVALID, u, 0, 5);
        res.bytes = v.dn; res.nchunks = v.nblocks; res._pad = 0;
        t.results[u] = res;
    }
}

// ---- read
struct RawRangePlan {
    const void* const* tables; const uint8_t* const* ins; const uint64_t* in_lens; uint32_t count;
    const uint32_t* unit; const uint64_t *lo, *len;
    uint8_t* const* outs;
    uint64_t* out_lens;
    sb_error* statuses;
    uint32_t nranges;
    RangeRec* rec;                 // nranges: first block, block count, first failing block
    uint64_t *pr_offs, *pr_tiles;  // scan over ranges of their block counts
    uint8_t* staging;              // 2 slots of K12_SLOT bytes per range
};

// Scratch of a read: K12's range part exactly (records, pair scan, staging). Returns the bytes used.
inline uint64_t k15_ranges_carve(void* scratch, uint32_t nranges, RawRangePlan* q) {
    RangePlan r;
    const uint64_t bytes = k12_carve(scratch, nranges, &r);
    if (q) { q->nranges = nranges; q->rec = r.rec; q->pr_offs = r.pr_offs; q->pr_tiles = r.pr_tiles; q->staging = r.staging; }
    return bytes;
}

SB_DEVICE const RawTableRec* k15_recs(const RawTableHead* h) { return (const RawTableRec*)(h + 1); }
SB_DEVICE bool k15_is_table(const RawTableHead* h) { return h && h->magic == K15_MAGIC; }

// range r's table header when the unit is in range and the table is one of this format built over a stream of the
// length given for the unit; null otherwise
SB_DEVICE const RawTableHead* k15_head(const RawRangePlan& q, uint32_t r) {
    const uint32_t u = q.unit[r];
    if (u >= q.count) return nullptr;
    const RawTableHead* h = (const RawTableHead*)q.tables[u];
    const uint64_t n = q.in_lens[u];
    return k15_is_table(h) && h->n == n && (q.ins[u] || n == 0) ? h : nullptr;
}
// the header bounds every build writes: dn < 2^32 and ceil(dn / 65536) blocks (so at most 65,536)
SB_DEVICE bool k15_head_ok(const RawTableHead* h) { return h->dn <= kMaxInput && h->nblocks == (h->dn + 65535) >> 16; }
// block j's record keeps the build's bounds: its bytes [off_j, off_{j+1} or n) lie inside [hl, n), offsets non-decreasing
SB_DEVICE bool k15_rec_ok(const RawTableHead* h, uint64_t j) {
    if (!k15_head_ok(h) || j >= h->nblocks) return false;
    const RawTableRec* t = k15_recs(h);
    const uint64_t a = t[j].off, b = j + 1 < h->nblocks ? t[j + 1].off : h->n;
    return h->hl <= a && a <= b && b <= h->n;
}

SB_DEVICE void k15_plan_body(const RawRangePlan& q) {
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < q.nranges) {
        const RawTableHead* h = k15_head(q, (uint32_t)i);
        uint32_t first = 0;
        if (h && h->seekable == 1 && k15_head_ok(h)) {
            const uint64_t lo = q.lo[i], end = k12_end(lo, q.len[i], h->dn);
            if (end > lo) { first = (uint32_t)(lo >> 16); v = (uint32_t)((end - 1) >> 16) - first + 1; }
        }
        RangeRec r;
        r.first = first; r.pairs = v; r.first_bad = K12_NONE; r._pad = 0;
        q.rec[i] = r;
    }
    scan_local_body(q.nranges + 1, [&](uint32_t) { return v; }, q.pr_offs, q.pr_tiles);
}
SB_DEVICE void k15_plan_tiles_body(const RawRangePlan& q) { scan_tiles_body(q.nranges + 1, 0, q.pr_tiles); }

// GATHER (the gather call, k17_table_gather.cuh): the head and tail pairs that are not inside [lo, end) are left to K17's
// gather decode (only they can straddle lo or end: blocks are implied by their index), so no warp needs staging and
// the whole grid decodes. HOST (the host-stream gather, k18_host_gather.cuh): only the pool's warps decode, warp w
// fetching each body that fits into its compressed slot cpool + w * K18_CSLOT first.
template <bool GATHER = false, bool HOST = false>
SB_DEVICE void k15_decode_body(const RawRangePlan& q, uint8_t* cpool = nullptr) {
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t pairs = k8b_at(q.pr_offs, q.pr_tiles, q.nranges);
    uint64_t nwarps = (uint64_t)grid_dim() * wpb;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id();
    if (HOST) { nwarps = k12_pool_warps(nwarps, q.nranges); if (w >= nwarps) return; }
    uint8_t* const cslot = HOST ? cpool + w * K18_CSLOT : nullptr;
    for (uint64_t g = w; g < pairs; g += nwarps) {
        const uint32_t r = k8b_unit_of(q.pr_offs, q.pr_tiles, q.nranges, g);
        const uint32_t first = q.rec[r].first, j = first + (uint32_t)(g - k8b_at(q.pr_offs, q.pr_tiles, r));
        const uint32_t u = q.unit[r];                                    // a range with pairs passed k15_head
        const RawTableHead* h = (const RawTableHead*)q.tables[u];
        uint32_t code = SB_E_INVALID;
        if (k15_rec_ok(h, j)) {
            const RawTableRec* t = k15_recs(h);
            const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->dn), off = (uint64_t)j << 16;
            const uint64_t dl = h->dn - off < 65536 ? h->dn - off : 65536;
            const uint32_t a = t[j].off, b = j + 1 < h->nblocks ? t[j + 1].off : (uint32_t)h->n;
            const bool inside = off >= lo && off + dl <= end;
            if (GATHER && !inside) { syncwarp(); continue; }
            uint8_t* dst = inside ? q.outs[r] + (off - lo) : q.staging + ((uint64_t)r * 2 + (j == first ? 0 : 1)) * K12_SLOT;
            if (GATHER) K17_COUNT_DECODE();
            if (HOST) code = k2_decode_stream<false>(k18_body<true>(q.ins[u] + a, b - a, cslot), b - a, dst, dl, nullptr, nullptr, elems);
            else code = k2_decode_stream<false>(q.ins[u] + a, b - a, dst, dl, nullptr, nullptr, elems);
            syncwarp();
            if (code == SB_OK && k3_warp_crc32c_masked(tab, dst, (uint32_t)dl) != t[j].crc) code = SB_CHECKSUM;
            if (code == SB_OK && !inside) {                               // the slice of [lo, end) a head or tail block holds
                const uint64_t s = off > lo ? off : lo, e = off + dl < end ? off + dl : end;
                warp_copy(q.outs[r] + (s - lo), dst + (s - off), (uint32_t)(e - s));
            }
        }
        if (code != SB_OK && lane_id() == 0) atomic_min(&q.rec[r].first_bad, j);
        syncwarp();
    }
}

// per range, in priority order: unit out of range, not a raw table of this stream, not seekable, the first covered block
// that breaks the build's bounds (c=3) or does not decode to its CRC (c=4), else Ok
SB_DEVICE void k15_finish_body(const RawRangePlan& q) {
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t r = (uint64_t)block_idx() * block_dim() + thread_idx(); r < q.nranges; r += nthreads) {
        const uint32_t u = q.unit[r];
        const RawTableHead* h = k15_head(q, (uint32_t)r);
        sb_error* st = &q.statuses[r];
        uint64_t got = 0;
        if (!h) {
            if (u >= q.count) set_status(st, SB_E_INVALID, u, q.count, 1);
            else {
                const RawTableHead* t = (const RawTableHead*)q.tables[u];
                set_status(st, SB_E_INVALID, q.in_lens[u], k15_is_table(t) ? t->n : 0, 2);
            }
        } else if (h->seekable != 1) set_status(st, SB_E_INVALID, u, 0, 5);
        else {
            const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->dn);
            const uint32_t bad = q.rec[r].first_bad;
            if (!k15_head_ok(h) && end > lo) set_status(st, SB_E_INVALID, lo >> 16, 0, 3);   // every block breaks them
            else if (bad != K12_NONE) {
                set_status(st, SB_E_INVALID, bad, 0, k15_rec_ok(h, bad) ? 4 : 3);
                const uint64_t stop = (uint64_t)bad << 16;
                got = stop > lo ? stop - lo : 0;
            } else {
                set_status(st, SB_OK, 0, 0, 0);
                got = end > lo ? end - lo : 0;
            }
        }
        q.out_lens[r] = got;
    }
}

}  // namespace sbk
