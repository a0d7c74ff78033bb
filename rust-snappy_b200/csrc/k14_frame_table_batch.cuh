// k14_frame_table_batch.cuh -- K14: seek tables of a batch of frame streams in one call
// (sb_frame_table_build_batch_device_ws).
//
// Replaces one sb_frame_table_build_device_ws per stream. K11's index phase (k11_plan .. k11_oscan_tiles, unchanged)
// leaves in its scratch everything a K13 table holds, for every unit that fits the batch's chunk table: its chunk
// records (chunks[range .. range + nchunks)), its live count and walk status (uctl), and every chunk's decoded offset
// (k11_out_at(j) - k11_out_at(range)). K14 writes those as K13 tables, packed back to back in batch order:
//   k14_size_local  thread per unit: its table size, 64 + 32 * nchunks when it fits, 64 (a header) when it does not;
//                   K4's generic scan over units (k14_size_tiles finishes it).
//   k14_export      thread per chunk slot: record k of unit u = chunks[range_u + k] + its offset, for k < nchunks_u;
//                   then thread per unit: d_table_offs, the header and d_results.
//
// Why a fitting unit's table is the single build's. The single build runs K5's index phase: K7 or the caller's index,
// K5's parse, the reader's walk when anything is unusual, and the scan of the decoded lengths. K11 runs the same device
// functions per unit and gives each unit that fits the reader's chunk list and stopping error (the argument in
// k11_frame_batch_decode.cuh): so the records, the live count, the walk status and, by the scan, every decoded offset
// and the total are the single build's. With a chunk table large enough the single build's table is never full, and a
// unit that fits never is either. Every header and record field is written explicitly (no struct padding exists), as are
// sb_error::_pad and sb_frame_result::_pad, so the bytes are equal too.
//
// A unit that does not fit (the first whose range ends past max_chunks, and every unit after it) gets a 64-byte header
// with total 0, nchunks 0, full = 1 and walk_err = Invalid{max_chunks, 1}, and the result {Invalid{max_chunks, 1}, 0, 0}:
// every read over it gives that status and no bytes, as a read over a single build whose chunk table was too small does.
//
// The scratch is not zeroed. Only fields K11 writes for every unit are read (range, and nchunks / walk_err after
// k11_fits, since k11_fill skips units that do not fit); the slot scan covers the live slots only.
#pragma once
#include "k11_frame_batch_decode.cuh"
#include "k13_frame_table.cuh"

namespace sbk {

struct TableBatchPlan {
    FrameDecodeBatchPlan q;            // K11's plan and scratch (its out_* fields are not read)
    uint8_t* tables;                   // 8-byte aligned, the tables back to back
    uint64_t* table_offs;              // count + 1
    sb_frame_result* results;          // count
    uint64_t *sz_offs, *sz_tiles;      // scan over units of their table sizes
};

// K11's carve, then the size scan. Returns the bytes used (a pure function of count, in_bytes and max_chunks).
inline uint64_t k14_carve(void* scratch, uint32_t count, uint64_t in_bytes, uint32_t max_chunks, TableBatchPlan* t) {
    const uint64_t k11 = k11_carve(scratch, count, in_bytes, max_chunks, t ? &t->q : nullptr);
    const uint64_t units = (uint64_t)count + 1;
    const uint64_t offs = (units + 1) * 8, tiles = (units / K4_TILE + 3) * 8;
    if (t) {
        const uintptr_t base = ((uintptr_t)scratch + k11 + 255) / 256 * 256;
        t->sz_offs = (uint64_t*)base;
        t->sz_tiles = (uint64_t*)(base + (offs + 255) / 256 * 256);
    }
    return k11 + (offs + 255) / 256 * 256 + (tiles + 255) / 256 * 256 + 256;
}

// the bound on the packed tables' total: a header per unit and a record per slot of the chunk table
inline uint64_t k14_tables_bytes(uint32_t count, uint32_t max_chunks) {
    return (uint64_t)count * sizeof(TableHead) + (uint64_t)max_chunks * sizeof(TableRec);
}

SB_DEVICE uint64_t k14_table_at(const TableBatchPlan& t, uint32_t u) { return k8b_at(t.sz_offs, t.sz_tiles, u); }

// Σ sizes of a tile stays below 2^32: at most 1,024 headers and max_chunks < 2^22 records
SB_DEVICE void k14_size_local_body(const TableBatchPlan& t) {
    const FrameDecodeBatchPlan& q = t.q;
    const uint32_t count = q.b.count;
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < count) {
        const uint32_t u = (uint32_t)i;
        v = (uint32_t)sizeof(TableHead) + (k11_fits(q, u) ? q.uctl[u].nchunks * (uint32_t)sizeof(TableRec) : 0u);
    }
    scan_local_body(count + 1, [&](uint32_t) { return v; }, t.sz_offs, t.sz_tiles);
}
SB_DEVICE void k14_size_tiles_body(const TableBatchPlan& t) { scan_tiles_body(t.q.b.count + 1, 0, t.sz_tiles); }

// threads [0, max_chunks): chunk slots; threads [max_chunks, max_chunks + count]: units (the last writes the total)
SB_DEVICE void k14_export_body(const TableBatchPlan& t) {
    const FrameDecodeBatchPlan& q = t.q;
    const uint32_t count = q.b.count;
    const uint64_t slots = k11_slots(q), items = (uint64_t)q.max_chunks + count + 1;
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = (uint64_t)block_idx() * block_dim() + thread_idx(); g < items; g += nthreads) {
        if (g < q.max_chunks) {
            if (g >= slots) continue;
            const uint32_t u = k11_live_unit(q, g);
            if (u == K11_NONE) continue;
            const uint64_t r = k11_range(q, u);
            const FChunk c = q.chunks[g];
            TableRec rec;
            rec.body_off = c.body_off; rec.body_len = c.body_len; rec.dlen = c.dlen; rec.want_crc = c.want_crc;
            rec.type = c.type; rec.off = k11_out_at(q, g) - k11_out_at(q, r);
            TableHead* h = (TableHead*)(t.tables + k14_table_at(t, u));
            ((TableRec*)(h + 1))[g - r] = rec;
            continue;
        }
        const uint32_t u = (uint32_t)(g - q.max_chunks);
        const uint64_t at = k14_table_at(t, u);
        t.table_offs[u] = at;
        if (u == count) continue;
        TableHead h;
        sb_frame_result res;
        h.magic = K13_MAGIC; h.n = unit_in_len(q.b, u);
        if (k11_fits(q, u)) {
            const FrameUnitCtl& c = q.uctl[u];
            h.total = k11_need(q, u); h.nchunks = c.nchunks;
            h.full = c.walk_err.code == SB_E_INVALID && c.walk_err.b == 1 ? 1u : 0u;
            h.walk_err = c.walk_err;
            h.walk_err._pad = 0;
        } else {
            h.total = 0; h.nchunks = 0; h.full = 1;
            set_status(&h.walk_err, SB_E_INVALID, q.max_chunks, 1, 0);
        }
        *(TableHead*)(t.tables + at) = h;
        res.status = h.walk_err; res.bytes = h.total; res.nchunks = h.nchunks; res._pad = 0;
        t.results[u] = res;
    }
}

}  // namespace sbk
