// k16_encode_tables.cuh -- K16: seek tables written by the batch encoders (sb_compress_batch_tabled_device_ws,
// sb_frame_encode_batch_tabled_device_ws).
//
// The batch encoders already know everything a seek table holds, so a tabled encode needs no pass over its output:
//   raw    K9's launch sequence unchanged, except that K1 (flags 0) also gets a `crcs` array of nk entries, carved after
//          K9's scratch; K1's emitter warp writes every entry's masked CRC-32C of its input bytes.
//   frame  K10's launch sequence unchanged (it already has K1's `crcs`).
// Then, over either plan:
//   k16_size_local  thread per unit: its table size, 64 + record size * blocks for a unit with output, 64 for any other;
//                   K4's generic scan over units (k16_size_tiles finishes it).
//   k16_raw_export / k16_frame_export
//                   thread per slot of the global slot list: its record; then thread per unit [0, count]: d_table_offs,
//                   the header, a single-block unit's one record and d_results.
//
// Record arithmetic. Block j of a unit of n input bytes decodes to [65536 j, min(65536 (j + 1), n)). Its masked CRC is
// crcs[count + g] for slot g (crcs[u] for a single-block unit u). Raw: its compressed bytes start at hl + bo[g] -
// bo[first slot of u], hl the varint header length (K9's gather puts them there). Frame: its chunk header starts at
// 10 + bo[g] - bo[first slot of u] (K10's gather), so the body starts 8 bytes later, and holds the stored input (type 1,
// n_j bytes) when K4_CHUNK_RAW(c, n_j), else the c compressed bytes (type 0).
//
// Why these are the builds' tables. A raw build (K15) of a unit's output reads the same header, so hl and dn agree; K8's
// cuts are the block starts of the stream, which are where K9 placed the blocks, and the build decodes each block to
// the encoder's input, so its CRCs are K1's. The build marks the stream seekable: every block decodes Ok alone. The one
// exception is a stream K8 declines to split because one of its segments needs more than 1,024 merge elements: the
// build then says "not split" (reason 3), while the encoder, knowing its own cuts, writes a seekable table whose reads
// are correct. A frame build (K14) of a unit's output walks or indexes exactly the chunks K10 wrote, each of which
// passes K5's chunk check, so its records are the ones above, its total is n and its walk status is Ok. A unit without
// output (rejected, or empty in frame mode) is a 0-byte stream: the raw build reads no header (not seekable, reason 1,
// result Invalid{u, 0, 5}); the frame build finds no chunk (an empty table, Ok). Every field, padding included, is
// written explicitly.
#pragma once
#include "k10_frame_batch_encode.cuh"
#include "k13_frame_table.cuh"
#include "k15_raw_table.cuh"

namespace sbk {

struct EncodeTablesPlan {
    FrameBatchPlan f;                  // K10's plan (raw: only f.r and f.crcs are used)
    uint8_t* tables;                   // 8-byte aligned, the tables back to back
    uint64_t* table_offs;              // count + 1
    sb_frame_result* results;          // count
    uint64_t *sz_offs, *sz_tiles;      // scan over units of their table sizes
};

// the size scan's arrays, from `base` on (null: just the size)
inline uint64_t k16_carve_sizes(uintptr_t base, uint32_t count, EncodeTablesPlan* t) {
    const uint64_t units = (uint64_t)count + 1;
    const uint64_t offs = ((units + 1) * 8 + 255) / 256 * 256, tiles = ((units / K4_TILE + 3) * 8 + 255) / 256 * 256;
    if (t) { t->sz_offs = (uint64_t*)base; t->sz_tiles = (uint64_t*)(base + offs); }
    return offs + tiles;
}
// Raw: K9's carve, then K1's CRCs and the size scan. Returns the bytes used, or UINT64_MAX as k9_carve does.
inline uint64_t k16_raw_carve(void* scratch, uint32_t count, uint64_t in_bytes, EncodeTablesPlan* t) {
    const uint64_t k9 = k9_carve(scratch, count, in_bytes, t ? &t->f.r : nullptr);
    if (k9 == ~0ull) return k9;
    const uint64_t nk = (uint64_t)count + k9_slot_bound(count, in_bytes);
    const uintptr_t base = ((uintptr_t)scratch + k9 + 255) / 256 * 256;
    const uint64_t crcs = (nk * 4 + 255) / 256 * 256;
    if (t) t->f.crcs = (uint32_t*)base;
    return k9 + crcs + k16_carve_sizes(base + crcs, count, t) + 256;
}
// Frame: K10's carve, then the size scan.
inline uint64_t k16_frame_carve(void* scratch, uint32_t count, uint64_t in_bytes, EncodeTablesPlan* t) {
    const uint64_t k10 = k10_carve(scratch, count, in_bytes, t ? &t->f : nullptr);
    if (k10 == ~0ull) return k10;
    const uintptr_t base = ((uintptr_t)scratch + k10 + 255) / 256 * 256;
    return k10 + k16_carve_sizes(base, count, t) + 256;
}

// the bound on the packed tables' total: a header per unit and a record per single-block unit or slot
inline uint64_t k16_raw_tables_bytes(uint32_t count, uint64_t in_bytes) {
    return (uint64_t)count * sizeof(RawTableHead) + ((uint64_t)count + k9_slot_bound(count, in_bytes)) * sizeof(RawTableRec);
}
inline uint64_t k16_frame_tables_bytes(uint32_t count, uint64_t in_bytes) {
    return (uint64_t)count * sizeof(TableHead) + ((uint64_t)count + k9_slot_bound(count, in_bytes)) * sizeof(TableRec);
}

// unit u was written: a raw unit that passed the checks (an empty one is the 1-byte stream "\0"), a frame unit of at
// least one chunk; a multi-block unit only when the batch is within its bound
SB_DEVICE bool k16_written(const RawCompressPlan& r, uint32_t u, bool frame) {
    const uint32_t c = r.cls[u];
    return c == K9_SINGLE || (c == K9_MULTI && !k9_over(r)) || (!frame && c == K9_EMPTY);
}
SB_DEVICE uint64_t k16_table_at(const EncodeTablesPlan& t, uint32_t u) { return k8b_at(t.sz_offs, t.sz_tiles, u); }

// Σ sizes of a tile stays below 2^32: at most 1,024 headers and 1,024 * 56,176 records of at most 32 bytes
template <bool FRAME>
SB_DEVICE void k16_size_local_body(const EncodeTablesPlan& t) {
    const RawCompressPlan& r = t.f.r;
    const uint32_t count = r.b.count, rec = FRAME ? (uint32_t)sizeof(TableRec) : (uint32_t)sizeof(RawTableRec);
    const uint64_t i = (uint64_t)block_idx() * K4_TILE + thread_idx();
    uint32_t v = 0;
    if (i < count) {
        const uint32_t u = (uint32_t)i;
        v = 64u + (k16_written(r, u, FRAME) ? k10_chunks(unit_in_len(r.b, u)) * rec : 0u);
    }
    scan_local_body(count + 1, [&](uint32_t) { return v; }, t.sz_offs, t.sz_tiles);
}
SB_DEVICE void k16_size_tiles_body(const EncodeTablesPlan& t) { scan_tiles_body(t.f.r.b.count + 1, 0, t.sz_tiles); }

// items [0, nslot): slots; items [nslot, nslot + count]: units (the last writes the total)
SB_DEVICE void k16_raw_export_body(const EncodeTablesPlan& t) {
    const RawCompressPlan& r = t.f.r;
    const uint32_t count = r.b.count;
    const uint64_t slots = k8b_at(r.sl_offs, r.sl_tiles, count), items = (uint64_t)r.nslot + count + 1;
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = (uint64_t)block_idx() * block_dim() + thread_idx(); g < items; g += nthreads) {
        if (g < r.nslot) {
            if (g >= slots) continue;
            const uint32_t u = k8b_unit_of(r.sl_offs, r.sl_tiles, count, g);
            const uint64_t first = k8b_at(r.sl_offs, r.sl_tiles, u);
            RawTableRec rec;
            rec.off = (uint32_t)(k9_varint_len(unit_in_len(r.b, u)) + k8b_at(r.bo_offs, r.bo_tiles, g) -
                                 k8b_at(r.bo_offs, r.bo_tiles, first));
            rec.crc = t.f.crcs[count + g];
            ((RawTableRec*)(t.tables + k16_table_at(t, u) + sizeof(RawTableHead)))[g - first] = rec;
            continue;
        }
        const uint32_t u = (uint32_t)(g - r.nslot);
        const uint64_t at = k16_table_at(t, u);
        t.table_offs[u] = at;
        if (u == count) continue;
        const bool w = k16_written(r, u, false);
        const uint64_t n = unit_in_len(r.b, u);
        RawTableHead h;
        h.magic = K15_MAGIC; h.n = r.b.out_lens[u];
        h.dn = w ? n : 0; h.hl = w ? k9_varint_len(n) : 0; h.nblocks = w ? k10_chunks(n) : 0;
        h.seekable = w ? 1u : 0u; h.reason = w ? K15_SEEKABLE : K15_BAD_HEADER; h._pad[0] = h._pad[1] = h._pad[2] = 0;
        *(RawTableHead*)(t.tables + at) = h;
        if (w && r.cls[u] == K9_SINGLE) {
            RawTableRec rec;
            rec.off = h.hl; rec.crc = t.f.crcs[u];
            *(RawTableRec*)(t.tables + at + sizeof(RawTableHead)) = rec;
        }
        sb_frame_result res;
        if (w) set_status(&res.status, SB_OK, 0, 0, 0);
        else set_status(&res.status, SB_E_INVALID, u, 0, 5);
        res.bytes = h.dn; res.nchunks = h.nblocks; res._pad = 0;
        t.results[u] = res;
    }
}

SB_DEVICE TableRec k16_frame_rec(uint64_t hdr_at, uint32_t n, uint32_t c, uint32_t crc, uint64_t off) {
    const bool raw = K4_CHUNK_RAW(c, n);
    TableRec rec;
    rec.body_off = hdr_at + K10_CHUNK_HDR; rec.body_len = raw ? n : c; rec.dlen = n; rec.want_crc = crc;
    rec.type = raw ? 1u : 0u; rec.off = off;
    return rec;
}

SB_DEVICE void k16_frame_export_body(const EncodeTablesPlan& t) {
    const RawCompressPlan& r = t.f.r;
    const uint32_t count = r.b.count;
    const uint64_t slots = k8b_at(r.sl_offs, r.sl_tiles, count), items = (uint64_t)r.nslot + count + 1;
    const uint64_t nthreads = (uint64_t)grid_dim() * block_dim();
    for (uint64_t g = (uint64_t)block_idx() * block_dim() + thread_idx(); g < items; g += nthreads) {
        if (g < r.nslot) {
            if (g >= slots) continue;
            const uint32_t u = k8b_unit_of(r.sl_offs, r.sl_tiles, count, g);
            const uint64_t first = k8b_at(r.sl_offs, r.sl_tiles, u), j = g - first;
            const uint64_t hdr = K10_IDENT + k8b_at(r.bo_offs, r.bo_tiles, g) - k8b_at(r.bo_offs, r.bo_tiles, first);
            ((TableRec*)(t.tables + k16_table_at(t, u) + sizeof(TableHead)))[j] =
                k16_frame_rec(hdr, r.k1_lens[count + g], r.k1_clens[count + g], t.f.crcs[count + g], j * kMaxBlock);
            continue;
        }
        const uint32_t u = (uint32_t)(g - r.nslot);
        const uint64_t at = k16_table_at(t, u);
        t.table_offs[u] = at;
        if (u == count) continue;
        const bool w = k16_written(r, u, true);
        const uint64_t n = unit_in_len(r.b, u);
        TableHead h;
        h.magic = K13_MAGIC; h.n = r.b.out_lens[u]; h.total = w ? n : 0; h.nchunks = w ? k10_chunks(n) : 0; h.full = 0;
        set_status(&h.walk_err, SB_OK, 0, 0, 0);
        *(TableHead*)(t.tables + at) = h;
        if (w && r.cls[u] == K9_SINGLE)
            *(TableRec*)(t.tables + at + sizeof(TableHead)) =
                k16_frame_rec(K10_IDENT, (uint32_t)n, r.k1_clens[u], t.f.crcs[u], 0);
        sb_frame_result res;
        res.status = h.walk_err; res.bytes = h.total; res.nchunks = h.nchunks; res._pad = 0;
        t.results[u] = res;
    }
}

}  // namespace sbk
