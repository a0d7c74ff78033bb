// k17_table_gather.cuh -- K17: many small byte ranges over tabled frame and raw streams in one call, every edge chunk
// decoded once (sb_frame_table_gather_device_ws, sb_raw_table_gather_device_ws).
//
// The range calls of K13 and K15 give every range two private 64 KiB staging slots and decode its head and tail chunk
// (the chunks straddling lo or end) into them, once per range. For point lookups, very many short ranges over many
// streams, that is 128 KiB of scratch per range and one decode of a whole chunk per range. The gather calls give the
// same result for every range with:
//   - the head and tail chunks, the edges, deduplicated over the call: an edge is keyed (unit << 32) | chunk, and each
//     key is decoded and checked once into a pool slot and serves every range it is an edge of, at most K17_GROUP per
//     work item (a key shared by more ranges gets ceil(count / K17_GROUP) items, so one hot key does not serialise the
//     call behind one warp);
//   - a staging pool of min(2 * nranges, 4096) slots, one per decoding warp, in place of the per-range slots.
// Interior chunks (inside [lo, end)) still decode straight into their range's buffer, once per range that holds them,
// and a chunk that is interior to one range and an edge of another is decoded once in each role.
//
// Launches (the same whatever count, nranges and the sharing pattern):
//   k13_plan / k15_plan, *_plan_tiles   unchanged: each range's verified run and K4's scan of the pair counts
//   k17_clear         the hash table (3 * nranges slots) emptied
//   k17_insert        thread per range: its head and tail edge (a pair that passes the record's bounds and is not
//                     inside [lo, end)) inserted by open addressing; the range's place in its slot's list by atomic_add
//   k17_scan_local/_tiles  K4's two-level scan over slots of the list lengths and of the work items per slot
//   k17_fill          thread per range: (range << 1) | side written to its slot's list, a CSR layout
//   interior decode   k13_decode_body<true> / k15_decode_body<true> on the range calls' grid: every pair inside
//                     [lo, end), straight into its range's buffer
//   k17_*_gather      warp per work item, grid-striding over the pool's warps: the edge decoded into the warp's slot
//                     and CRC-checked, then each range of the item gets its slice by a warp copy, or the chunk as its
//                     first failing one by atomic_min
//   finish            k13_finish_body<true>, warp per range on the pool's warps: first the middle pairs that are not
//                     inside [lo, end), which only a table whose offsets were tampered with has, decoded one after
//                     another into the warp's slot; then a failing chunk's status from a decode into that slot /
//                     k15_finish_body unchanged
// A range's result depends on which of its chunks fail, never on the order of the lists or the warps.
#pragma once
#include "k13_frame_table.cuh"
#include "k15_raw_table.cuh"

namespace sbk {

static const uint32_t K17_GROUP = 256;                 // ranges one work item serves at most
static const uint32_t K17_MAX_RANGES = 1u << 28;       // 3 * nranges hash slots and their scans stay below 2^32
static const uint64_t K17_EMPTY = ~0ull;               // a free hash slot (units are below 2^31)
static const uint32_t K17_NONE = 0xFFFFFFFFu;

template <class P>
struct GatherPlan {
    P q;                           // the range plan: q.staging is the pool
    uint32_t nh;                   // hash slots: 3 * nranges
    unsigned long long* keys;      // nh keys; the list scan's offsets reuse this array once the inserts are done
    uint32_t* cnt;                 // nh: ranges per slot
    uint32_t *eslot, *epos;        // 2 * nranges: the slot of each range's head and tail edge (K17_NONE) and its place
    uint64_t *l_offs, *l_tiles;    // scan over slots of cnt: where each slot's list starts
    uint64_t *i_offs, *i_tiles;    // scan over slots of ceil(cnt / K17_GROUP): each slot's first work item
    uint32_t* list;                // 2 * nranges: (range << 1) | side, grouped by slot
};

// Scratch of a gather: the range records and pair scan of K12's layout, the hash table, the edge lists and their scans,
// then the pool. Every array 256-byte aligned from `scratch` (null: just the size). Returns the bytes used:
// 108 * nranges bytes of bookkeeping, 64 KiB per pool slot and a few KiB of alignment and scan tiles.
template <class P>
inline uint64_t k17_carve(void* scratch, uint32_t nranges, GatherPlan<P>* g) {
    const uint64_t n = nranges, units = n + 1, nh = 3 * n, slots = nh + 1;
    const uintptr_t base = ((uintptr_t)scratch + 255) / 256 * 256;
    uint64_t at = 0;
    auto take = [&](uint64_t bytes) { const uint64_t a = at; at += (bytes + 255) / 256 * 256; return (void*)(base + a); };
    RangeRec* rec = (RangeRec*)take(n * sizeof(RangeRec));
    uint64_t* pr_offs = (uint64_t*)take((units + 1) * 8);
    uint64_t* pr_tiles = (uint64_t*)take((units / K4_TILE + 3) * 8);
    void* keys = take((slots + 1) * 8);                              // nh keys, then slots + 1 list offsets
    uint64_t* l_tiles = (uint64_t*)take((slots / K4_TILE + 3) * 8);
    uint64_t* i_offs = (uint64_t*)take((slots + 1) * 8);
    uint64_t* i_tiles = (uint64_t*)take((slots / K4_TILE + 3) * 8);
    uint32_t* cnt = (uint32_t*)take(nh * 4);
    uint32_t* eslot = (uint32_t*)take(2 * n * 4);
    uint32_t* epos = (uint32_t*)take(2 * n * 4);
    uint32_t* list = (uint32_t*)take(2 * n * 4);
    uint8_t* pool = (uint8_t*)take(k17_pool_slots(nranges) * K12_SLOT);
    if (g) {
        g->q.nranges = nranges; g->q.rec = rec; g->q.pr_offs = pr_offs; g->q.pr_tiles = pr_tiles; g->q.staging = pool;
        g->nh = (uint32_t)nh; g->keys = (unsigned long long*)keys; g->cnt = cnt; g->eslot = eslot; g->epos = epos;
        g->l_offs = (uint64_t*)keys; g->l_tiles = l_tiles; g->i_offs = i_offs; g->i_tiles = i_tiles; g->list = list;
    }
    return at + 256;
}

// ---- range r's edges. side 0: its first verified chunk, side 1: its last when it has two or more. An edge is a pair
// the interior decode leaves alone: its record keeps the build's bounds and it is not inside [lo, end).
SB_DEVICE bool k17_edge(const TablePlan& q, uint32_t r, uint32_t side, uint32_t* k) {
    const RangeRec rr = q.rec[r];
    if (rr.pairs <= side) return false;
    *k = side ? rr.first + rr.pairs - 1 : rr.first;
    const TableHead* h = (const TableHead*)q.tables[q.unit[r]];      // a range with pairs passed k13_head
    const TableRec t = k13_recs(h)[*k];
    const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->total);
    return k13_rec_ok(t, h->n, lo, end) && !(t.off >= lo && t.off + t.dlen <= end);
}
SB_DEVICE bool k17_edge(const RawRangePlan& q, uint32_t r, uint32_t side, uint32_t* k) {
    const RangeRec rr = q.rec[r];
    if (rr.pairs <= side) return false;
    const uint32_t j = side ? rr.first + rr.pairs - 1 : rr.first;
    *k = j;
    const RawTableHead* h = (const RawTableHead*)q.tables[q.unit[r]];   // a range with pairs passed k15_head
    const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->dn), off = (uint64_t)j << 16;
    const uint64_t dl = h->dn - off < 65536 ? h->dn - off : 65536;
    return k15_rec_ok(h, j) && !(off >= lo && off + dl <= end);
}

SB_DEVICE uint32_t k17_hash(unsigned long long key, uint32_t nh) {
    uint64_t x = key * 0x9E3779B97F4A7C15ull;
    x ^= x >> 29;
    return (uint32_t)(((x >> 32) * (uint64_t)nh) >> 32);
}

template <class P>
SB_DEVICE void k17_clear_body(const GatherPlan<P>& g) {
    const uint64_t nt = (uint64_t)grid_dim() * block_dim();
    for (uint64_t i = (uint64_t)block_idx() * block_dim() + thread_idx(); i < g.nh; i += nt) {
        g.keys[i] = K17_EMPTY;
        g.cnt[i] = 0;
    }
}

// thread per range: at most two keys, each found or claimed by linear probing (the table holds at most 2 * nranges keys
// in 3 * nranges slots, so a probe always ends)
template <class P>
SB_DEVICE void k17_insert_body(const GatherPlan<P>& g) {
    const uint64_t nt = (uint64_t)grid_dim() * block_dim();
    for (uint64_t r = (uint64_t)block_idx() * block_dim() + thread_idx(); r < g.q.nranges; r += nt) {
        for (uint32_t side = 0; side < 2; side++) {
            uint32_t k = 0, slot = K17_NONE, pos = 0;
            if (k17_edge(g.q, (uint32_t)r, side, &k)) {
                const unsigned long long key = ((unsigned long long)g.q.unit[r] << 32) | k;
                uint32_t s = k17_hash(key, g.nh);
                for (;;) {
                    const unsigned long long old = atomic_cas(&g.keys[s], K17_EMPTY, key);
                    if (old == K17_EMPTY || old == key) break;
                    s = s + 1 == g.nh ? 0 : s + 1;
                }
                slot = s;
                pos = atomic_add(&g.cnt[s], 1u);
            }
            g.eslot[2 * r + side] = slot;
            g.epos[2 * r + side] = pos;
        }
    }
}

// K4's scans over slots [0, nh]: list lengths into l_offs (over the keys, which no later kernel reads), work items into
// i_offs. One tile's sums stay below 2^32: at most 2 * nranges ranges in all.
template <class P>
SB_DEVICE void k17_scan_local_body(const GatherPlan<P>& g) {
    scan_local_body(g.nh + 1, [&](uint32_t i) { return i < g.nh ? g.cnt[i] : 0u; }, g.l_offs, g.l_tiles);
    syncthreads();
    scan_local_body(g.nh + 1, [&](uint32_t i) { return i < g.nh ? (g.cnt[i] + K17_GROUP - 1) / K17_GROUP : 0u; },
                    g.i_offs, g.i_tiles);
}
template <class P>
SB_DEVICE void k17_scan_tiles_body(const GatherPlan<P>& g) {
    scan_tiles_body(g.nh + 1, 0, g.l_tiles);
    syncthreads();
    scan_tiles_body(g.nh + 1, 0, g.i_tiles);
}

template <class P>
SB_DEVICE void k17_fill_body(const GatherPlan<P>& g) {
    const uint64_t nt = (uint64_t)grid_dim() * block_dim();
    for (uint64_t r = (uint64_t)block_idx() * block_dim() + thread_idx(); r < g.q.nranges; r += nt) {
        for (uint32_t side = 0; side < 2; side++) {
            const uint32_t s = g.eslot[2 * r + side];
            if (s != K17_NONE) g.list[k8b_at(g.l_offs, g.l_tiles, s) + g.epos[2 * r + side]] = (uint32_t)(r << 1) | side;
        }
    }
}

// work item i: its slot's list [a, b) of at most K17_GROUP ranges, and the range and side of the slot's first entry
// (every entry of a slot names the same unit and chunk)
struct GatherItem { uint64_t a, b; uint32_t r0, side0; };
template <class P>
SB_DEVICE GatherItem k17_item(const GatherPlan<P>& g, uint64_t i) {
    const uint32_t s = k8b_unit_of(g.i_offs, g.i_tiles, g.nh, i);
    const uint64_t l0 = k8b_at(g.l_offs, g.l_tiles, s), l1 = k8b_at(g.l_offs, g.l_tiles, s + 1);
    GatherItem it;
    it.a = l0 + (i - k8b_at(g.i_offs, g.i_tiles, s)) * K17_GROUP;
    it.b = it.a + K17_GROUP < l1 ? it.a + K17_GROUP : l1;
    const uint32_t e = g.list[l0];
    it.r0 = e >> 1; it.side0 = e & 1u;
    return it;
}

// ---- gather decode: warp w of the pool's warps on slot w. HOST (k18_host_gather.cuh): the edge's body is fetched into
// the warp's compressed slot cpool + w * K18_CSLOT first.
template <bool HOST = false>
SB_DEVICE void k17_frame_gather_body(const GatherPlan<TablePlan>& g, uint8_t* cpool = nullptr) {
    const TablePlan& q = g.q;
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const unsigned wpb = block_dim() >> 5;
    sb_error* sink = (sb_error*)(smem() + K3_TABLE_BYTES + wpb * K2_SMEM_PER_WARP) + warp_id();
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id();
    const uint64_t nw = k12_pool_warps((uint64_t)grid_dim() * wpb, q.nranges);
    if (w >= nw) return;
    uint8_t* slot = q.staging + w * K12_SLOT;
    uint8_t* const cslot = HOST ? cpool + w * K18_CSLOT : nullptr;
    const uint64_t items = k8b_at(g.i_offs, g.i_tiles, g.nh);
    for (uint64_t i = w; i < items; i += nw) {
        const GatherItem it = k17_item(g, i);
        const RangeRec r0 = q.rec[it.r0];
        const uint32_t k = it.side0 ? r0.first + r0.pairs - 1 : r0.first, u = q.unit[it.r0];
        const TableHead* h = (const TableHead*)q.tables[u];
        const TableRec t = k13_recs(h)[k];                              // its bounds passed k13_rec_ok at the insert
        K17_COUNT_DECODE();
        FChunk c = k13_chunk(t);
        const uint8_t* in = q.ins[u];
        if (HOST) { in = k18_body<true>(in + t.body_off, t.body_len, cslot); c.body_off = 0; }
        const uint32_t code = k5_decode_chunk(tab, elems, c, in, slot, sink);
        for (uint64_t e = it.a; e < it.b; e++) {
            const uint32_t r = g.list[e] >> 1;
            if (code != SB_OK) { if (lane_id() == 0) atomic_min(&q.rec[r].first_bad, k); continue; }
            const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->total);   // a non-negative slice (k13_rec_ok)
            const uint64_t a = t.off > lo ? t.off : lo, b = t.off + t.dlen < end ? t.off + t.dlen : end;
            warp_copy(q.outs[r] + (a - lo), slot + (a - t.off), (uint32_t)(b - a));
        }
        syncwarp();
    }
}

template <bool HOST = false>
SB_DEVICE void k17_raw_gather_body(const GatherPlan<RawRangePlan>& g, uint8_t* cpool = nullptr) {
    const RawRangePlan& q = g.q;
    uint32_t* tab = (uint32_t*)smem();                                // K3 slicing tables (4 KB)
    k3_build_tables(tab);
    uint32_t* elems = (uint32_t*)(smem() + K3_TABLE_BYTES) + warp_id() * 64;
    const unsigned wpb = block_dim() >> 5;
    const uint64_t w = (uint64_t)block_idx() * wpb + warp_id();
    const uint64_t nw = k12_pool_warps((uint64_t)grid_dim() * wpb, q.nranges);
    if (w >= nw) return;
    uint8_t* slot = q.staging + w * K12_SLOT;
    uint8_t* const cslot = HOST ? cpool + w * K18_CSLOT : nullptr;
    const uint64_t items = k8b_at(g.i_offs, g.i_tiles, g.nh);
    for (uint64_t i = w; i < items; i += nw) {
        const GatherItem it = k17_item(g, i);
        const RangeRec r0 = q.rec[it.r0];
        const uint32_t j = it.side0 ? r0.first + r0.pairs - 1 : r0.first, u = q.unit[it.r0];
        const RawTableHead* h = (const RawTableHead*)q.tables[u];       // block j passed k15_rec_ok at the insert
        const RawTableRec* t = k15_recs(h);
        const uint64_t off = (uint64_t)j << 16, dl = h->dn - off < 65536 ? h->dn - off : 65536;
        const uint32_t a = t[j].off, b = j + 1 < h->nblocks ? t[j + 1].off : (uint32_t)h->n;
        K17_COUNT_DECODE();
        const uint8_t* in = q.ins[u] + a;
        if (HOST) in = k18_body<true>(in, b - a, cslot);
        uint32_t code = k2_decode_stream<false>(in, b - a, slot, dl, nullptr, nullptr, elems);
        syncwarp();
        if (code == SB_OK && k3_warp_crc32c_masked(tab, slot, (uint32_t)dl) != t[j].crc) code = SB_CHECKSUM;
        for (uint64_t e = it.a; e < it.b; e++) {
            const uint32_t r = g.list[e] >> 1;
            if (code != SB_OK) { if (lane_id() == 0) atomic_min(&q.rec[r].first_bad, j); continue; }
            const uint64_t lo = q.lo[r], end = k12_end(lo, q.len[r], h->dn);
            const uint64_t s = off > lo ? off : lo, x = off + dl < end ? off + dl : end;
            warp_copy(q.outs[r] + (s - lo), slot + (s - off), (uint32_t)(x - s));
        }
        syncwarp();
    }
}

}  // namespace sbk
