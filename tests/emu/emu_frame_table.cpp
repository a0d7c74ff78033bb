// emu_frame_table.cpp -- TEST TOOLING ONLY. Seek-table build and ranges over tabled streams (the k13_* bodies of
// rust-snappy_b200/csrc/k13_frame_table.cuh, the build behind K7's and K5's index-phase bodies) compiled by g++ against
// the fiber warp emulator, exposed to tests/test_frame_table_emu.py through a C interface. Built by that test into
// tests/emu/_build/libemu_frame_table.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k13_frame_table.cuh"
#include "../../rust-snappy_b200/csrc/k7_frame_index.cuh"

typedef sbk::TablePlan Plan;
struct ExportArgs { sbk::DecodePlan p; sbk::TableHead* t; };
static void k5_parse_entry(void* a) { sbk::k5_parse_body(*(sbk::DecodePlan*)a); }
static void k5_walk_entry(void* a) { sbk::k5_walk_body(*(sbk::DecodePlan*)a); }
static void k5_scan_local_entry(void* a) { sbk::k5_scan_local_body(*(sbk::DecodePlan*)a); }
static void k5_scan_tiles_entry(void* a) { sbk::k5_scan_tiles_body(*(sbk::DecodePlan*)a); }
static void k7_survivors_entry(void* a) { sbk::k7_survivors_body(*(sbk::IndexPlan*)a); }
static void k7_stitch_entry(void* a) { sbk::k7_stitch_body(*(sbk::IndexPlan*)a); }
static void k7_emit_entry(void* a) { sbk::k7_emit_body(*(sbk::IndexPlan*)a); }
static void export_entry(void* a) { sbk::k13_export_body(((ExportArgs*)a)->p, ((ExportArgs*)a)->t); }
static void plan_entry(void* a) { sbk::k13_plan_body(*(Plan*)a); }
static void plan_tiles_entry(void* a) { sbk::k13_plan_tiles_body(*(Plan*)a); }
static void decode_entry(void* a) { sbk::k13_decode_body(*(Plan*)a); }
static void finish_entry(void* a) { sbk::k13_finish_body(*(Plan*)a); }

static uint64_t up256(uint64_t v) { return (v + 255) / 256 * 256; }
// decode_ws_bytes of csrc/snapb200.cu
static uint64_t decode_ws_bytes(uint64_t m) {
    return up256(m * sizeof(sbk::FChunk) + 64) + up256((m + 1) * 8) + up256((m / sbk::K4_TILE + 3) * 8) +
           up256(m * sizeof(sb_error) + 64) + 512;
}

extern "C" {

uint64_t emu_frame_table_bytes(uint32_t nchunks) { return sbk::k13_table_bytes(nchunks); }
uint64_t emu_frame_table_build_scratch_bytes(uint32_t max_chunks) { return decode_ws_bytes(max_chunks); }
uint64_t emu_frame_table_ranges_scratch_bytes(uint32_t nranges) { return sbk::k13_carve(nullptr, nranges, nullptr); }

// sb_frame_table_build_device_ws under the emulator: the call-level checks, make_decode_plan's scratch layout and the
// launch sequence of launch_frame_table_build in csrc/snapb200.cu (decode_index_phase, then k13_export), with small
// grids. seg: K7 segment length (0: the library's default). Returns 202 (SB_E_INVALID) where the library does.
int emu_frame_table_build(const uint8_t* in, uint64_t n, const uint64_t* cidx, uint32_t nchunks, uint32_t flags,
                          void* table, uint64_t table_bytes, uint32_t max_chunks, sb_frame_result* result, void* scratch,
                          uint64_t scratch_bytes, uint64_t seg) {
    if ((!in && n) || !table || !result || !scratch) return 202;
    if (max_chunks == 0 || max_chunks > sbk::K12_MAX_CHUNKS) return 202;
    if (cidx && nchunks > max_chunks) return 202;
    if (table_bytes < sbk::k13_table_bytes(max_chunks) || scratch_bytes < decode_ws_bytes(max_chunks)) return 202;
    sbk::DecodePlan p;
    memset(&p, 0, sizeof p);
    uint8_t* w = (uint8_t*)up256((uint64_t)scratch);
    p.chunks = (sbk::FChunk*)w; w += up256((uint64_t)max_chunks * sizeof(sbk::FChunk) + 64);
    p.ooff = (uint64_t*)w; w += up256(((uint64_t)max_chunks + 1) * 8);
    p.tiles = (uint64_t*)w; w += up256(((uint64_t)max_chunks / sbk::K4_TILE + 3) * 8);
    p.statuses = (sb_error*)w; w += up256((uint64_t)max_chunks * sizeof(sb_error) + 64);
    p.ctl = (sbk::DecodeCtl*)w;
    p.in = in; p.n = n; p.index = cidx; p.index_n = cidx ? nchunks : 0; p.fragment = flags & 1u;
    p.cap_chunks = max_chunks; p.out = nullptr; p.cap = ~0ull; p.result = result;
    if (!cidx) { p.index = p.ooff; p.index_count = &p.ctl->index_count; }
    // decode_index_phase
    memset(p.ctl, 0, sizeof(sbk::DecodeCtl));
    if (p.index_count) {
        sbk::IndexPlan k = sbk::k7_plan_for_decode(p, seg ? seg : sbk::K7_SEG_DEFAULT);
        sbemu::launch(k.nseg ? (k.nseg + 3) / 4 : 1, 128, 0, k7_survivors_entry, &k);
        sbemu::launch(1, sbk::K7_STITCH_THREADS, sbk::K7_STITCH_SMEM, k7_stitch_entry, &k);
        sbemu::launch(k.nseg ? (k.nseg + 127) / 128 : 1, 128, 0, k7_emit_entry, &k);
    }
    if (p.index) {
        const uint64_t threads = p.index_count ? p.cap_chunks : p.index_n;
        sbemu::launch(threads ? (unsigned)((threads + 255) / 256) : 1, 256, 0, k5_parse_entry, &p);
    }
    sbemu::launch(1, 32, 0, k5_walk_entry, &p);
    const unsigned ntiles = (max_chunks + sbk::K4_TILE - 1) / sbk::K4_TILE;
    sbemu::launch(ntiles ? ntiles : 1, sbk::K4_TILE, 128, k5_scan_local_entry, &p);
    sbemu::launch(1, 1024, 1024 * 8, k5_scan_tiles_entry, &p);
    // K13's export: thread per slot plus the header's
    ExportArgs e;
    e.p = p; e.t = (sbk::TableHead*)table;
    sbemu::launch((unsigned)(((uint64_t)max_chunks + 1 + 255) / 256), 256, 0, export_entry, &e);
    return 0;
}

// sb_frame_table_decode_ranges_device_ws under the emulator: the call-level checks, the scratch layout and the launch
// sequence of launch_frame_table_ranges, with small grids (so every grid-stride loop takes several turns).
// *staging_at: the staging's offset in the scratch.
int emu_frame_table_decode_ranges(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                                  uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len,
                                  uint8_t* const* outs, uint64_t* out_lens, sb_error* statuses, uint32_t nranges,
                                  void* scratch, uint64_t scratch_bytes, uint64_t* staging_at) {
    if (count >= sbk::K13_MAX_COUNT || nranges >= sbk::K12_MAX_RANGES) return 202;
    if (nranges == 0) return 0;
    if (count && (!tables || !ins || !in_lens)) return 202;
    if (!unit || !lo || !len || !outs || !out_lens || !statuses || !scratch) return 202;
    if (scratch_bytes < sbk::k13_carve(nullptr, nranges, nullptr)) return 202;
    Plan q;
    memset(&q, 0, sizeof q);
    q.tables = tables; q.ins = ins; q.in_lens = in_lens; q.count = count;
    q.unit = unit; q.lo = lo; q.len = len; q.outs = outs; q.out_lens = out_lens; q.statuses = statuses;
    sbk::k13_carve(scratch, nranges, &q);
    *staging_at = (uint64_t)(q.staging - (uint8_t*)scratch);
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const uint32_t smem = sbk::K3_TABLE_BYTES + 4 * sbk::K2_SMEM_PER_WARP;
    sbemu::launch(ptiles, sbk::K4_TILE, 128, plan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, plan_tiles_entry, &q);
    sbemu::launch(2, 128, smem + 4 * sizeof(sb_error), decode_entry, &q);
    sbemu::launch(2, 128, smem, finish_entry, &q);
    return 0;
}

}
