// emu_frame_table_batch.cpp -- TEST TOOLING ONLY. Seek tables of a batch of frame streams (K11's index-part bodies of
// rust-snappy_b200/csrc/k11_frame_batch_decode.cuh, then the k14_* bodies of k14_frame_table_batch.cuh) compiled by g++
// against the fiber warp emulator, exposed to tests/test_frame_table_batch_emu.py through a C interface. Built by that
// test into tests/emu/_build/libemu_frame_table_batch.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k14_frame_table_batch.cuh"

typedef sbk::FrameDecodeBatchPlan Plan;
typedef sbk::TableBatchPlan TPlan;
static void plan_entry(void* a) { sbk::k11_plan_body(*(Plan*)a); }
static void plan_tiles_entry(void* a) { sbk::k11_plan_tiles_body(*(Plan*)a); }
static void survivors_entry(void* a) { sbk::k11_survivors_body(*(Plan*)a); }
static void stitch_entry(void* a) { sbk::k11_stitch_body(*(Plan*)a); }
static void link_entry(void* a) { sbk::k11_link_body(*(Plan*)a); }
static void count_entry(void* a) { sbk::k11_count_body(*(Plan*)a); }
static void range_tiles_entry(void* a) { sbk::k11_range_tiles_body(*(Plan*)a); }
static void emit_entry(void* a) { sbk::k11_emit_body(*(Plan*)a); }
static void parse_entry(void* a) { sbk::k11_parse_body(*(Plan*)a); }
static void fill_entry(void* a) { sbk::k11_fill_body(*(Plan*)a); }
static void oscan_local_entry(void* a) { sbk::k11_oscan_local_body(*(Plan*)a); }
static void oscan_tiles_entry(void* a) { sbk::k11_oscan_tiles_body(*(Plan*)a); }
static void size_local_entry(void* a) { sbk::k14_size_local_body(*(TPlan*)a); }
static void size_tiles_entry(void* a) { sbk::k14_size_tiles_body(*(TPlan*)a); }
static void export_entry(void* a) { sbk::k14_export_body(*(TPlan*)a); }

extern "C" {

uint64_t emu_frame_table_batch_bytes(uint32_t count, uint32_t max_chunks) { return sbk::k14_tables_bytes(count, max_chunks); }
uint64_t emu_frame_table_build_batch_scratch_bytes(uint32_t count, uint64_t in_bytes, uint32_t max_chunks) {
    return sbk::k14_carve(nullptr, count, in_bytes, max_chunks, nullptr);
}

// sb_frame_table_build_batch_device_ws under the emulator: the call-level checks, the scratch layout of k14_carve and the
// launch sequence of launch_frame_table_build_batch in csrc/snapb200.cu (K11's index part, then K14), with small grids
// (so every grid-stride loop takes several turns). seg: K7 segment length (0: the library's default). Returns 202
// (SB_E_INVALID) where the library does.
int emu_frame_table_build_batch(const sb_batch* b, uint64_t in_bytes, uint32_t flags, const uint64_t* cidx,
                                const uint64_t* cidx_at, uint32_t max_chunks, void* tables, uint64_t tables_bytes,
                                uint64_t* table_offs, sb_frame_result* results, void* scratch, uint64_t scratch_bytes,
                                uint64_t seg) {
    if (!b || !tables || !table_offs || !results || !scratch) return 202;
    if (b->count >= sbk::K11_MAX_COUNT || !cidx != !cidx_at) return 202;
    if (max_chunks == 0 || max_chunks > sbk::K11_MAX_CHUNKS) return 202;
    if (b->count == 0) return 0;
    if (tables_bytes < sbk::k14_tables_bytes(b->count, max_chunks)) return 202;
    if (scratch_bytes < sbk::k14_carve(nullptr, b->count, in_bytes, max_chunks, nullptr)) return 202;
    TPlan t;
    memset(&t, 0, sizeof t);
    Plan& q = t.q;
    q.b = *b; q.fragment = flags & 1u; q.cidx = cidx; q.cidx_at = cidx_at; q.unit_chunks = nullptr;
    q.seg = seg ? (seg < sbk::K7_SEG_MIN ? sbk::K7_SEG_MIN : seg) : sbk::K7_SEG_DEFAULT;
    sbk::k14_carve(scratch, b->count, in_bytes, max_chunks, &t);
    t.tables = (uint8_t*)tables; t.table_offs = table_offs; t.results = results;
    const unsigned utiles = (unsigned)(((uint64_t)b->count + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const unsigned stiles = (unsigned)(((uint64_t)max_chunks + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    // K11's index part
    *q.in_total = 0;
    sbemu::launch(utiles, sbk::K4_TILE, 128, plan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, plan_tiles_entry, &q);
    if (cidx) {
        sbemu::launch(2, 64, 0, link_entry, &q);
    } else {
        sbemu::launch(2, 64, 0, survivors_entry, &q);
        sbemu::launch(b->count < 3 ? b->count : 3, sbk::K7_STITCH_THREADS, sbk::K7_STITCH_SMEM, stitch_entry, &q);
    }
    sbemu::launch(utiles, sbk::K4_TILE, 128, count_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, range_tiles_entry, &q);
    if (!cidx) sbemu::launch(2, 32, 0, emit_entry, &q);
    sbemu::launch(2, 64, 0, parse_entry, &q);
    sbemu::launch(2, 32, 0, fill_entry, &q);
    sbemu::launch(stiles, sbk::K4_TILE, 128, oscan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, oscan_tiles_entry, &q);
    // K14
    sbemu::launch(utiles, sbk::K4_TILE, 128, size_local_entry, &t);
    sbemu::launch(1, 1024, 1024 * 8, size_tiles_entry, &t);
    sbemu::launch(2, 64, 0, export_entry, &t);
    return 0;
}

}
