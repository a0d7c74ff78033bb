// emu_table_gather.cpp -- TEST TOOLING ONLY. The gathers over tabled frame and raw streams (the k17_* bodies of
// rust-snappy_b200/csrc/k17_table_gather.cuh with the K13 and K15 plan, decode and finish bodies they run) compiled by
// g++ against the fiber warp emulator, exposed to tests/test_table_gather_emu.py through a C interface. The tables are
// built, and the range calls run, by the harnesses of tests/emu/emu_frame_table.cpp and tests/emu/emu_raw_table.cpp.
// Built by that test into tests/emu/_build/libemu_table_gather.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k17_table_gather.cuh"

typedef sbk::TablePlan F;
typedef sbk::RawRangePlan R;
typedef sbk::GatherPlan<F> GF;
typedef sbk::GatherPlan<R> GR;
static void fplan_entry(void* a) { sbk::k13_plan_body(((GF*)a)->q); }
static void fplan_tiles_entry(void* a) { sbk::k13_plan_tiles_body(((GF*)a)->q); }
static void rplan_entry(void* a) { sbk::k15_plan_body(((GR*)a)->q); }
static void rplan_tiles_entry(void* a) { sbk::k15_plan_tiles_body(((GR*)a)->q); }
template <class G> static void clear_entry(void* a) { sbk::k17_clear_body(*(G*)a); }
template <class G> static void insert_entry(void* a) { sbk::k17_insert_body(*(G*)a); }
template <class G> static void scan_local_entry(void* a) { sbk::k17_scan_local_body(*(G*)a); }
template <class G> static void scan_tiles_entry(void* a) { sbk::k17_scan_tiles_body(*(G*)a); }
template <class G> static void fill_entry(void* a) { sbk::k17_fill_body(*(G*)a); }
static void finterior_entry(void* a) { sbk::k13_decode_body<true>(((GF*)a)->q); }
static void rinterior_entry(void* a) { sbk::k15_decode_body<true>(((GR*)a)->q); }
static void fgather_entry(void* a) { sbk::k17_frame_gather_body(*(GF*)a); }
static void rgather_entry(void* a) { sbk::k17_raw_gather_body(*(GR*)a); }
static void ffinish_entry(void* a) { sbk::k13_finish_body<true>(((GF*)a)->q); }
static void rfinish_entry(void* a) { sbk::k15_finish_body(((GR*)a)->q); }

// the call checks of gather_call in csrc/snapb200.cu, the carve, the plan's arguments
template <class P>
static int setup(sbk::GatherPlan<P>* g, const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                 uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len, uint8_t* const* outs,
                 uint64_t* out_lens, sb_error* statuses, uint32_t nranges, void* scratch, uint64_t scratch_bytes) {
    if (count >= sbk::K13_MAX_COUNT || nranges > sbk::K17_MAX_RANGES) return 202;
    if (nranges == 0) return 0;
    if (count && (!tables || !ins || !in_lens)) return 202;
    if (!unit || !lo || !len || !outs || !out_lens || !statuses || !scratch) return 202;
    if (scratch_bytes < sbk::k17_carve<P>(nullptr, nranges, nullptr)) return 202;
    memset(g, 0, sizeof *g);
    P& q = g->q;
    q.tables = tables; q.ins = ins; q.in_lens = in_lens; q.count = count;
    q.unit = unit; q.lo = lo; q.len = len; q.outs = outs; q.out_lens = out_lens; q.statuses = statuses;
    sbk::k17_carve(scratch, nranges, g);
    return -1;
}

// launch_gather_lists, with small grids (every grid-stride loop takes several turns)
template <class G>
static void lists(G* g) {
    const unsigned stiles = (unsigned)(((uint64_t)g->nh + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(2, 64, 0, clear_entry<G>, g);
    sbemu::launch(2, 64, 0, insert_entry<G>, g);
    sbemu::launch(stiles, sbk::K4_TILE, 128, scan_local_entry<G>, g);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry<G>, g);
    sbemu::launch(2, 64, 0, fill_entry<G>, g);
}

extern "C" {

uint64_t emu_frame_table_gather_scratch_bytes(uint32_t nranges) { return sbk::k17_carve<F>(nullptr, nranges, nullptr); }
uint64_t emu_raw_table_gather_scratch_bytes(uint32_t nranges) { return sbk::k17_carve<R>(nullptr, nranges, nullptr); }
uint32_t emu_gather_group(void) { return sbk::K17_GROUP; }

// sb_frame_table_gather_device_ws under the emulator: the launch sequence of launch_frame_table_gather with small grids
// and 4 decoding warps, so that work items grid-stride over the pool's slots. *decodes: the chunk decodes of the call
// (interior and gather, not the finish's).
int emu_frame_table_gather(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens, uint32_t count,
                           const uint32_t* unit, const uint64_t* lo, const uint64_t* len, uint8_t* const* outs,
                           uint64_t* out_lens, sb_error* statuses, uint32_t nranges, void* scratch, uint64_t scratch_bytes,
                           uint64_t* decodes) {
    GF g;
    const int rc = setup(&g, tables, ins, in_lens, count, unit, lo, len, outs, out_lens, statuses, nranges, scratch,
                         scratch_bytes);
    if (rc >= 0) return rc;
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const uint32_t smem = sbk::K3_TABLE_BYTES + 2 * sbk::K2_SMEM_PER_WARP;
    sbemu::launch(ptiles, sbk::K4_TILE, 128, fplan_entry, &g);
    sbemu::launch(1, 1024, 1024 * 8, fplan_tiles_entry, &g);
    lists(&g);
    sbk::g_emu_decodes = 0;
    sbemu::launch(2, 64, smem + 2 * sizeof(sb_error), finterior_entry, &g);
    sbemu::launch(2, 64, smem + 2 * sizeof(sb_error), fgather_entry, &g);
    if (decodes) *decodes = sbk::g_emu_decodes;
    sbemu::launch(2, 64, smem, ffinish_entry, &g);
    return 0;
}

// sb_raw_table_gather_device_ws under the emulator: the launch sequence of launch_raw_table_gather, as above
int emu_raw_table_gather(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens, uint32_t count,
                         const uint32_t* unit, const uint64_t* lo, const uint64_t* len, uint8_t* const* outs,
                         uint64_t* out_lens, sb_error* statuses, uint32_t nranges, void* scratch, uint64_t scratch_bytes,
                         uint64_t* decodes) {
    GR g;
    const int rc = setup(&g, tables, ins, in_lens, count, unit, lo, len, outs, out_lens, statuses, nranges, scratch,
                         scratch_bytes);
    if (rc >= 0) return rc;
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const uint32_t smem = sbk::K3_TABLE_BYTES + 2 * sbk::K2_SMEM_PER_WARP;
    sbemu::launch(ptiles, sbk::K4_TILE, 128, rplan_entry, &g);
    sbemu::launch(1, 1024, 1024 * 8, rplan_tiles_entry, &g);
    lists(&g);
    sbk::g_emu_decodes = 0;
    sbemu::launch(2, 64, smem, rinterior_entry, &g);
    sbemu::launch(2, 64, smem, rgather_entry, &g);
    if (decodes) *decodes = sbk::g_emu_decodes;
    sbemu::launch(2, 32, 0, rfinish_entry, &g);
    return 0;
}

}
