// emu_table_gather_host.cpp -- TEST TOOLING ONLY. The host-stream gathers (the HOST instantiations of the K13, K15 and
// K17 decode bodies, rust-snappy_b200/csrc/k18_host_gather.cuh) compiled by g++ against the fiber warp emulator, exposed
// to tests/test_table_gather_host_emu.py through a C interface. The emulator has one address space, so "host" streams
// are plain buffers here: what the tests check is that the fetch policy gives the device gather's results at the
// documented cost. Built by that test into tests/emu/_build/libemu_table_gather_host.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k17_table_gather.cuh"

typedef sbk::TablePlan F;
typedef sbk::RawRangePlan R;
template <class P>
struct Host { sbk::GatherPlan<P> g; uint8_t* cpool; };
typedef Host<F> HF;
typedef Host<R> HR;
static void fplan_entry(void* a) { sbk::k13_plan_body(((HF*)a)->g.q); }
static void fplan_tiles_entry(void* a) { sbk::k13_plan_tiles_body(((HF*)a)->g.q); }
static void rplan_entry(void* a) { sbk::k15_plan_body(((HR*)a)->g.q); }
static void rplan_tiles_entry(void* a) { sbk::k15_plan_tiles_body(((HR*)a)->g.q); }
template <class H> static void clear_entry(void* a) { sbk::k17_clear_body(((H*)a)->g); }
template <class H> static void insert_entry(void* a) { sbk::k17_insert_body(((H*)a)->g); }
template <class H> static void scan_local_entry(void* a) { sbk::k17_scan_local_body(((H*)a)->g); }
template <class H> static void scan_tiles_entry(void* a) { sbk::k17_scan_tiles_body(((H*)a)->g); }
template <class H> static void fill_entry(void* a) { sbk::k17_fill_body(((H*)a)->g); }
static void finterior_entry(void* a) { sbk::k13_decode_body<true, true>(((HF*)a)->g.q, ((HF*)a)->cpool); }
static void rinterior_entry(void* a) { sbk::k15_decode_body<true, true>(((HR*)a)->g.q, ((HR*)a)->cpool); }
static void fgather_entry(void* a) { sbk::k17_frame_gather_body<true>(((HF*)a)->g, ((HF*)a)->cpool); }
static void rgather_entry(void* a) { sbk::k17_raw_gather_body<true>(((HR*)a)->g, ((HR*)a)->cpool); }
static void ffinish_entry(void* a) { sbk::k13_finish_body<true>(((HF*)a)->g.q); }
static void rfinish_entry(void* a) { sbk::k15_finish_body(((HR*)a)->g.q); }

template <class P>
static uint64_t scratch_bytes_of(uint32_t nranges) {
    return sbk::k18_carve(nullptr, sbk::k17_carve<P>(nullptr, nranges, nullptr), sbk::k17_pool_slots(nranges), nullptr);
}

// the call checks of gather_call in csrc/snapb200.cu with the host scratch, the carve, the plan's arguments
template <class P>
static int setup(Host<P>* h, const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                 uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len, uint8_t* const* outs,
                 uint64_t* out_lens, sb_error* statuses, uint32_t nranges, void* scratch, uint64_t scratch_bytes) {
    if (count >= sbk::K13_MAX_COUNT || nranges > sbk::K17_MAX_RANGES) return 202;
    if (nranges == 0) return 0;
    if (count && (!tables || !ins || !in_lens)) return 202;
    if (!unit || !lo || !len || !outs || !out_lens || !statuses || !scratch) return 202;
    if (scratch_bytes < scratch_bytes_of<P>(nranges)) return 202;
    memset(h, 0, sizeof *h);
    P& q = h->g.q;
    q.tables = tables; q.ins = ins; q.in_lens = in_lens; q.count = count;
    q.unit = unit; q.lo = lo; q.len = len; q.outs = outs; q.out_lens = out_lens; q.statuses = statuses;
    const uint64_t bytes = sbk::k17_carve(scratch, nranges, &h->g);
    sbk::k18_carve(scratch, bytes, sbk::k17_pool_slots(nranges), &h->cpool);
    return -1;
}

// launch_gather_lists, with small grids (every grid-stride loop takes several turns)
template <class H>
static void lists(H* h) {
    const unsigned stiles = (unsigned)(((uint64_t)h->g.nh + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(2, 64, 0, clear_entry<H>, h);
    sbemu::launch(2, 64, 0, insert_entry<H>, h);
    sbemu::launch(stiles, sbk::K4_TILE, 128, scan_local_entry<H>, h);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry<H>, h);
    sbemu::launch(2, 64, 0, fill_entry<H>, h);
}

extern "C" {

uint64_t emu_frame_table_gather_host_scratch_bytes(uint32_t nranges) { return scratch_bytes_of<F>(nranges); }
uint64_t emu_raw_table_gather_host_scratch_bytes(uint32_t nranges) { return scratch_bytes_of<R>(nranges); }
uint64_t emu_cslot_bytes(void) { return sbk::K18_CSLOT; }

// sb_frame_table_gather_host_streams_ws under the emulator: the launch sequence of launch_frame_table_gather with
// cpool, small grids and 4 warps, so that the pool's warps grid-stride. *decodes: the chunk decodes of the call (interior
// and gather, not the finish's); *fetched: the compressed bytes copied into slots.
int emu_frame_table_gather_host(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                                uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len,
                                uint8_t* const* outs, uint64_t* out_lens, sb_error* statuses, uint32_t nranges,
                                void* scratch, uint64_t scratch_bytes, uint64_t* decodes, uint64_t* fetched) {
    HF h;
    const int rc = setup(&h, tables, ins, in_lens, count, unit, lo, len, outs, out_lens, statuses, nranges, scratch,
                         scratch_bytes);
    if (rc >= 0) return rc;
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const uint32_t smem = sbk::K3_TABLE_BYTES + 2 * sbk::K2_SMEM_PER_WARP;
    sbemu::launch(ptiles, sbk::K4_TILE, 128, fplan_entry, &h);
    sbemu::launch(1, 1024, 1024 * 8, fplan_tiles_entry, &h);
    lists(&h);
    sbk::g_emu_decodes = 0;
    sbk::g_emu_fetched = 0;
    sbemu::launch(2, 64, smem + 2 * sizeof(sb_error), finterior_entry, &h);
    sbemu::launch(2, 64, smem + 2 * sizeof(sb_error), fgather_entry, &h);
    if (decodes) *decodes = sbk::g_emu_decodes;
    if (fetched) *fetched = sbk::g_emu_fetched;
    sbemu::launch(2, 64, smem, ffinish_entry, &h);
    return 0;
}

// sb_raw_table_gather_host_streams_ws under the emulator, as above
int emu_raw_table_gather_host(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                              uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len,
                              uint8_t* const* outs, uint64_t* out_lens, sb_error* statuses, uint32_t nranges,
                              void* scratch, uint64_t scratch_bytes, uint64_t* decodes, uint64_t* fetched) {
    HR h;
    const int rc = setup(&h, tables, ins, in_lens, count, unit, lo, len, outs, out_lens, statuses, nranges, scratch,
                         scratch_bytes);
    if (rc >= 0) return rc;
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    const uint32_t smem = sbk::K3_TABLE_BYTES + 2 * sbk::K2_SMEM_PER_WARP;
    sbemu::launch(ptiles, sbk::K4_TILE, 128, rplan_entry, &h);
    sbemu::launch(1, 1024, 1024 * 8, rplan_tiles_entry, &h);
    lists(&h);
    sbk::g_emu_decodes = 0;
    sbk::g_emu_fetched = 0;
    sbemu::launch(2, 64, smem, rinterior_entry, &h);
    sbemu::launch(2, 64, smem, rgather_entry, &h);
    if (decodes) *decodes = sbk::g_emu_decodes;
    if (fetched) *fetched = sbk::g_emu_fetched;
    sbemu::launch(2, 32, 0, rfinish_entry, &h);
    return 0;
}

}
