// emu_raw_table.cpp -- TEST TOOLING ONLY. Raw seek tables (K8b's split-part bodies of
// rust-snappy_b200/csrc/k8_raw_split.cuh, then the k15_* build bodies of k15_raw_table.cuh) and ranges over tabled raw
// streams (the k15_* read bodies) compiled by g++ against the fiber warp emulator, exposed to
// tests/test_raw_table_emu.py through a C interface. Built by that test into tests/emu/_build/libemu_raw_table.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k15_raw_table.cuh"

typedef sbk::RawBatchPlan Q;
typedef sbk::RawTableBuildPlan T;
typedef sbk::RawRangePlan R;
static void plan_entry(void* a) { sbk::k8b_plan_body(*(Q*)a); }
static void plan_tiles_entry(void* a) { sbk::k8b_plan_tiles_body(*(Q*)a); }
static void chains_entry(void* a) { sbk::k8b_chains_body(*(Q*)a); }
static void merge_entry(void* a) { sbk::k8b_merge_body(*(Q*)a); }
static void stitch_entry(void* a) { sbk::k8b_stitch_body(*(Q*)a); }
static void counts_entry(void* a) { sbk::k8b_counts_body(*(Q*)a); }
static void scan_local_entry(void* a) { sbk::k8b_scan_local_body(*(Q*)a); }
static void scan_tiles_entry(void* a) { sbk::k8b_scan_tiles_body(*(Q*)a); }
static void cuts_entry(void* a) { sbk::k8b_cuts_body(*(Q*)a); }
static void validate_entry(void* a) { sbk::k15_validate_body(*(T*)a); }
static void size_local_entry(void* a) { sbk::k15_size_local_body(*(T*)a); }
static void size_tiles_entry(void* a) { sbk::k15_size_tiles_body(*(T*)a); }
static void export_entry(void* a) { sbk::k15_export_body(*(T*)a); }
static void rplan_entry(void* a) { sbk::k15_plan_body(*(R*)a); }
static void rplan_tiles_entry(void* a) { sbk::k15_plan_tiles_body(*(R*)a); }
static void decode_entry(void* a) { sbk::k15_decode_body(*(R*)a); }
static void finish_entry(void* a) { sbk::k15_finish_body(*(R*)a); }

extern "C" {

uint64_t emu_raw_table_bytes(uint32_t nblocks) { return sbk::k15_table_bytes(nblocks); }
uint64_t emu_raw_table_batch_bytes(uint32_t count, uint64_t in_bytes) { return sbk::k15_tables_bytes(count, in_bytes); }
uint64_t emu_raw_table_build_batch_scratch_bytes(uint32_t count, uint64_t in_bytes) {
    return sbk::k15_carve(nullptr, count, in_bytes, nullptr);
}
uint64_t emu_raw_table_ranges_scratch_bytes(uint32_t nranges) { return sbk::k15_ranges_carve(nullptr, nranges, nullptr); }

// sb_raw_table_build_batch_device_ws under the emulator: the call-level checks, the scratch layout of k15_carve and the
// launch sequence of launch_raw_table_build_batch in csrc/snapb200.cu (K8b's split part, then K15), with small grids (so
// every grid-stride loop takes several turns). seg: K8 segment length (0: the default). Returns 202 (SB_E_INVALID) where
// the library does.
int emu_raw_table_build_batch(const sb_batch* b, uint64_t in_bytes, void* tables, uint64_t tables_bytes,
                              uint64_t* table_offs, sb_frame_result* results, void* scratch, uint64_t scratch_bytes,
                              uint64_t seg) {
    if (!b || !tables || !table_offs || !results || !scratch) return 202;
    if (b->count >= sbk::K8B_MAX_COUNT) return 202;
    if (b->count == 0) return 0;
    if (tables_bytes < sbk::k15_tables_bytes(b->count, in_bytes)) return 202;
    if (scratch_bytes < sbk::k15_carve(nullptr, b->count, in_bytes, nullptr)) return 202;
    sb_batch u;
    memset(&u, 0, sizeof u);
    u.in_ptrs = b->in_ptrs; u.in_base = b->in_base; u.in_stride = b->in_stride; u.in_lens = b->in_lens;
    u.in_len_uniform = b->in_len_uniform; u.out_cap_uniform = 0xFFFFFFFFu; u.count = b->count;
    T t;
    memset(&t, 0, sizeof t);
    Q& q = t.q;
    q.b = u; q.seg = sbk::k8_seg_len(seg); q.unit_blocks = nullptr;
    sbk::k15_carve(scratch, b->count, in_bytes, &t);
    t.tables = (uint8_t*)tables; t.table_offs = table_offs; t.results = results;
    // K8b's split part
    memset(q.bctl, 0, sizeof(sbk::RawBatchCtl));
    const unsigned utiles = (unsigned)(((uint64_t)b->count + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(utiles, sbk::K4_TILE, 128, plan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, plan_tiles_entry, &q);
    sbemu::launch(3, 128, 0, chains_entry, &q);
    sbemu::launch(3, 128, 0, merge_entry, &q);
    sbemu::launch(b->count < 3 ? b->count : 3, sbk::K8_STITCH_THREADS, sbk::K8_STITCH_THREADS * 16 + 16, stitch_entry, &q);
    sbemu::launch(3, 128, 0, counts_entry, &q);
    const unsigned ctiles = (unsigned)(((uint64_t)q.nseg_cap + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(ctiles, sbk::K4_TILE, 128, scan_local_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, scan_tiles_entry, &q);
    sbemu::launch(3, 128, 0, cuts_entry, &q);
    // K15
    sbemu::launch(2, 96, sbk::K3_TABLE_BYTES + 3 * sbk::K2_SMEM_PER_WARP, validate_entry, &t);
    sbemu::launch(utiles, sbk::K4_TILE, 128, size_local_entry, &t);
    sbemu::launch(1, 1024, 1024 * 8, size_tiles_entry, &t);
    sbemu::launch(2, 64, 0, export_entry, &t);
    return 0;
}

// sb_raw_table_decode_ranges_device_ws under the emulator: the call-level checks, the scratch layout and the launch
// sequence of launch_raw_table_ranges, with small grids. *staging_at: the staging's offset in the scratch.
int emu_raw_table_decode_ranges(const void* const* tables, const uint8_t* const* ins, const uint64_t* in_lens,
                                uint32_t count, const uint32_t* unit, const uint64_t* lo, const uint64_t* len,
                                uint8_t* const* outs, uint64_t* out_lens, sb_error* statuses, uint32_t nranges,
                                void* scratch, uint64_t scratch_bytes, uint64_t* staging_at) {
    if (count >= sbk::K15_MAX_COUNT || nranges >= sbk::K12_MAX_RANGES) return 202;
    if (nranges == 0) return 0;
    if (count && (!tables || !ins || !in_lens)) return 202;
    if (!unit || !lo || !len || !outs || !out_lens || !statuses || !scratch) return 202;
    if (scratch_bytes < sbk::k15_ranges_carve(nullptr, nranges, nullptr)) return 202;
    R q;
    memset(&q, 0, sizeof q);
    q.tables = tables; q.ins = ins; q.in_lens = in_lens; q.count = count;
    q.unit = unit; q.lo = lo; q.len = len; q.outs = outs; q.out_lens = out_lens; q.statuses = statuses;
    sbk::k15_ranges_carve(scratch, nranges, &q);
    if (staging_at) *staging_at = (uint64_t)(q.staging - (uint8_t*)scratch);
    const unsigned ptiles = (unsigned)(((uint64_t)nranges + 1 + sbk::K4_TILE - 1) / sbk::K4_TILE);
    sbemu::launch(ptiles, sbk::K4_TILE, 128, rplan_entry, &q);
    sbemu::launch(1, 1024, 1024 * 8, rplan_tiles_entry, &q);
    sbemu::launch(3, 64, sbk::K3_TABLE_BYTES + 2 * sbk::K2_SMEM_PER_WARP, decode_entry, &q);
    sbemu::launch(2, 32, 0, finish_entry, &q);
    return 0;
}

}
