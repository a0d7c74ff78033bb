// emu_raw_batch.cpp -- TEST TOOLING ONLY. K8 over a batch of raw streams (the k8b_* bodies of
// rust-snappy_b200/csrc/k8_raw_split.cuh) compiled by g++ against the fiber warp emulator, exposed to
// tests/test_raw_batch_split_emu.py through a C interface. Built by that test into tests/emu/_build/libemu_raw_batch.so.
#define SB_EMU 1
#include "simt_emu.h"
#include "../../rust-snappy_b200/csrc/k8_raw_split.cuh"

static void plan_entry(void* a) { sbk::k8b_plan_body(*(sbk::RawBatchPlan*)a); }
static void plan_tiles_entry(void* a) { sbk::k8b_plan_tiles_body(*(sbk::RawBatchPlan*)a); }
static void chains_entry(void* a) { sbk::k8b_chains_body(*(sbk::RawBatchPlan*)a); }
static void merge_entry(void* a) { sbk::k8b_merge_body(*(sbk::RawBatchPlan*)a); }
static void stitch_entry(void* a) { sbk::k8b_stitch_body(*(sbk::RawBatchPlan*)a); }
static void counts_entry(void* a) { sbk::k8b_counts_body(*(sbk::RawBatchPlan*)a); }
static void scan_local_entry(void* a) { sbk::k8b_scan_local_body(*(sbk::RawBatchPlan*)a); }
static void scan_tiles_entry(void* a) { sbk::k8b_scan_tiles_body(*(sbk::RawBatchPlan*)a); }
static void cuts_entry(void* a) { sbk::k8b_cuts_body(*(sbk::RawBatchPlan*)a); }
static void blocks_entry(void* a) { sbk::k8b_blocks_body(*(sbk::RawBatchPlan*)a); }
static void finish_entry(void* a) { sbk::k8b_finish_body(*(sbk::RawBatchPlan*)a); }

extern "C" {

uint64_t emu_raw_batch_scratch_bytes(uint32_t count, uint64_t in_bytes) { return sbk::k8b_carve(nullptr, count, in_bytes, nullptr); }

// sb_decompress_batch_device_ws under the emulator: the scratch layout of k8b_carve and the launch sequence of
// launch_raw_batch in csrc/snapb200.cu, with small grids (so every grid-stride loop takes several turns). seg: segment
// length (0: the default). After the cuts, cut_at[i] (count entries) receives where unit i's cut table starts and
// cuts[0..cuts_cap) a copy of the cut array. Returns 202 (SB_E_INVALID) when the scratch is too small.
int emu_raw_batch_decode(const sb_batch* b, uint64_t in_bytes, uint32_t* unit_blocks, void* scratch, uint64_t scratch_bytes,
                         uint64_t seg, uint64_t* cut_at, uint32_t* cuts, uint64_t cuts_cap) {
    if (scratch_bytes < sbk::k8b_carve(nullptr, b->count, in_bytes, nullptr)) return 202;
    if (b->count == 0) return 0;
    sbk::RawBatchPlan q;
    memset(&q, 0, sizeof q);
    q.b = *b; q.seg = sbk::k8_seg_len(seg); q.unit_blocks = unit_blocks;
    sbk::k8b_carve(scratch, b->count, in_bytes, &q);
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
    if (cut_at)
        for (uint32_t i = 0; i < b->count; i++) cut_at[i] = sbk::k8b_at(q.bk_offs, q.bk_tiles, i) + i;
    if (cuts) memcpy(cuts, q.cut, cuts_cap * 4);
    sbemu::launch(3, 128, 4 * sbk::K2_SMEM_PER_WARP, blocks_entry, &q);
    sbemu::launch(2, 128, 4 * sbk::K2_SMEM_PER_WARP, finish_entry, &q);
    return 0;
}

}
